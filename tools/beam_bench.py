"""Time ``ctc_crf.ctc_beam_search`` in both modes, with the den forward pass and the fused loss for scale, at the headline shape.

    python tools/beam_bench.py [--N 64] [--T 1500] [--V 218] [--B 1,16,64,128] [--cutoff 40] [--rounds 5] [--reps 3]

N=64 utterances of T=1500 frames, V=218.  The den graph is a CTC-shaped T o LM graph of 1.10 M arcs (a deterministic random
phone LM of 1800 states with 24 successors each, composed with the CTC topology): crf mode needs a graph whose LM states
have no two successors of one label, which the synthetic graph bench.py measures does not satisfy.  Every case is timed
with CUDA events after a warm-up, in alternation round by round, and the card's name, power limit and maximum SM clock are
printed next to the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctc_crf  # noqa: E402
from cat_b200 import _C, _lib, fst  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:   # the numbers stand without it, but say so
        out = f"nvidia-smi unavailable ({e})"
    return torch.cuda.get_device_name(0), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=64)
    ap.add_argument("--T", type=int, default=1500)
    ap.add_argument("--V", type=int, default=218)
    ap.add_argument("--B", default="1,16,64,128")
    ap.add_argument("--cutoff", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="calls per timed window")
    a = ap.parse_args()
    Bs = [int(b) for b in a.B.split(",")]
    tmp = tempfile.mkdtemp(prefix="beam_bench_")
    path = os.path.join(tmp, "den.fst")
    fst.write_fst(path, fst.compose_ctc_lm(fst.make_random_lm(H=1800, V=a.V, d=24, seed=1)))
    ctx = ctc_crf.CRFContext(path, gpus=0)
    N, T, V = a.N, a.T, a.V
    g = torch.Generator(device="cuda").manual_seed(1)
    x = 3.0 * torch.randn((N, T, V), device="cuda", generator=g)
    y = torch.log_softmax(x, -1).contiguous()
    lx = torch.full((N,), T, dtype=torch.int32)
    ly = torch.full((N,), T // 6, dtype=torch.int32)
    labels = torch.randint(1, V, (int(ly.sum()),), dtype=torch.int32)
    L = _lib.lib()
    lx_d = lx.cuda()
    alpha = torch.empty(int(L.ccb_den_alpha_floats(N, T)), dtype=torch.float32, device="cuda")
    aux = torch.empty(int(L.ccb_den_aux_bytes(N, T)), dtype=torch.uint8, device="cuda")
    logz = torch.empty(N, dtype=torch.float32, device="cuda")

    def den_forward():
        rc = L.ccb_den_forward_backward(y.data_ptr(), 0, T * V, V, N, T, V, lx_d.data_ptr(), alpha.data_ptr(), aux.data_ptr(),
                                        None, 0, 0, 0.0, logz.data_ptr(), None,
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, _lib.last_error()

    def loss():
        _C.ctc_crf_loss_fwd(y, labels, lx, ly, 0.01, True)

    cases = [(f"beam {'crf' if crf else 'plain'} B={b}", (lambda b=b, crf=crf: ctc_crf.ctc_beam_search(y, lx, b, a.cutoff, crf)))
             for crf in (False, True) for b in Bs]
    cases += [("den forward", den_forward), ("fused loss + gradient", loss)]
    for _, fn in cases:      # warm-up (the first crf call checks the graph and uploads its out-arc table)
        fn()
    torch.cuda.synchronize()
    times = {name: [] for name, _ in cases}
    for _ in range(a.rounds):
        for name, fn in cases:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.reps)
    name, smi = card()
    res = {"card": name, "nvidia_smi(name,power.limit,clocks.max.sm)": smi, "N": N, "T": T, "V": V, "cutoff_top_n": a.cutoff,
           "den_arcs": _C.den_info()["file_arcs"],
           "ms": {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in times.items()}}
    print(json.dumps(res, indent=1))
    del ctx


if __name__ == "__main__":
    main()
