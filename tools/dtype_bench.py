"""The fused CTC-CRF loss (`_C.ctc_crf_loss_fwd`, loss plus gradient) by logits dtype, on one GPU, at the headline shape:
1.02 M-arc den graph (H=20 000), N=64, T=1500, V=218.

Six arms: fp32, bf16 and fp16 logits, each as log-probs and as raw encoder outputs (from_logits=True).  The raw logits are
z = 3 randn, the log-probs log_softmax(z), both made in fp32 and rounded once to the arm's dtype.  Each call is timed with
CUDA events; the arms are alternated call by call (--reps of each, after one warm-up call of each).  The card's name, power
limit and max SM clock are read in the same run (nvidia-smi, query only).

Prints one JSON line.  Usage: python tools/dtype_bench.py [--reps 5]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if args.reps < 3:
        ap.error("--reps must be at least 3")
    if not torch.cuda.is_available():
        raise SystemExit("dtype_bench needs a CUDA device")
    import ctc_crf
    from cat_b200 import _C, fst
    from bench import synth_labels
    from fwd_only_bench import card
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    H, N, T, V, lamb, seed = 20000, 64, 1500, 218, 0.01, 1234
    path = os.path.join(tempfile.mkdtemp(prefix="dtype_bench_"), f"den_{H}.fst")
    fst.write_fst(path, fst.make_synthetic_den(H, 24, V, seed=7))
    ctx = ctc_crf.CRFContext(path, gpus=0)
    lab, lens, ly = synth_labels(N, T, V, seed)
    lab, lx, ly = torch.tensor(lab), torch.tensor(lens), torch.tensor(ly)
    g = torch.Generator(device=dev).manual_seed(seed)
    z = 3.0 * torch.randn(N, T, V, device=dev, generator=g)
    y = torch.log_softmax(z, -1)
    dtypes = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
    arms = {}
    for dname, dt in dtypes.items():
        arms[f"{dname}_logprobs"] = (y.to(dt).contiguous(), False)
        arms[f"{dname}_raw"] = (z.to(dt).contiguous(), True)

    def call(name):
        x, from_logits = arms[name]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        loss, grad, _ = _C.ctc_crf_loss_fwd(x, lab, lx, ly, lamb, True, from_logits=from_logits)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), float(loss.item())

    for name in arms:       # warm-up (allocator, kernel attributes)
        call(name)
    ms = {k: [] for k in arms}
    loss = {}
    for _ in range(args.reps):
        for name in arms:
            t, loss[name] = call(name)
            ms[name].append(round(t, 3))
    med = {k: statistics.median(v) for k, v in ms.items()}
    out = {
        "card": card(), "graph_arcs": int(_C.den_info()["file_arcs"]), "N": N, "T": T, "V": V, "reps": args.reps,
        "timing": "CUDA events per _C.ctc_crf_loss_fwd call (loss + gradient), arms alternated, median of reps",
        "ms": ms, "median_ms": med,
        "f16_over_bf16": {k: med[f"f16_{k}"] / med[f"bf16_{k}"] for k in ("logprobs", "raw")},
        "f16_over_f32": {k: med[f"f16_{k}"] / med[f"f32_{k}"] for k in ("logprobs", "raw")},
        "loss": loss,
    }
    del ctx
    print(json.dumps(out))


if __name__ == "__main__":
    main()
