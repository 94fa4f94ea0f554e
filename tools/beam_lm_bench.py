"""Time ``ctc_crf.ctc_beam_search`` without and with a token n-gram LM fused in, and the ARPA loader.

    python tools/beam_lm_bench.py [--N 64] [--T 1500] [--B 1,16,64,128] [--cutoff 40] [--rounds 5] [--reps 3]

N = 64 utterances of T = 1500 frames, cutoff_top_n = 40, alpha 0.25, beta -0.5 (CAT's CTC-CRF template recipe).  Two LMs,
written by ``ngram.make_random_arpa``: V = 218 with a 3-gram of about 0.5 M n-grams (a phone or small token inventory), and
V = 5000 with a 4-gram of about 1.4 M n-grams once suffix-closed (a BPE vocabulary).  For each B the plain search and the search with the LM are
timed with CUDA events after a warm-up, alternating round by round; the card's name, power limit and maximum SM clock are
printed next to the numbers.  The loader's wall time on each file is a host number.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctc_crf  # noqa: E402
from cat_b200.ngram import NGramLM, make_random_arpa  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:   # the numbers stand without it, but say so
        out = f"nvidia-smi unavailable ({e})"
    return torch.cuda.get_device_name(0), out


def labels_for(V):
    return ["<s>", "<unk>"] + [str(i) for i in range(2, V)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=64)
    ap.add_argument("--T", type=int, default=1500)
    ap.add_argument("--B", default="1,16,64,128")
    ap.add_argument("--cutoff", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="calls per timed window")
    ap.add_argument("--alpha", type=float, default=0.25)
    ap.add_argument("--beta", type=float, default=-0.5)
    a = ap.parse_args()
    Bs = [int(b) for b in a.B.split(",")]
    tmp = tempfile.mkdtemp(prefix="beam_lm_bench_")
    setups = [(218, 3, [40000, 450000]), (5000, 4, [200000, 250000, 250000])]
    res = {"N": a.N, "T": a.T, "cutoff_top_n": a.cutoff, "alpha": a.alpha, "beta": a.beta, "lms": []}
    for V, order, counts in setups:
        path = make_random_arpa(os.path.join(tmp, f"lm_{V}_{order}.arpa"), V, order, counts, seed=1)
        t0 = time.perf_counter()
        lm = NGramLM(path, labels_for(V))
        load_s = time.perf_counter() - t0
        g = torch.Generator(device="cuda").manual_seed(1)
        y = torch.log_softmax(3.0 * torch.randn((a.N, a.T, V), device="cuda", generator=g), -1).contiguous()
        lx = torch.full((a.N,), a.T, dtype=torch.int32)
        cases = []
        for b in Bs:
            cases.append((f"plain B={b}", lambda b=b: ctc_crf.ctc_beam_search(y, lx, b, a.cutoff)))
            cases.append((f"lm B={b}", lambda b=b: ctc_crf.ctc_beam_search(y, lx, b, a.cutoff, lm=lm, alpha=a.alpha,
                                                                              beta=a.beta)))
        for _, fn in cases:      # warm-up (the first LM call uploads the tables)
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
        ms = {k: float(np.median(v)) for k, v in times.items()}
        res["lms"].append({"V": V, "order": order, "ngrams": sum(lm.counts), "states": lm.num_states, "arcs": lm.num_arcs,
                           "load_s": load_s,
                           "ms": {k: {"median": ms[k], "min": float(np.min(v)), "max": float(np.max(v))}
                                  for k, v in times.items()},
                           "lm_over_plain": {b: ms[f"lm B={b}"] / ms[f"plain B={b}"] for b in Bs}})
        del lm, y
    name, smi = card()
    res["card"] = name
    res["nvidia_smi(name,power.limit,clocks.max.sm)"] = smi
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
