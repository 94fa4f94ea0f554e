"""Time ``ctc_crf.fst_decode`` (TLG word decoding) on a several-million-arc ``make_tlg`` graph.

    python tools/wfst_decode_bench.py [--N 1,64] [--T 1500] [--beam 8,17] [--max-active 1000,7000] [--rounds 3] [--reps 2]

The graph is the one tests/test_gpu_wfst_decode.py checks at size: V = 72 tokens, 3000 words of 2-6 tokens, a 3-gram of
60 000 bigrams and 60 000 trigrams (about 1.46 M states and 3.7 M arcs), so that the numbers describe a lexicon-sized search
rather than a toy one.  The logits are peaky along the CTC alignment of a random word sequence, as an acoustic model's are.
Every (N, beam, max_active) is timed with CUDA events after a warm-up, the cases alternating round by round; ms per call
and frames per second (N T / time) are reported with the card's name, power limit and maximum SM clock.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "tests"))
sys.path.insert(0, os.path.join(HERE, "tools"))
import ctc_crf  # noqa: E402
from beam_lm_bench import card  # noqa: E402
from test_gpu_wfst_decode import aligned_logits, headline_graph  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", default="1,64")
    ap.add_argument("--T", type=int, default=1500)
    ap.add_argument("--beam", default="8,17")
    ap.add_argument("--max-active", default="1000,7000")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2, help="calls per timed window")
    a = ap.parse_args()
    Ns = [int(x) for x in a.N.split(",")]
    beams = [float(x) for x in a.beam.split(",")]
    Ks = [int(x) for x in a.max_active.split(",")]
    tmp = tempfile.mkdtemp(prefix="wfst_bench_")
    t0 = time.perf_counter()
    path, lex = headline_graph(__import__("pathlib").Path(tmp))
    build_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    dg = ctc_crf.DecodingGraph(path)
    load_s = time.perf_counter() - t0
    y = torch.tensor(aligned_logits(lex, max(Ns), a.T, 72, seed=1), device="cuda")
    lx = torch.full((max(Ns),), a.T, dtype=torch.int32)
    cases = [((n, b, k), lambda n=n, b=b, k=k: ctc_crf.fst_decode(y[:n], lx[:n], dg, beam=b, max_active=k))
             for n in Ns for b in beams for k in Ks]
    for _, fn in cases:          # warm-up (the first call uploads the graph)
        fn()
    torch.cuda.synchronize()
    times = {c: [] for c, _ in cases}
    for _ in range(a.rounds):
        for c, fn in cases:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                fn()
            e1.record()
            e1.synchronize()
            times[c].append(e0.elapsed_time(e1) / a.reps)
    name, smi = card()
    res = {"T": a.T, "graph": {"states": dg.num_states, "arcs": dg.num_arcs, "L": dg.L, "E": dg.E, "max_out": dg.max_out,
                               "build_s": build_s, "load_s": load_s},
           "card": name, "nvidia_smi(name,power.limit,clocks.max.sm)": smi, "cases": []}
    for (n, b, k), v in times.items():
        ms = float(np.median(v))
        res["cases"].append({"N": n, "beam": b, "max_active": k, "ms": ms, "min_ms": float(np.min(v)),
                             "max_ms": float(np.max(v)), "frames_per_s": n * a.T / (ms / 1e3)})
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
