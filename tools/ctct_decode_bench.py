"""CTC-T beam search (``cat_b200.ctct_decode.ctct_beam_search``) on the workload of tools/rnnt_decode_bench.py: N = 64
utterances of T = 120 encoder frames, V = 4232, a one-layer LSTM predictor with hdim 512 and no head, a JointNet ("add")
with hdim 512, beam 1, 4 and 16, in fp32 and under fp16 autocast.  Random weights: the search does the same work whatever
the hypotheses are.  Reports ms per batch and utterances/s (CUDA events around whole calls, after a warm-up), the split of
GPU time between the step kernel, the predictor and the joiner from a separate torch.profiler run, and the per-hypothesis
torch restatement of CAT's CTCTDecoder (tests/ctct_decode_oracle.py) on the first `--ref-n` utterances for comparison.
Prints one JSON line per configuration; the card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from cat_b200.ctct_decode import ctct_beam_search  # noqa: E402
from ctct_decode_oracle import cat_decode  # noqa: E402
from rnnt_decode_bench import card, split, timed  # noqa: E402
from rnnt_decode_oracle import JointNet, LSTMPredictor  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--t", type=int, default=120)
    ap.add_argument("--v", type=int, default=4232)
    ap.add_argument("--h", type=int, default=512)
    ap.add_argument("--beams", default="1,4,16")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-n", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ctct_decode_bench measures on a GPU"
    torch.manual_seed(0)
    dev = torch.device("cuda")
    pred = LSTMPredictor(args.v, args.h).to(dev).eval()
    joiner = JointNet(args.h, args.h, args.v, args.h).to(dev).eval()
    enc = torch.randn(args.n, args.t, args.h, device=dev)
    lens = torch.full((args.n,), args.t, dtype=torch.int32)
    info = card()
    for amp in (False, True):
        for B in (int(b) for b in args.beams.split(",")):
            with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                def run():
                    return ctct_beam_search(enc, lens, pred, joiner, beam_size=B)
                ms = timed(run, args.reps)
                sp = split(run, pred, joiner, "ctct_beam_step_kernel")
                t0 = time.perf_counter()
                cat_decode(enc[:args.ref_n], lens[:args.ref_n], pred, joiner, B)
                torch.cuda.synchronize()
                ref_s = (time.perf_counter() - t0) / args.ref_n
            print(json.dumps({"card": info, "dtype": "fp16-autocast" if amp else "fp32", "N": args.n, "T": args.t,
                              "V": args.v, "beam": B, "ms_per_batch": round(ms, 2),
                              "utt_per_s": round(args.n / ms * 1e3, 1), "profile_ms": sp,
                              "cat_restatement_s_per_utt": round(ref_s, 3),
                              "cat_restatement_utt_per_s": round(1 / ref_s, 2)}), flush=True)


if __name__ == "__main__":
    main()
