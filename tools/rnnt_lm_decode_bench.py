"""RNN-T beam search with LM fusion and ILM estimation (``cat_b200.rnnt_decode.rnnt_beam_search(..., lm, alpha, beta,
ilm_weight)``) on the aishell-like shape of tools/rnnt_decode_bench.py: N = 64 utterances of T = 120 encoder frames,
V = 4232, a one-layer LSTM predictor and a JointNet ("add") of hdim 512.  Arms: no fusion; a random 5-gram token LM
(``make_random_arpa``, ``--ngrams`` n-grams per order 2..5) through ``NGramLM``; a one-layer LSTM LM of hdim 512; ILM
estimation; the 5-gram with ILM.  Each at beam 4 and 16, in fp32 and under fp16 autocast.  Reports ms per batch (CUDA
events around whole calls, after a warm-up; the median of --rounds rounds that alternate the arms) and the split of GPU
time between the step kernel (plain or fused), the n-gram rows kernel and the networks (every other kernel: predictor,
joiner, LM) from torch.profiler runs.  Prints one JSON line per configuration; the card's name and power limit are read in
the same run.
"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from cat_b200.ngram import NGramLM, make_random_arpa  # noqa: E402
from cat_b200.rnnt_decode import rnnt_beam_search  # noqa: E402
from rnnt_decode_bench import card, split, timed  # noqa: E402
from rnnt_fusion_oracle import JointNet, LSTMLM  # noqa: E402
from rnnt_decode_oracle import LSTMPredictor  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--t", type=int, default=120)
    ap.add_argument("--v", type=int, default=4232)
    ap.add_argument("--h", type=int, default=512)
    ap.add_argument("--beams", default="4,16")
    ap.add_argument("--ngrams", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "rnnt_lm_decode_bench measures on a GPU"
    torch.manual_seed(0)
    dev = torch.device("cuda")
    pred = LSTMPredictor(args.v, args.h).to(dev).eval()
    joiner = JointNet(args.h, args.h, args.v, args.h).to(dev).eval()
    lstm_lm = LSTMLM(args.v, args.h).to(dev).eval()
    enc = torch.randn(args.n, args.t, args.h, device=dev)
    lens = torch.full((args.n,), args.t, dtype=torch.int32)
    with tempfile.TemporaryDirectory() as tmp:
        arpa = make_random_arpa(os.path.join(tmp, "5gram.arpa"), args.v, 5, args.ngrams, seed=0)
        ngram = NGramLM(arpa, ["<blk>", "<unk>"] + [str(i) for i in range(2, args.v)])
    arms = {"none": {}, "5gram": dict(lm=ngram, alpha=0.28125, beta=0.5), "lstm_lm": dict(lm=lstm_lm, alpha=0.28125, beta=0.5),
            "ilm": dict(ilm_weight=-0.3125), "5gram+ilm": dict(lm=ngram, alpha=0.28125, beta=0.5, ilm_weight=-0.3125)}
    info = card()
    for amp in (False, True):
        for B in (int(b) for b in args.beams.split(",")):
            def runner(kw):
                return lambda: rnnt_beam_search(enc, lens, pred, joiner, beam_size=B, **kw)
            # ms per batch: the arms alternated over --rounds rounds (the host shares the machine), the median kept
            times = {arm: [] for arm in arms}
            with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                for _ in range(args.rounds):
                    for arm, kw in arms.items():
                        times[arm].append(timed(runner(kw), args.reps))
            for arm, kw in arms.items():
                ms = sorted(times[arm])[len(times[arm]) // 2]
                run = runner(kw)
                with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                    sp = split(run, pred, joiner)
                    rows_ms = split(run, pred, joiner, kernel="ngram_slot_rows_kernel")["step_kernel"] if "5gram" in arm \
                        else 0.0
                gpu = {"step_kernel": sp["step_kernel"], "ngram_rows_kernel": rows_ms,
                       "networks": round(sp["all_kernels"] - sp["step_kernel"] - rows_ms, 2), "all_kernels": sp["all_kernels"]}
                print(json.dumps({"card": info, "arm": arm, "dtype": "fp16-autocast" if amp else "fp32", "N": args.n,
                                  "T": args.t, "V": args.v, "beam": B, "ngram_counts": ngram.counts if "5gram" in arm else None,
                                  "ms_per_batch": round(ms, 2), "ms_rounds": [round(x, 1) for x in times[arm]],
                                  "utt_per_s": round(args.n / ms * 1e3, 1), "gpu_ms": gpu}), flush=True)


if __name__ == "__main__":
    main()
