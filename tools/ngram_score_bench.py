"""N-gram sentence scoring (``NGramLM.score``, one ``ccb_ngram_score`` launch per call) on three shapes:
  aishell   N-best rescoring as cat.lm.rescore feeds it: 7,176 utterances x 16 hypotheses = 114,816 rows of 8-30 tokens
            plus the leading 0, V = 4232, a random 5-gram (``make_random_arpa``, --ngrams n-grams per order 2..5);
  ppl       a cat.lm.ppl corpus: 10,000 sentences of 10-200 tokens;
  long      R = 16 rows of U = 8192 tokens (the one-CTA-per-row layout).
Reports ms per call (CUDA events around --reps calls after a warm-up; the median of --rounds rounds), sentences/s and
words/s (words = sum of lengths + 1 per row, the terms the kernel sums).  Prints one JSON line per shape; the card's name
and power limit are read in the same run.  Writes only to a temporary directory.
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
from cat_b200.ngram import NGramLM, make_random_arpa  # noqa: E402
from rnnt_decode_bench import card, timed  # noqa: E402


def shape(name, V, g):
    if name == "aishell":
        R, lo, hi = 7176 * 16, 8, 30
    elif name == "ppl":
        R, lo, hi = 10000, 10, 200
    else:
        R, lo, hi = 16, 8191, 8191
    lens = torch.randint(lo, hi + 1, (R,), generator=g) + 1          # the leading 0 counts, as in CAT's in_lens
    U = int(lens.max())
    ids = torch.randint(1, V, (R, U), generator=g)
    ids[:, 0] = 0
    return ids, torch.zeros((R, 1), dtype=torch.int64), lens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--v", type=int, default=4232)
    ap.add_argument("--ngrams", type=int, default=200000)
    ap.add_argument("--shapes", default="aishell,ppl,long")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ngram_score_bench measures on a GPU"
    gpu = card()
    g = torch.Generator().manual_seed(0)
    with tempfile.TemporaryDirectory() as tmp:
        labels = ["<s>", "<unk>"] + [str(i) for i in range(2, args.v)]
        lm = NGramLM(make_random_arpa(os.path.join(tmp, "5gram.arpa"), args.v, 5, args.ngrams, seed=0), labels)
    for name in args.shapes.split(","):
        ids, tg, lens = shape(name, args.v, g)
        x = (ids.cuda(), tg.cuda(), lens.cuda())
        fn = lambda: lm.score(*x)
        ms = statistics.median(timed(fn, args.reps) for _ in range(args.rounds))
        R, words = int(ids.shape[0]), int(lens.sum()) + int(ids.shape[0])
        print(json.dumps(dict(shape=name, R=R, U=int(ids.shape[1]), words=words, order=lm.order, V=args.v,
                              ngrams_per_order=lm.counts, ms_per_call=round(ms, 4), sentences_per_s=round(R / ms * 1e3),
                              words_per_s=round(words / ms * 1e3), gpu=gpu)), flush=True)


if __name__ == "__main__":
    main()
