"""RNN-T beam search with LM fusion and ILM estimation (``cat_b200.rnnt_decode.rnnt_beam_search(..., lm, alpha, beta,
ilm_weight)``) on the aishell-like shape of tools/rnnt_decode_bench.py: N = 64 utterances of T = 120 encoder frames,
V = 4232, a one-layer LSTM predictor and a JointNet ("add") of hdim 512.  Arms: no fusion; a random 5-gram token LM
(``make_random_arpa``, ``--ngrams`` n-grams per order 2..5) through ``NGramLM``; a one-layer LSTM LM of hdim 512; ILM
estimation; the 5-gram with ILM; and LODR mixes (``MultiLM``): the 5-gram with a pruned bigram (``make_random_arpa``
at order 2 with --lodr-bigrams bigrams, the --topk default of CAT's prep_wlm_lodr.sh), the same with ILM, and the LSTM LM
with the bigram.  Each at beam 4 and 16, in fp32 and under fp16 autocast (--arms picks a subset).  Reports ms per batch
(CUDA events around whole calls, after a warm-up; the median of --rounds rounds that alternate the arms) and the split of
GPU time between the step kernel (plain or fused), the n-gram or mix rows kernel and the networks (every other kernel:
predictor, joiner, LM) from torch.profiler runs.  Prints one JSON line per configuration; the card's name and power limit
are read in the same run.

With --mix-rows it also times the LODR rows alone, T frames of the beam's (N*B, V) rows with random parents and tokens:
one ``ccb_lm_mix_slot_rows`` launch per frame, against the same mix composed without it (two ``ccb_ngram_slot_rows``
launches and a torch weighted add in fp64, rounded to fp32), and checks that both give the same bits.
"""
import ctypes as C
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
from cat_b200 import _lib  # noqa: E402
from cat_b200.ngram import NGramLM, make_random_arpa  # noqa: E402
from cat_b200.rnnt_decode import MultiLM, rnnt_beam_search  # noqa: E402
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
    ap.add_argument("--lodr-bigrams", type=int, default=20000)
    ap.add_argument("--arms", default="none,5gram,lstm_lm,ilm,5gram+ilm,lodr,lodr+ilm,lstm_lm+lodr")
    ap.add_argument("--mix-rows", action="store_true")
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
        bi = make_random_arpa(os.path.join(tmp, "lodr_2gram.arpa"), args.v, 2, args.lodr_bigrams, seed=1)
        bigram = NGramLM(bi, ["<blk>", "<unk>"] + [str(i) for i in range(2, args.v)])
    # LODR as CAT's aishell rnnt-v1 recipe runs it: the LM mix [elm 0.28125, bigram -0.3125] with alpha 1
    lodr = MultiLM([0.28125, -0.3125], [ngram, bigram])
    arms = {"none": {}, "5gram": dict(lm=ngram, alpha=0.28125, beta=0.5), "lstm_lm": dict(lm=lstm_lm, alpha=0.28125, beta=0.5),
            "ilm": dict(ilm_weight=-0.3125), "5gram+ilm": dict(lm=ngram, alpha=0.28125, beta=0.5, ilm_weight=-0.3125),
            "lodr": dict(lm=lodr, alpha=1.0, beta=0.5), "lodr+ilm": dict(lm=lodr, alpha=1.0, beta=0.5, ilm_weight=-0.3125),
            "lstm_lm+lodr": dict(lm=MultiLM([0.28125, -0.3125], [lstm_lm, bigram]), alpha=1.0, beta=0.5)}
    arms = {a: arms[a] for a in args.arms.split(",")}
    info = card()
    if args.mix_rows:
        for B in (int(b) for b in args.beams.split(",")):
            mix_rows_bench(info, args, ngram, bigram, B)
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
                    rk = "ngram_slot_rows_kernel" if "5gram" in arm else "lm_mix_slot_rows_kernel" if "lodr" in arm else None
                    rows_ms = split(run, pred, joiner, kernel=rk)["step_kernel"] if rk else 0.0
                gpu = {"step_kernel": sp["step_kernel"], "rows_kernel": rows_ms,
                       "networks": round(sp["all_kernels"] - sp["step_kernel"] - rows_ms, 2), "all_kernels": sp["all_kernels"]}
                print(json.dumps({"card": info, "arm": arm, "dtype": "fp16-autocast" if amp else "fp32", "N": args.n,
                                  "T": args.t, "V": args.v, "beam": B,
                                  "ngram_counts": ngram.counts if "5gram" in arm or arm.startswith("lodr") else None,
                                  "bigram_counts": bigram.counts if "lodr" in arm else None,
                                  "ms_per_batch": round(ms, 2), "ms_rounds": [round(x, 1) for x in times[arm]],
                                  "utt_per_s": round(args.n / ms * 1e3, 1), "gpu_ms": gpu}), flush=True)


def mix_rows_bench(info, args, ngram, bigram, B):
    """ms per batch of T frames of LODR rows: the mix kernel against two n-gram rows launches plus a torch weighted add"""
    L = _lib.lib()
    N, V, R, T = args.n, args.v, args.n * B, args.t
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(B)
    par = [torch.randint(0, B, (N, B), device=dev, generator=g, dtype=torch.int32) for _ in range(T)]
    tok = [torch.where(torch.rand((N, B), device=dev, generator=g) < 0.3, -1,
                       torch.randint(1, V, (N, B), device=dev, generator=g)).int() for _ in range(T)]
    lms, w = [ngram, bigram], [0.28125, -0.3125]
    st = [[torch.zeros((N, B), dtype=torch.int32, device=dev) for _ in range(2)] for _ in lms]
    one = [torch.empty((R, V), device=dev) for _ in lms]
    fused, composed = torch.empty((R, V), device=dev), torch.empty((R, V), device=dev)
    vp = C.c_void_p

    def frame(t, kernel):
        pp, tp = (None, None) if t == 0 else (par[t].data_ptr(), tok[t].data_ptr())
        if kernel:
            rc = L.ccb_lm_mix_slot_rows(2, (vp * 2)(*[lm.handle for lm in lms]), (C.c_double * 2)(*w),
                                        (vp * 2)(*[s[0].data_ptr() for s in st]), (vp * 2)(*[s[1].data_ptr() for s in st]),
                                        0, None, None, None, (C.c_int * 2)(0, 1), N, B, V, pp, tp, fused.data_ptr(), None)
            assert rc == 0, _lib.last_error()
        else:
            for lm, s, r in zip(lms, st, one):
                rc = L.ccb_ngram_slot_rows(lm.handle, N, B, V, pp, tp, s[0].data_ptr() if pp else None, s[1].data_ptr(),
                                           r.data_ptr(), None)
                assert rc == 0, _lib.last_error()
            dead = (one[0] == float("-inf")) | (one[1] == float("-inf"))
            composed.copy_(torch.where(dead, float("-inf"), one[0].double() * w[0] + one[1].double() * w[1]))
        for s in st:
            s.reverse()

    def batch(kernel):
        def run():
            for t in range(T):
                frame(t, kernel)
        return run

    same = True
    for t in range(T):   # both compositions from the same states, frame by frame
        frame(t, True)
        for s in st:
            s.reverse()
        frame(t, False)
        same &= bool(torch.equal(fused.view(torch.int32), composed.view(torch.int32)))
    times = {"mix_kernel": [], "composed": []}
    for _ in range(args.rounds):
        times["mix_kernel"].append(timed(batch(True), args.reps))
        times["composed"].append(timed(batch(False), args.reps))
    med = {k: round(sorted(v)[len(v) // 2], 3) for k, v in times.items()}
    print(json.dumps({"card": info, "bench": "lodr_mix_rows", "N": N, "T": T, "V": V, "beam": B,
                      "ngram_counts": ngram.counts, "bigram_counts": bigram.counts, "ms_per_batch": med,
                      "ms_rounds": {k: [round(x, 2) for x in v] for k, v in times.items()}, "same_bits": same}),
          flush=True)


if __name__ == "__main__":
    main()
