"""K label sequences per utterance: K separate CTC_CRF_LOSS / WARP_CTC_LOSS calls against one call with `utt` (the den passes
once per utterance, every numerator in one launch).  One GPU, CUDA events, arms alternated so that neither owns the warmer
clocks or allocator.

Shapes: N = 16 utterances of T = 500 frames, K = 4 and 8 sequences each (20 to 60 labels), the 1.02 M-arc synthetic den graph
(H = 20 000, V = 218); loss + gradient (the gradient of the mean, as a trainer takes it) and under torch.no_grad.
Prints the card's name, power limit and max SM clock with the numbers, as one JSON line.

Usage: python tools/multi_seq_bench.py [--reps 5] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card(dev):
    info = {"gpu": torch.cuda.get_device_name(dev)}
    try:   # read-only query
        q = subprocess.run(["nvidia-smi", f"--id={dev.index}", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        pl, clk = [x.strip() for x in q.strip().split(",")[:2]]
        info.update(power_limit_W=float(pl), max_sm_clock_MHz=int(float(clk)))
    except Exception as e:       # noqa: BLE001 -- the numbers are still worth printing without it
        info["card_query_error"] = str(e)
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import ctc_crf
    from cat_b200 import fst
    dev = torch.device("cuda", 0)
    N, T, V, lamb = 16, 500, 218, 0.01
    tmp = tempfile.mkdtemp(prefix="multi_seq_")
    path = os.path.join(tmp, "den_20000.fst")
    fst.write_fst(path, fst.make_synthetic_den(20000, 24, V, seed=7))
    ctx = ctc_crf.CRFContext(path, gpus=0)
    g = torch.Generator(device=dev).manual_seed(1)
    y = torch.log_softmax(3.0 * torch.randn(N, T, V, device=dev, generator=g), -1).contiguous()
    lx = torch.full((N,), T, dtype=torch.int32)
    rng = torch.Generator().manual_seed(2)

    def time_ms(fn):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    out = dict(card(dev), N=N, T=T, V=V, den_arcs=ctc_crf._C.den_info()["file_arcs"], reps=args.reps, rounds=args.rounds)
    for K in (4, 8):
        sets = []
        for _ in range(K):
            ly = torch.randint(20, 61, (N,), generator=rng, dtype=torch.int32)
            sets.append((torch.randint(1, V, (int(ly.sum()),), generator=rng, dtype=torch.int32), ly))
        # the same K*N sequences as one call: sequence k*N + n is set k's sequence of utterance n
        utt = torch.arange(N, dtype=torch.int32).repeat(K)
        labels = torch.cat([s[0] for s in sets])
        ly_all = torch.cat([s[1] for s in sets])
        res = {}
        for name, crit in (("ctc_crf", ctc_crf.CTC_CRF_LOSS(lamb=lamb)), ("warp_ctc", ctc_crf.WARP_CTC_LOSS())):
            def sep_grad():
                yg = y.detach().requires_grad_(True)
                sum(crit(yg, lab, lx, ly) for lab, ly in sets).div(K).backward()

            def one_grad():
                yg = y.detach().requires_grad_(True)
                crit(yg, labels, lx, ly_all, utt=utt).backward()

            def sep_eval():
                with torch.no_grad():
                    for lab, ly in sets:
                        crit(y, lab, lx, ly)

            def one_eval():
                with torch.no_grad():
                    crit(y, labels, lx, ly_all, utt=utt)

            r = {"K_calls_grad_ms": [], "one_call_grad_ms": [], "K_calls_no_grad_ms": [], "one_call_no_grad_ms": []}
            for i in range(args.rounds):
                arms = [("K_calls_grad_ms", sep_grad), ("one_call_grad_ms", one_grad),
                        ("K_calls_no_grad_ms", sep_eval), ("one_call_no_grad_ms", one_eval)]
                if i % 2:
                    arms = arms[1::-1] + arms[:1:-1]
                for key, fn in arms:
                    r[key].append(time_ms(fn))
            for mode in ("grad", "no_grad"):
                r[f"speedup_{mode}"] = min(r[f"K_calls_{mode}_ms"]) / min(r[f"one_call_{mode}_ms"])
            res[name] = r
        out[f"K{K}"] = res
    del ctx
    print(json.dumps(out))


if __name__ == "__main__":
    main()
