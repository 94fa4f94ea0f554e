"""Timings behind the slice planner's CKPT_WIDTH and the cost of the checkpointed denominator (DESIGN.md "Checkpointed
α").  One GPU, CUDA events, arms alternated so that neither owns the warmer clocks or allocator:

  * config 4's den graph (H=100 000, 5.09 M arcs), T=2000: one checkpointed slice of W utterances against two
    full-spill slices of W/2, for W = 64, 32, 16; then N=64 through CTC_CRF_LOSS with the slices and checkpoint
    interval the planner chooses, and the peak memory allocated;
  * the headline shape (H=20 000, N=64, T=1500): the fused loss checkpointed (K = ceil(sqrt(T))) against the full spill.

Prints one JSON line.  Usage: python tools/ckpt_width_bench.py [--reps 3] [--rounds 2]
"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import ctc_crf
    from cat_b200 import _C, _lib, fst
    from bench import synth_labels
    dev = torch.device("cuda", 0)
    V, lamb = 218, 0.01
    tmp = tempfile.mkdtemp(prefix="ckpt_width_")

    def run(y, lab, lx, ly, k):
        _C._ckpt_k_override = k
        try:
            return _C.ctc_crf_loss_fwd(y, lab, lx, ly, lamb, True)[0]
        finally:
            _C._ckpt_k_override = None

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

    def batch(N, T, seed):
        lab, lens, ly = synth_labels(N, T, V, seed)
        g = torch.Generator(device=dev).manual_seed(seed)
        y = torch.log_softmax(3.0 * torch.randn(N, T, V, device=dev, generator=g), -1).contiguous()
        return y, torch.tensor(lab), torch.tensor(lens), torch.tensor(ly)

    def graph(H):
        path = os.path.join(tmp, f"den_{H}.fst")
        fst.write_fst(path, fst.make_synthetic_den(H, 24, V, seed=7))
        return path

    out = {"gpu": torch.cuda.get_device_name(dev), "reps": args.reps, "rounds": args.rounds}
    # config 4's graph: one checkpointed slice of W against two full-spill halves
    ctx = ctc_crf.CRFContext(graph(100000), gpus=0)
    T = 2000
    k = _C.ckpt_interval(T)
    widths = {}
    for W in (64, 32, 16):
        y, lab, lx, ly = batch(W, T, 100 + W)
        h = W // 2
        halves = [(y[:h].contiguous(), lab[:int(ly[:h].sum())], lx[:h], ly[:h]),
                  (y[h:].contiguous(), lab[int(ly[:h].sum()):], lx[h:], ly[h:])]
        ck, two = [], []
        for _ in range(args.rounds):
            ck.append(time_ms(lambda: run(y, lab, lx, ly, k)))
            two.append(time_ms(lambda: [run(*p, None) for p in halves]))
        widths[W] = {"ckpt_one_slice_ms": ck, "full_two_halves_ms": two, "K": k}
        del y, halves
        torch.cuda.empty_cache()
    out["config4_T2000"] = widths
    # config 4's graph, N=64, T=2000 through CTC_CRF_LOSS with the planner's own choice (its full spill, 102.6 GB, does
    # not fit one call): frames/s, the slices and K it chose, peak memory torch allocated during the steps
    N4 = 64
    y, lab, lx, ly = batch(N4, T, 4343)
    crit = ctc_crf.CTC_CRF_LOSS(lamb=lamb, size_average=True)
    plan = _C._plan_slices(_lib.lib(), lx, ly, N4, V, dev)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    ms = time_ms(lambda: crit(y, lab, lx, ly))
    out["config4_N64_T2000_loss"] = {
        "ms_per_step": ms, "frames_per_s": int(lx.sum()) / (ms * 1e-3),
        "slices": [{"n0": s[0], "n1": s[1], "tmax": s[2], "ckpt_k": s[4]} for s in plan],
        "peak_allocated_GB": torch.cuda.max_memory_allocated(dev) / 1e9, "inputs_GB": base / 1e9,
        "full_spill_one_call_GB": int(_lib.lib().ccb_den_alpha_floats(N4, T)) * 4 / 1e9}
    del y
    torch.cuda.empty_cache()
    del ctx
    # headline shape: checkpointed against the full spill
    ctx = ctc_crf.CRFContext(graph(20000), gpus=0)
    T = 1500
    k = _C.ckpt_interval(T)
    y, lab, lx, ly = batch(64, T, 1234)
    ck, full = [], []
    for _ in range(args.rounds):
        full.append(time_ms(lambda: run(y, lab, lx, ly, None)))
        ck.append(time_ms(lambda: run(y, lab, lx, ly, k)))
    out["headline_N64_T1500"] = {"full_ms": full, "ckpt_ms": ck, "K": k}
    del ctx
    print(json.dumps(out))


if __name__ == "__main__":
    main()
