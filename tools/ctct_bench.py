"""CTC-T loss, loss + gradient, at CAT-sized shapes (DESIGN.md §7 "CTC-T loss").

Arms, each timed as one loss and its gradient, on the compact joint (sum T(U+1), V) of N(0,1) raw logits with uniform
lengths and labels drawn without adjacent repeats (so T >= U + repeats holds for every utterance):
  (a) a_ctct_logsoftmax: fp32 log_softmax + ctct_loss, compact;
  (b) b_ctct_logits_fp32 / b_ctct_logits_fp16: ctct_loss(from_logits=True) on fp32 and fp16 logits;
  (c) c_rnnt_logsoftmax / c_rnnt_logits_fp32: rnnt_loss on the same tensors as (a) and (b), the sibling cost;
  (d) d_ctct_simple / d_ctct_materialised: ctct_simple_loss(f, g) against log_softmax(f[:, :, None] + g[:, None]) +
      ctct_loss, from f (N, T, V) and g (N, U+1, V), fp32.
Per arm: ms per loss + gradient (CUDA events, median of alternated rounds) and peak memory above the inputs
(torch.cuda.max_memory_allocated); with --profile the per-kernel split of the from-logits CTC-T and RNN-T arms.  The
card's name and power limit are read in the same run.

usage: python tools/ctct_bench.py [--rounds 7] [--iters 5] [--profile]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from rnnt_simple_bench import card  # noqa: E402

SHAPES = {"aishell": (64, 150, 20, 4232), "libri": (32, 400, 120, 1024)}


def labels_without_repeats(N, U, V, gen):
    y = torch.randint(1, V, (N, U), dtype=torch.int32, device="cuda", generator=gen)
    for u in range(1, U):
        y[:, u] = torch.where(y[:, u] == y[:, u - 1], y[:, u] % (V - 1) + 1, y[:, u])
    return y


def timed(arms, rounds, iters):
    times, peaks, oom = {k: [] for k in arms}, {}, {}
    for k, fn in list(arms.items()):
        try:
            fn()
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            peaks[k] = torch.cuda.max_memory_allocated() - base
        except torch.cuda.OutOfMemoryError as e:
            oom[k] = str(e).splitlines()[0][:160]
            del arms[k]
            torch.cuda.empty_cache()
    for _ in range(rounds):
        for k, fn in arms.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            e.synchronize()
            times[k].append(s.elapsed_time(e) / iters)
    out = {}
    for k in list(times) + list(oom):
        if k in oom:
            out[k] = {"status": f"out of memory: {oom[k]}"}
        else:
            out[k] = {"ms": round(statistics.median(times[k]), 3), "ms_min": round(min(times[k]), 3),
                      "ms_max": round(max(times[k]), 3), "peak_GB": round(peaks[k] / 1e9, 4)}
    return out


def profile(fn, iters):
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as prof_
    with prof_(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ev = [(e.key, e.self_device_time_total) for e in p.key_averages() if e.self_device_time_total > 0]
    top = sorted(ev, key=lambda x: -x[1])[:8]
    return {k[:60]: round(t / iters, 1) for k, t in top}, round(sum(t for _, t in ev) / iters, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--shapes", default="aishell,libri")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "ctct_bench needs a GPU"
    from warp_ctct import ctct_loss, ctct_simple_loss
    from warp_rnnt import rnnt_loss
    print(json.dumps({"card": card()}))
    for name in a.shapes.split(","):
        N, T, U, V = SHAPES[name]
        gen = torch.Generator(device="cuda").manual_seed(0)
        x32 = torch.randn(N * T * (U + 1), V, device="cuda", generator=gen)
        x16 = x32.half()
        y = labels_without_repeats(N, U, V, gen)
        yc = y.reshape(-1)
        lx = torch.full((N,), T, dtype=torch.int32)
        ly = torch.full((N,), U, dtype=torch.int32)

        def joint(loss, x, from_logits):
            def fn():
                xg = x.detach().requires_grad_(True)
                inp = xg if from_logits else xg.log_softmax(-1)
                loss(inp, yc, lx, ly, compact=True, from_logits=from_logits).backward()
            return fn

        arms = {"a_ctct_logsoftmax": joint(ctct_loss, x32, False), "b_ctct_logits_fp32": joint(ctct_loss, x32, True),
                "b_ctct_logits_fp16": joint(ctct_loss, x16, True), "c_rnnt_logsoftmax": joint(rnnt_loss, x32, False),
                "c_rnnt_logits_fp32": joint(rnnt_loss, x32, True)}
        for k, r in timed(arms, a.rounds, a.iters).items():
            print(json.dumps({"shape": name, "N": N, "T": T, "U": U, "V": V, "arm": k, **r}), flush=True)
        if a.profile:
            for k in ("b_ctct_logits_fp32", "c_rnnt_logits_fp32"):
                top, tot = profile(arms[k], a.iters)
                print(json.dumps({"shape": name, "profile": k, "us_per_call": top, "total_us_per_call": tot}), flush=True)
        del arms, x32, x16
        torch.cuda.empty_cache()

        f0 = torch.randn(N, T, V, device="cuda", generator=gen)
        g0 = torch.randn(N, U + 1, V, device="cuda", generator=gen)

        def simple():
            f, g = f0.detach().requires_grad_(True), g0.detach().requires_grad_(True)
            ctct_simple_loss(f, g, y, lx, ly).backward()

        def materialised():
            f, g = f0.detach().requires_grad_(True), g0.detach().requires_grad_(True)
            ctct_loss((f[:, :, None] + g[:, None]).log_softmax(-1), y, lx, ly).backward()

        for k, r in timed({"d_ctct_simple": simple, "d_ctct_materialised": materialised}, a.rounds, a.iters).items():
            print(json.dumps({"shape": name, "N": N, "T": T, "U": U, "V": V, "arm": k, **r}), flush=True)
        del f0, g0
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
