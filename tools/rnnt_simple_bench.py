"""RNN-T loss of the LogAdd joiner, loss + gradients on f and g, at CAT-sized shapes (DESIGN.md §7 "RNN-T loss, LogAdd
joiner").

Arms, each timed as one loss and its gradients with respect to the encoder output f and the predictor output g:
  (a) the materialised LogAdd path: (f[:, :, None] + g[:, None]) -> rnnt_loss(from_logits=True), padded layout;
  (b) rnnt_loss_simple(f, g, ...).
Inputs: "random" (N(0,1) entries: no cell underflows) and "peaked" (f and g peak by 60 on disjoint token sets, so that
S(t,u) < 2^-64 in every cell: the underflow fix-up's worst case).  Per arm: ms per loss + gradients (CUDA events, median
of alternated rounds), peak memory above the inputs (torch.cuda.max_memory_allocated), the GEMM FLOP and bytes from the
shapes, the share of flagged cells, and with --profile the share of each kernel in arm (b).  The card's name and power
limit are read in the same run.  Where arm (a) runs out of memory it says so.

usage: python tools/rnnt_simple_bench.py [--rounds 7] [--iters 5] [--profile]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"aishell": (64, 150, 20, 4232), "libri": (32, 400, 120, 1024)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return q


def make_inputs(N, T, U, V, dtype, kind):
    gen = torch.Generator(device="cuda").manual_seed(0)
    f = torch.randn(N, T, V, device="cuda", generator=gen)
    g = torch.randn(N, U + 1, V, device="cuda", generator=gen)
    if kind == "peaked":
        a = torch.randint(1, V // 2, (N, T, 1), device="cuda", generator=gen)
        b = torch.randint(V // 2, V, (N, U + 1, 1), device="cuda", generator=gen)
        f.scatter_(2, a, 60.0)
        g.scatter_(2, b, 60.0)
    y = torch.randint(1, V, (N, U), dtype=torch.int32, device="cuda", generator=gen)
    lx = torch.full((N,), T, dtype=torch.int32, device="cuda")
    ly = torch.full((N,), U, dtype=torch.int32, device="cuda")
    return f.to(dtype), g.to(dtype), y, lx, ly


def flagged_share(f, g):
    """The share of cells with S(t,u) < 2^-64, from an fp64 restatement of the normaliser (every cell is live here)."""
    f, g = f.double(), g.double()
    S = torch.bmm(torch.exp(f - f.amax(-1, keepdim=True)), torch.exp(g - g.amax(-1, keepdim=True)).transpose(1, 2))
    return float((S < 2.0 ** -64).double().mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--shapes", default="aishell,libri")
    ap.add_argument("--dtypes", default="fp32,fp16")
    ap.add_argument("--kinds", default="random,peaked")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "rnnt_simple_bench needs a GPU"
    from warp_rnnt import rnnt_loss, rnnt_loss_simple
    print(json.dumps({"card": card()}))
    dts = {"fp32": torch.float32, "fp16": torch.float16}
    for name in a.shapes.split(","):
        N, T, U, V = SHAPES[name]
        cells = N * T * (U + 1)
        flop = 2 * cells * V
        for dn in a.dtypes.split(","):
            dtype = dts[dn]
            for kind in a.kinds.split(","):
                f0, g0, y, lx, ly = make_inputs(N, T, U, V, dtype, kind)
                esz = f0.element_size()
                share = flagged_share(f0, g0)

                def arm_a():
                    f, g = f0.detach().requires_grad_(True), g0.detach().requires_grad_(True)
                    rnnt_loss(f[:, :, None] + g[:, None], y, lx, ly, from_logits=True).backward()

                def arm_b():
                    f, g = f0.detach().requires_grad_(True), g0.detach().requires_grad_(True)
                    rnnt_loss_simple(f, g, y, lx, ly).backward()

                arms = {"a_materialised": arm_a, "b_simple": arm_b}
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
                for _ in range(a.rounds):
                    for k, fn in arms.items():
                        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        s.record()
                        for _ in range(a.iters):
                            fn()
                        e.record()
                        e.synchronize()
                        times[k].append(s.elapsed_time(e) / a.iters)
                for k in times:
                    rec = {"shape": name, "N": N, "T": T, "U": U, "V": V, "dtype": dn, "input": kind, "arm": k,
                           "flagged_share": round(share, 4)}
                    if k in oom:
                        rec["status"] = f"out of memory: {oom[k]}"
                    else:
                        ms = statistics.median(times[k])
                        rec.update({"ms": round(ms, 3), "ms_min": round(min(times[k]), 3), "ms_max": round(max(times[k]), 3),
                                    "peak_GB": round(peaks[k] / 1e9, 4)})
                    if k == "b_simple":
                        # forward GEMM + two gradient GEMMs; f and g read by each (rows of the other operand once per
                        # tile are not counted), gradients written once
                        rec.update({"gemm_GFLOP": round(3 * flop / 1e9, 2),
                                    "gemm_bytes_MB": round((3 * (f0.numel() + g0.numel()) + f0.numel() + g0.numel())
                                                           * esz / 1e6, 1)})
                    print(json.dumps(rec), flush=True)
                if a.profile and "b_simple" in arms:
                    from torch.profiler import ProfilerActivity, profile
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for _ in range(a.iters):
                            arm_b()
                        torch.cuda.synchronize()
                    ev = [(e.key, e.self_device_time_total) for e in prof.key_averages() if e.self_device_time_total > 0]
                    tot = sum(t for _, t in ev)
                    top = sorted(ev, key=lambda x: -x[1])[:8]
                    print(json.dumps({"shape": name, "dtype": dn, "input": kind, "profile_b_simple_us_per_call":
                                      {k[:60]: round(t / a.iters, 1) for k, t in top},
                                      "total_us_per_call": round(tot / a.iters, 1)}), flush=True)
                del arms, f0, g0
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
