"""RNN-T loss + gradient at CAT-sized shapes (DESIGN.md §7 "RNN-T loss").

Arms, each timed as one loss and its gradient with respect to the joiner output:
  (a) CAT's path: fp32 log_softmax, the log-prob loss (compact), backward through both;
  (b) from_logits=True on the fp32 and on the fp16 joiner output (compact);
  (c) torchaudio's CUDA rnnt_loss on the padded layout (fused log-softmax), when the installed torchaudio has it.
Per arm: ms per loss + gradient (CUDA events, median of alternated rounds), peak memory above the inputs
(torch.cuda.max_memory_allocated), bytes moved (from shapes: each pass over a (rows, V) tensor counted once) and the
bandwidth that implies.  The card's name and power limit are read in the same run.

usage: python tools/rnnt_bench.py [--rounds 7] [--iters 5]
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


def make_arms(N, T, U, V):
    from warp_rnnt import rnnt_loss
    g = torch.Generator(device="cuda").manual_seed(0)
    lx = torch.full((N,), T, dtype=torch.int32, device="cuda")
    ly = torch.full((N,), U, dtype=torch.int32, device="cuda")
    rows = N * T * (U + 1)
    z32 = torch.randn(rows, V, device="cuda", generator=g)
    z16 = z32.half()
    y = torch.randint(1, V, (N * U,), dtype=torch.int32, device="cuda", generator=g)
    esz = {torch.float32: 4, torch.float16: 2}
    RV = rows * V

    def arm_a():
        z = z32.detach().requires_grad_(True)
        rnnt_loss(z.log_softmax(-1), y, lx, ly, compact=True).backward()

    def arm_b(zz):
        def f():
            z = zz.detach().requires_grad_(True)
            rnnt_loss(z, y, lx, ly, compact=True, from_logits=True).backward()
        return f

    arms = {
        # log_softmax: read + write; loss backward: write the gradient; log_softmax backward: read two, write one
        "a_cat_logsoftmax_fp32": (arm_a, 6 * RV * 4),
        # row pass reads the logits; gradient pass reads them again and writes the gradient
        "b_from_logits_fp32": (arm_b(z32), 3 * RV * esz[torch.float32]),
        "b_from_logits_fp16": (arm_b(z16), 3 * RV * esz[torch.float16]),
    }
    try:
        import torchaudio.functional as F
        zp = z32.view(N, T, U + 1, V)
        yp = y.view(N, U)
        F.rnnt_loss(zp[:1, :2, :2].contiguous(), yp[:1, :1].contiguous(), lx[:1].clamp(max=2), ly[:1].clamp(max=1))

        def arm_c():
            z = zp.detach().requires_grad_(True)
            F.rnnt_loss(z, yp, lx, ly, blank=0, reduction="mean").backward()
        # at least: read the logits once, write the gradient once, scale it by grad_output (read + write)
        arms["c_torchaudio_padded_fp32"] = (arm_c, 4 * RV * 4)
        ta = "available"
    except Exception as e:      # noqa: BLE001
        ta = f"not available ({type(e).__name__}: {str(e)[:120]})"
    return arms, ta, rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--shapes", default="aishell,libri")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "rnnt_bench needs a GPU"
    print(json.dumps({"card": card()}))
    for name in a.shapes.split(","):
        N, T, U, V = SHAPES[name]
        arms, ta, rows = make_arms(N, T, U, V)
        times = {k: [] for k in arms}
        peaks = {}
        for k, (f, _) in arms.items():          # warm-up, and the peak memory of one call above what is allocated now
            f()
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            f()
            torch.cuda.synchronize()
            peaks[k] = torch.cuda.max_memory_allocated() - base
        for _ in range(a.rounds):
            for k, (f, _) in arms.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(a.iters):
                    f()
                e.record()
                e.synchronize()
                times[k].append(s.elapsed_time(e) / a.iters)
        for k, (f, nbytes) in arms.items():
            ms = statistics.median(times[k])
            print(json.dumps({"shape": name, "N": N, "T": T, "U": U, "V": V, "rows": rows, "arm": k,
                              "ms": round(ms, 3), "ms_min": round(min(times[k]), 3), "ms_max": round(max(times[k]), 3),
                              "peak_GB": round(peaks[k] / 1e9, 3), "bytes_GB": round(nbytes / 1e9, 3),
                              "GB_per_s": round(nbytes / 1e9 / (ms / 1e3), 1)}))
        if "c_torchaudio_padded_fp32" not in arms:
            print(json.dumps({"shape": name, "arm": "c_torchaudio_padded_fp32", "status": ta}))
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
