"""Forward-only CTC-CRF loss (CTC_CRF_LOSS under torch.no_grad) against the loss plus gradient (grad mode on), on one GPU:

  * the headline shape: 1.02 M-arc den graph (H=20 000), N=64, T=1500, V=218;
  * config 4's den graph (H=100 000, 5.09 M arcs), N=64, T=2000, V=218.

Each call is timed with CUDA events, the two arms alternated call by call (--reps of each, after one warm-up of each), and
the peak memory torch allocated during each arm is reported as the rise over what the inputs hold.  The card's name,
power limit and max SM clock are read in the same run (nvidia-smi, query only).

Prints one JSON line.  Usage: python tools/fwd_only_bench.py [--reps 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clock = [c.strip() for c in r.stdout.strip().splitlines()[0].split(",")]
        out.update({"name": name, "power_limit_W": float(power), "max_sm_clock_MHz": float(clock)})
    except Exception as e:      # nvidia-smi missing: the device name alone
        out["nvidia_smi"] = f"unavailable ({type(e).__name__})"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if args.reps < 3:
        ap.error("--reps must be at least 3")
    import ctc_crf
    from cat_b200 import _C, _lib, fst
    from bench import synth_labels
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    V, lamb = 218, 0.01
    tmp = tempfile.mkdtemp(prefix="fwd_only_bench_")
    L = _lib.lib()

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        rise = torch.cuda.max_memory_allocated(dev) - base
        del out
        return ms, rise

    def shape(H, N, T, seed):
        path = os.path.join(tmp, f"den_{H}.fst")
        fst.write_fst(path, fst.make_synthetic_den(H, 24, V, seed=7))
        ctx = ctc_crf.CRFContext(path, gpus=0)
        lab, lens, ly = synth_labels(N, T, V, seed)
        g = torch.Generator(device=dev).manual_seed(seed)
        y = torch.log_softmax(3.0 * torch.randn(N, T, V, device=dev, generator=g), -1).contiguous()
        lab, lx, ly = torch.tensor(lab), torch.tensor(lens), torch.tensor(ly)
        crit = ctc_crf.CTC_CRF_LOSS(lamb=lamb, size_average=True)

        def fwd_only():
            with torch.no_grad():
                return crit(y, lab, lx, ly)

        def loss_and_grad():      # grad mode on, logits not requiring grad: the loss plus its (N,T,V) gradient
            return crit(y, lab, lx, ly)

        arms = {"fwd_only": fwd_only, "loss_and_grad": loss_and_grad}
        ms = {k: [] for k in arms}
        peak = {k: 0 for k in arms}
        for fn in arms.values():   # warm-up (allocator, kernel attributes)
            timed(fn)
        for _ in range(args.reps):
            for k, fn in arms.items():
                t, rise = timed(fn)
                ms[k].append(round(t, 3))
                peak[k] = max(peak[k], rise)
        ev = float(fwd_only().item())
        tr = float(loss_and_grad().item())
        med = {k: statistics.median(v) for k, v in ms.items()}
        res = {
            "graph_arcs": int(_C.den_info()["file_arcs"]), "N": N, "T": T, "V": V,
            "ms": ms, "median_ms": med, "fwd_only_over_loss_and_grad": med["fwd_only"] / med["loss_and_grad"],
            "peak_rise_MB": {k: v / 1e6 for k, v in peak.items()},
            "fwd_only_ring_MB": int(L.ccb_den_fwd_alpha_floats(min(N, _C.MAX_UTTS_PER_CALL))) * 4 / 1e6,
            "full_spill_one_call_GB": int(L.ccb_den_alpha_floats(N, T)) * 4 / 1e9,
            "training_slices": [{"n0": s[0], "n1": s[1], "ckpt_k": s[4]} for s in _C._plan_slices(L, lx, ly, N, V, dev)],
            "loss_fwd_only": ev, "loss_training": tr, "loss_rel_diff": abs(ev - tr) / max(1.0, abs(tr)),
        }
        del y, ctx
        torch.cuda.empty_cache()
        return res

    out = {"card": card(), "reps": args.reps, "timing": "CUDA events per call, arms alternated, median of reps"}
    out["headline_N64_T1500"] = shape(20000, 64, 1500, 1234)
    out["config4_graph_N64_T2000"] = shape(100000, 64, 2000, 4343)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
