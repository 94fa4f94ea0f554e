"""Transducer beam search (``cat_b200.rnnt_decode.rnnt_beam_search``) on an aishell-like shape: N = 64 utterances of T = 120
encoder frames, V = 4232, a one-layer LSTM predictor with hdim 512 and no head, a JointNet ("add") with hdim 512 (CAT's
aishell ``rnnt-v1``), beam 1, 4 and 16, in fp32 and under fp16 autocast.  Random weights: the search does the same work
whatever the hypotheses are.  Reports ms per batch and utterances/s (CUDA events around whole calls, after a warm-up), the
split of GPU time between the step kernel, the predictor and the joiner from a separate torch.profiler run, and the
per-hypothesis torch restatement of CAT's decoder (tests/rnnt_decode_oracle.py) on the first `--ref-n` utterances for
comparison.  Prints one JSON line per configuration; the card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from cat_b200.rnnt_decode import rnnt_beam_search  # noqa: E402
from rnnt_decode_oracle import JointNet, LSTMPredictor, cat_decode  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the card's name from torch at least
        out = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return out


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def split(fn, pred, joiner, kernel="rnnt_beam_step_kernel"):
    """GPU time of the step kernel (named ``kernel``), the predictor and the joiner in one profiled call (ms)."""
    rf = {}

    def pre(name):
        def h(m, a):
            rf[id(m)] = torch.autograd.profiler.record_function(name)
            rf[id(m)].__enter__()
        return h

    def post(m, a, o):
        rf.pop(id(m)).__exit__(None, None, None)

    hs = [pred.register_forward_pre_hook(pre("bench::predictor")), pred.register_forward_hook(post)]
    for m in (joiner.fc_enc, joiner.fc_dec, joiner.fc):
        hs += [m.register_forward_pre_hook(pre("bench::joiner")), m.register_forward_hook(post)]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA, torch.profiler.ProfilerActivity.CPU]) as p:
        fn()
        torch.cuda.synchronize()
    for h in hs:
        h.remove()
    out = {"step_kernel": 0.0, "predictor": 0.0, "joiner": 0.0, "all_kernels": 0.0}
    for e in p.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
        if e.key == "bench::predictor":
            out["predictor"] += t
        elif e.key == "bench::joiner":
            out["joiner"] += t
        elif kernel in e.key:
            out["step_kernel"] += t
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            out["all_kernels"] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return {k: round(v, 2) for k, v in out.items()}


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
    assert torch.cuda.is_available(), "rnnt_decode_bench measures on a GPU"
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
                    return rnnt_beam_search(enc, lens, pred, joiner, beam_size=B)
                ms = timed(run, args.reps)
                sp = split(run, pred, joiner)
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
