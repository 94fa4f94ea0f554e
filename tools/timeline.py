"""Per-warp timeline of the persistent den kernels (profiling aid): where does a frame's time go?
   python tools/timeline.py [--T 200] -> gpurun_out/timeline.npz + a text summary"""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import ctc_crf
from cat_b200 import _lib, _C, fst

ap = argparse.ArgumentParser(); ap.add_argument("--T", type=int, default=200); ap.add_argument("--N", type=int, default=64)
ap.add_argument("--H", type=int, default=20000); a = ap.parse_args()
N, T, V = a.N, a.T, 218
path = f"/tmp/ccb_tl_{a.H}.fst"
if not os.path.exists(path): fst.write_fst(path, fst.make_synthetic_den(a.H, 24, V, seed=7))
ctx = ctc_crf.CRFContext(path, gpus=0)
L = _lib.lib()
y = torch.log_softmax(3 * torch.randn(N, T, V, device="cuda"), -1)
lens = torch.full((N,), T, dtype=torch.int32, device="cuda")
alpha = torch.empty(int(L.ccb_den_alpha_floats(N, T)), device="cuda"); aux = torch.empty(int(L.ccb_den_aux_bytes(N, T)), dtype=torch.uint8, device="cuda")
grad = torch.zeros(N, T, V, device="cuda"); logz = torch.empty(N, device="cuda")
n_ctas = torch.cuda.get_device_properties(0).multi_processor_count   # one CTA per SM (den_graph.cc)
n_chunks = n_ctas * 16; steps, step0 = 16, T // 2   # 16 warps per CTA, one chunk each
stream = torch.cuda.current_stream().cuda_stream
def run():
    rc = L.ccb_den_forward_backward(y.data_ptr(), 0, T * V, V, N, T, V, lens.data_ptr(), alpha.data_ptr(), aux.data_ptr(), grad.data_ptr(), T * V, V, 1.0, logz.data_ptr(), None, stream)
    assert rc == 0, _lib.last_error()
run(); torch.cuda.synchronize()
out = {}
for name in ("fwd", "bwd"):
    tl = torch.zeros(steps * n_chunks * 4, dtype=torch.int64, device="cuda")
    # forward frames are indexed by t, backward by (Tmax - tau); both kernels write the same buffer, so run twice and
    # keep the pass we want by looking at which pass ran last is not possible -> use separate runs with grad on/off
    L.ccb_debug_timeline(tl.data_ptr(), step0, steps)
    if name == "fwd":
        rc = L.ccb_den_forward_backward(y.data_ptr(), 0, T * V, V, N, T, V, lens.data_ptr(), alpha.data_ptr(), aux.data_ptr(), None, T * V, V, 1.0, logz.data_ptr(), None, stream)
    else:
        run()   # backward overwrites the forward's records
    torch.cuda.synchronize(); L.ccb_debug_timeline(None, 0, 0)
    out[name] = tl.cpu().numpy().reshape(steps, n_chunks, 4)
os.makedirs("gpurun_out", exist_ok=True); np.savez_compressed("gpurun_out/timeline.npz", **out)
for name, r in out.items():
    work = (r[:, :, 2] - r[:, :, 1]).astype(np.float64); total = (r[:, :, 3] - r[:, :, 1]).astype(np.float64)
    g0 = r[:, :, 0].astype(np.float64); step_ns = np.diff(g0.min(1))
    print(f"{name}: frame period {step_ns.mean()/1e3:.2f} us (globaltimer); per-warp work cycles mean {work.mean():.0f} p50 {np.median(work):.0f} p99 {np.percentile(work,99):.0f} max {work.max():.0f}; frame cycles mean {total.mean():.0f}")
    cta = work.reshape(steps, n_ctas, -1).max(2)
    print(f"   slowest warp per CTA: mean {cta.mean():.0f} max {cta.max():.0f} min {cta.min():.0f}; start skew across CTAs (ns) p50 {np.median(g0.max(1)-g0.min(1)):.0f}")
    print("   work/frame ratio mean %.2f ; (max work)/frame %.2f" % ((work/total).mean(), (work.max(1)/total.mean(1)).mean()))
    wait = total - work
    print(f"   barrier wait cycles mean {wait.mean():.0f} p50 {np.median(wait):.0f}; walk of the slowest warp per frame mean {work.max(1).mean():.0f}")
