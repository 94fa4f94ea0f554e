"""At size: config 4's den graph (H=100 000 -> 5.09 M arcs, S=199 999) with 8 utterances of up to 3000 frames.  Its arc
stream does not fit shared memory, so every batch takes at least 32 lanes and the full alpha spill of this batch is
77 GB: the slice planner must choose the checkpointed denominator by itself (no hook)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3


def test_config4_graph_t3000_runs_checkpointed(tmp_path):
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C, _lib, fst
    V, N, lamb = 218, 8, 0.01
    g = fst.make_synthetic_den(100000, 24, V, seed=7)
    path = str(tmp_path / "den_100000.fst")
    fst.write_fst(path, g)
    ctx = ctc_crf.CRFContext(path, gpus=0)
    lens = np.array([3000, 2950, 2600, 2100, 1500, 900, 520, 301], np.int32)
    T = int(lens.max())
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=1234, lens=lens)
    yt = torch.tensor(y, device="cuda")
    lab_t, lx_t, ly_t = (torch.tensor(a, dtype=torch.int32) for a in (labels, lens, ly))
    L = _lib.lib()
    full = int(L.ccb_den_alpha_floats(N, T)) * 4
    assert full > 70e9
    slices = _C._plan_slices(L, lx_t, ly_t, N, V, yt.device)
    assert len(slices) == 1 and slices[0][4] == _C.ckpt_interval(T), slices
    k = slices[0][4]
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    loss, grad, parts = _C.ctc_crf_loss_fwd(yt, lab_t, lx_t, ly_t, lamb, True, want_parts=True)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    bound = (int(L.ccb_den_ckpt_alpha_floats(N, T, k)) * 4 + int(L.ccb_den_aux_bytes(N, T))
             + int(L.ccb_ctc_workspace_bytes(N, T, int(ly.max()))) + N * T * V * 4 + (64 << 20))
    print(f"config 4 graph, N={N}, T={T}: K={k}, peak rise {rise / 2**30:.2f} GiB (bound {bound / 2**30:.2f} GiB, "
          f"full spill would be {full / 2**30:.1f} GiB)")
    assert rise <= bound
    assert np.isfinite(float(loss.item()))
    for n in range(N):
        assert not bool(grad[n, lens[n]:].any())
    sub = [0, N - 1]
    off = np.concatenate([[0], np.cumsum(ly)])
    sub_labels = np.concatenate([labels[off[i]:off[i + 1]] for i in sub])
    oloss, ograd, oparts = oracle.ctc_crf(g, y[sub], sub_labels, lens[sub], ly[sub], lamb, size_average=False,
                                          nthreads=len(sub), fast=True)
    got = grad[torch.tensor(sub)].cpu().numpy() * N
    d = np.abs(got - ograd).max()
    print("config 4 graph checkpointed max |grad - oracle| (x N):", d)
    assert d < GRAD_ATOL
    p = parts.cpu().numpy()
    np.testing.assert_allclose(p[:N][sub], oparts["logz_alpha"], rtol=LOSS_RTOL)
    np.testing.assert_allclose(p[N:][sub], oparts["logp_ctc"], rtol=LOSS_RTOL)
    del ctx
