"""Forward-only loss on the GPU (`_C.ctc_crf_loss_fwd_only`, `_C.ctc_loss_fwd_only`, and CTC_CRF_LOSS / WARP_CTC_LOSS
under torch.no_grad): the den forward pass on the ring of frames, the numerator without its cell spill, no gradient.

Against the training path (`_C.ctc_crf_loss_fwd`) on the same inputs: loss and logZ 1e-6 relative, logp_ctc bit-identical
(the numerator's arithmetic is the same).  Against the fp64 oracle, once per group: the north_star tolerances (1e-4).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32)


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _close(a, b, rtol):
    """(A length-0 utterance that cannot reach a final state has logZ = -inf and makes the batch loss NaN on both paths.)"""
    if not np.isfinite(b):
        assert np.isnan(a) if np.isnan(b) else a == b, (a, b)
        return
    assert abs(a - b) <= rtol * max(1.0, abs(b)), (a, b)


def _both(y_t, labels, lens, ly, lamb, from_logits=False):
    """(loss, parts) of the training path and of the forward-only path on the same inputs."""
    from cat_b200 import _C
    args = (y_t, _i32(labels), _i32(lens), _i32(ly), lamb, True)
    l0, _, p0 = _C.ctc_crf_loss_fwd(*args, want_parts=True, from_logits=from_logits)
    l1, p1 = _C.ctc_crf_loss_fwd_only(*args, want_parts=True, from_logits=from_logits)
    return (float(l0.item()), p0.cpu().numpy()), (float(l1.item()), p1.cpu().numpy())


def _same_as_training(train, fwd):
    (l0, p0), (l1, p1) = train, fwd
    N = p0.size // 2
    _close(l1, l0, 1e-6)
    for a, b in zip(p1[:N], p0[:N]):       # logZ
        _close(float(a), float(b), 1e-6)
    assert np.array_equal(p1[N:], p0[N:]), np.abs(p1[N:] - p0[N:]).max()   # logp_ctc, bit for bit


def _edge_lens(N, T, seed):
    """Lengths T, 0 and 1 first, the rest random in [1, T]."""
    lens = np.random.default_rng(seed).integers(1, T + 1, size=N).astype(np.int32)
    special = [T, 0, 1]
    lens[:min(N, 3)] = special[:N]
    return lens


def _check_oracle(g, y, labels, lens, ly, lamb, fwd):
    from oracle import oracle
    loss, parts = fwd
    N = len(lens)
    oloss, _, oparts = oracle.ctc_crf(g, y, labels, lens, ly, lamb)
    if np.isfinite(oloss):
        _close(loss, oloss, LOSS_RTOL)
    else:
        assert not np.isfinite(loss), (loss, oloss)
    np.testing.assert_allclose(parts[:N], oparts["logz_alpha"], rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(parts[N:], oparts["logp_ctc"], rtol=LOSS_RTOL, atol=1e-4)


@pytest.mark.parametrize("name,N", [("tlm_small", 5), ("random_split", 5), ("tlm_mid", 40), ("tlm_mid", 64), ("tlm_mid", 130)])
def test_fwd_only_matches_training_path(tmp_graphs, name, N):
    """N = 5: small-batch rows (16 floats); 40 / 64: one / two utterances per lane; 130: three slices (64, 64, 2).
    Lengths 0, 1 and T."""
    from oracle import oracle
    path, g, V = tmp_graphs[name]
    ctx = _ctx(path)
    T = 23
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=90 + N, lens=_edge_lens(N, T, seed=N))
    yt = torch.tensor(y, device="cuda")
    train, fwd = _both(yt, labels, lens, ly, 0.1)
    _same_as_training(train, fwd)
    if N == 40:
        _check_oracle(g, y, labels, lens, ly, 0.1, fwd)
    del ctx


@pytest.mark.parametrize("env", ["HUBS", "CCB_ARCS_IN_GLOBAL", "CCB_NO_TMA", "CCB_NO_PAIRS", "CCB_NO_MERGE", "CCB_NO_OWN"])
def test_fwd_only_tiers(tmp_graphs, monkeypatch, env):
    """Every forward tier the test hooks select: hub rows accumulated from parts, arcs in global memory, register gathers
    instead of TMA staging, the un-paired plan, two segments per pair, no own-row terms."""
    if env == "HUBS":
        monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
        monkeypatch.setenv("CCB_PART_ARCS", "7")
    else:
        monkeypatch.setenv(env, "1")
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    T = 30
    for N in (40, 12, 130):
        y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=70 + N, lens=_edge_lens(N, T, seed=N + 1))
        yt = torch.tensor(y, device="cuda")
        train, fwd = _both(yt, labels, lens, ly, 0.05)
        _same_as_training(train, fwd)
        if N == 12:
            _check_oracle(g, y, labels, lens, ly, 0.05, fwd)
    del ctx


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fwd_only_raw_logits_and_bf16(tmp_graphs, dtype):
    """The raw-logit entry (its logZ normalised by the per-utterance log-normaliser on the ring too) and bf16 logits."""
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 8, 40
    _, labels, lens, ly = oracle.synth_batch(N, T, V, seed=23, lens=[40, 40, 35, 21, 14, 7, 6, 1])
    z = (4.0 * np.random.default_rng(5).standard_normal((N, T, V)) + 7.0).astype(np.float32)
    zt = torch.tensor(z, device="cuda").to(dtype).contiguous()
    z_used = zt.float().cpu().numpy()
    for from_logits in (True, False):
        y_in = zt if from_logits else torch.log_softmax(zt.float(), -1).to(dtype).contiguous()
        train, fwd = _both(y_in, labels, lens, ly, 0.1, from_logits)
        _same_as_training(train, fwd)
        if from_logits:
            oloss, _, oparts = oracle.ctc_crf_from_logits(g, z_used, labels, lens, ly, 0.1, size_average=True)
            _close(fwd[0], oloss, LOSS_RTOL)
            np.testing.assert_allclose(fwd[1][:N], oparts["logz_alpha"], rtol=1e-4, atol=1e-3)
            np.testing.assert_allclose(fwd[1][N:], oparts["logp_ctc"], rtol=1e-4, atol=1e-3)
    del ctx


def test_modules_under_no_grad(tmp_graphs):
    """CTC_CRF_LOSS and WARP_CTC_LOSS under torch.no_grad / inference_mode: the loss of grad mode, no gradient, the
    forward-only launches only, and no more memory than the ring, the aux block and the log-likelihoods."""
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C, _lib
    L = _lib.lib()
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 48, 60
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=31)
    yt = torch.tensor(y, device="cuda")
    lab, lx, lyt = _i32(labels), _i32(lens), _i32(ly)
    for from_logits in (False, True):
        crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits)
        trained = crit(yt.clone().requires_grad_(True), lab, lx, lyt)
        with torch.no_grad():
            c0 = _C.launch_count()
            ev = crit(yt, lab, lx, lyt)
            launches = _C.launch_count() - c0
        with torch.inference_mode():
            ev2 = crit(yt, lab, lx, lyt)
        assert not ev.requires_grad and ev.shape == (1,) and ev.is_cuda
        _close(float(ev.item()), float(trained.item()), 1e-6)
        _close(float(ev2.item()), float(ev.item()), 1e-6)    # (the den passes sum with atomics: not bit for bit)
        assert launches == (5 if from_logits else 4), launches      # frame max (+ normaliser), den forward, numerator, loss
    # peak memory: the ring, the aux block and N floats of log-likelihoods, nothing of size N x T x V
    crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        crit(yt, lab, lx, lyt)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    bound = (int(L.ccb_den_fwd_alpha_floats(N)) * 4 + int(L.ccb_den_aux_bytes(N, T)) + int(L.ccb_num_fwd_only_bytes(N))
             + (64 << 20))
    assert rise <= bound, (rise, bound)
    # an infeasible utterance (more labels than frames) still makes the loss +inf
    ly_bad = ly.copy()
    ly_bad[3] = lens[3] + 2
    labels_bad = np.random.default_rng(4).integers(1, V, size=int(ly_bad.sum())).astype(np.int32)
    with torch.no_grad():
        bad = ctc_crf.CTC_CRF_LOSS(lamb=0.1)(yt, _i32(labels_bad), lx, _i32(ly_bad))
    assert float(bad.item()) == float("inf")
    # WARP_CTC_LOSS: the same loss as with grad mode on, bit for bit, from two launches (numerator, sum)
    warp = ctc_crf.WARP_CTC_LOSS()
    trained = warp(yt.clone().requires_grad_(True), lab, lx, lyt)
    with torch.no_grad():
        c0 = _C.launch_count()
        ev = warp(yt, lab, lx, lyt)
        assert _C.launch_count() - c0 == 2
    assert float(ev.item()) == float(trained.item())
    for dt in (torch.float32, torch.bfloat16):
        yd = yt.to(dt).contiguous()
        _, _, lp0 = _C.ctc_loss_fwd(yd, lab, lx, lyt, True)
        l1, lp1 = _C.ctc_loss_fwd_only(yd, lab, lx, lyt, True)
        assert torch.equal(lp0, lp1)
    with torch.no_grad():
        assert float(warp(yt, _i32(labels_bad), lx, _i32(ly_bad)).item()) == float("inf")
    del ctx


def test_fwd_only_config4_graph_one_call(tmp_path):
    """At size: config 4's den graph (H=100 000 -> 5.09 M arcs), N=64, T=2000.  The training path's full alpha spill of
    this batch is 102.6 GB; forward-only it is one native call whose memory is the ring (about 0.36 GB), and its loss is the
    training path's.  Two utterances' parts against the fp64 oracle."""
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C, _lib, fst
    V, N, T, lamb = 218, 64, 2000, 0.01
    g = fst.make_synthetic_den(100000, 24, V, seed=7)
    path = str(tmp_path / "den_100000.fst")
    fst.write_fst(path, g)
    ctx = _ctx(path)
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=4343)
    yt = torch.tensor(y, device="cuda")
    lab, lx, lyt = _i32(labels), _i32(lens), _i32(ly)
    L = _lib.lib()
    assert len(_C._plan_fwd_only_slices(L, lx, lyt, N, yt.device)) == 1
    crit = ctc_crf.CTC_CRF_LOSS(lamb=lamb)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        ev = crit(yt, lab, lx, lyt)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    ring = int(L.ccb_den_fwd_alpha_floats(N)) * 4
    bound = ring + int(L.ccb_den_aux_bytes(N, T)) + int(L.ccb_num_fwd_only_bytes(N)) + (64 << 20)
    print(f"config 4 graph, N={N}, T={T}, forward only: peak rise {rise / 2**30:.3f} GiB (ring {ring / 2**30:.3f} GiB, "
          f"bound {bound / 2**30:.3f} GiB; full spill {int(L.ccb_den_alpha_floats(N, T)) * 4 / 1e9:.1f} GB)")
    assert rise <= bound
    trained = crit(yt, lab, lx, lyt)
    _close(float(ev.item()), float(trained.item()), 1e-6)
    _, parts = _C.ctc_crf_loss_fwd_only(yt, lab, lx, lyt, lamb, True, want_parts=True)
    p = parts.cpu().numpy()
    sub = [0, N - 1]
    off = np.concatenate([[0], np.cumsum(ly)])
    sub_labels = np.concatenate([labels[off[i]:off[i + 1]] for i in sub])
    _, _, oparts = oracle.ctc_crf(g, y[sub], sub_labels, lens[sub], ly[sub], lamb, size_average=False,
                                  nthreads=len(sub), fast=True)
    np.testing.assert_allclose(p[:N][sub], oparts["logz_alpha"], rtol=LOSS_RTOL)
    np.testing.assert_allclose(p[N:][sub], oparts["logp_ctc"], rtol=LOSS_RTOL)
    del ctx
