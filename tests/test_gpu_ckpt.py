"""Checkpointed denominator on the GPU: alpha kept on a ring of frames plus a checkpoint every K frames, each backward
segment recomputed from its checkpoint.  The slice planner's test hook `_C._ckpt_k_override` forces K on every slice.

Against the full spill on the same inputs: loss 1e-6 relative, both logZ parts 1e-6 relative, gradient 1e-5 absolute
(the recomputed rows equal the first pass's except where hub-row atomics reorder sums).  Against the fp64 oracle: the
north_star tolerances (loss 1e-4 relative, gradient 1e-3 absolute).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _loss(monkeypatch, y_t, labels, lens, ly, lamb, K, from_logits=False):
    """Fused loss with every slice checkpointed every K frames (K None: the planner's choice, the full spill here)."""
    from cat_b200 import _C
    monkeypatch.setattr(_C, "_ckpt_k_override", K)
    loss, grad, parts = _C.ctc_crf_loss_fwd(y_t, torch.tensor(labels, dtype=torch.int32), torch.tensor(lens, dtype=torch.int32),
                                            torch.tensor(ly, dtype=torch.int32), lamb, True, want_parts=True,
                                            from_logits=from_logits)
    monkeypatch.setattr(_C, "_ckpt_k_override", None)
    return float(loss.item()), grad.cpu().numpy(), parts.cpu().numpy()


def _edge_lens(N, T, K, seed):
    """Lengths 0, 1, K, K+1, 2K and T (those that fit in T), the rest random in [1, T]."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, T + 1, size=N).astype(np.int32)
    special = [T, 0, 1] + [v for v in (K, K + 1, 2 * K) if v <= T]
    lens[:min(N, len(special))] = special[:N]
    return lens


def _close(a, b, rtol):
    """(An utterance of length 0 that cannot reach a final state has logZ = -inf, which makes the batch loss NaN on both
    paths: then both must be NaN.)"""
    if not np.isfinite(b):
        assert np.isnan(a) if np.isnan(b) else a == b, (a, b)
        return
    assert abs(a - b) <= rtol * max(1.0, abs(b)), (a, b)


def _close_or_both_infinite(a, oracle_loss):
    if np.isfinite(oracle_loss):
        _close(a, oracle_loss, LOSS_RTOL)
    else:
        assert not np.isfinite(a), (a, oracle_loss)


def _same_as_full(full, ck):
    (l0, g0, p0), (l1, g1, p1) = full, ck
    _close(l1, l0, 1e-6)
    assert np.isfinite(g1).all()
    assert np.abs(g1 - g0).max() < 1e-5
    fin = np.isfinite(p0)
    assert (np.isfinite(p1) == fin).all()
    np.testing.assert_allclose(p1[fin], p0[fin], rtol=1e-6, atol=1e-5)


@pytest.mark.parametrize("name,N", [("tlm_small", 5), ("random_split", 5), ("tlm_mid", 40), ("tlm_mid", 64), ("tlm_mid", 130)])
def test_ckpt_matches_full_spill_and_oracle(tmp_graphs, monkeypatch, name, N):
    """N = 5: small-batch rows (16 floats); 40 / 64: one / two utterances per lane; 130: four per lane forward, 256 lanes.
    K = 1, 2, 7, Tmax and beyond Tmax; lengths 0, 1, K, K+1, a multiple of K and Tmax."""
    from oracle import oracle
    path, g, V = tmp_graphs[name]
    ctx = _ctx(path)
    T = 23
    for K in (1, 2, 7, T, T + 5):
        lens = _edge_lens(N, T, K, seed=K)
        y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=50 + K, lens=lens)
        yt = torch.tensor(y, device="cuda")
        full = _loss(monkeypatch, yt, labels, lens, ly, 0.1, None)
        ck = _loss(monkeypatch, yt, labels, lens, ly, 0.1, K)
        _same_as_full(full, ck)
        for n in range(N):
            assert not ck[1][n, lens[n]:].any()
        if K == 7:
            oloss, ograd, oparts = oracle.ctc_crf(g, y, labels, lens, ly, 0.1)
            _close_or_both_infinite(ck[0], oloss)
            np.testing.assert_allclose(ck[1], ograd, rtol=0, atol=GRAD_ATOL)
            np.testing.assert_allclose(ck[2][:N], oparts["logz_alpha"], rtol=LOSS_RTOL, atol=1e-4)
    del ctx


@pytest.mark.parametrize("env", ["HUBS", "CCB_ARCS_IN_GLOBAL", "CCB_NO_TMA", "CCB_NO_PAIRS", "CCB_NO_MERGE", "CCB_NO_OWN",
                                 "HUBS+CCB_ARCS_IN_GLOBAL"])
def test_ckpt_tiers(tmp_graphs, monkeypatch, env):
    """Every kernel tier under checkpointing: hub rows accumulated from parts, the streamed-arc backward (arcs in global
    memory), register gathers instead of TMA staging, the un-paired plan, two segments per pair, no own-row terms."""
    from oracle import oracle
    for e in env.split("+"):
        if e == "HUBS":
            monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
            monkeypatch.setenv("CCB_PART_ARCS", "7")
        else:
            monkeypatch.setenv(e, "1")
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    T = 30
    for N in (40, 12, 130):
        lens = _edge_lens(N, T, 4, seed=N)
        y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=60 + N, lens=lens)
        yt = torch.tensor(y, device="cuda")
        full = _loss(monkeypatch, yt, labels, lens, ly, 0.05, None)
        ck = _loss(monkeypatch, yt, labels, lens, ly, 0.05, 4)
        _same_as_full(full, ck)
        if N == 12:
            oloss, ograd, _ = oracle.ctc_crf(g, y, labels, lens, ly, 0.05)
            _close_or_both_infinite(ck[0], oloss)
            np.testing.assert_allclose(ck[1], ograd, rtol=0, atol=GRAD_ATOL)
    del ctx


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ckpt_raw_logits_and_bf16(tmp_graphs, monkeypatch, dtype):
    """The raw-logit entry (log_softmax inside) and bf16 logits, checkpointed against the full spill and the oracle."""
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 8, 40
    lens = [40, 40, 35, 21, 14, 7, 6, 1]
    _, labels, lens, ly = oracle.synth_batch(N, T, V, seed=23, lens=lens)
    rng = np.random.default_rng(5)
    z = (4.0 * rng.standard_normal((N, T, V)) + 7.0).astype(np.float32)
    zt = torch.tensor(z, device="cuda").to(dtype).contiguous()
    z_used = zt.float().cpu().numpy()
    for from_logits in (True, False):
        y_in = zt if from_logits else torch.log_softmax(zt.float(), -1).to(dtype).contiguous()
        full = _loss(monkeypatch, y_in, labels, lens, ly, 0.1, None, from_logits)
        ck = _loss(monkeypatch, y_in, labels, lens, ly, 0.1, 7, from_logits)
        _same_as_full(full, ck)
        if from_logits:
            oloss, odz, oparts = oracle.ctc_crf_from_logits(g, z_used, labels, lens, ly, 0.1, size_average=True)
            _close(ck[0], oloss, LOSS_RTOL)
            assert np.abs(ck[1] - odz).max() < GRAD_ATOL
            np.testing.assert_allclose(ck[2][:N], oparts["logz_alpha"], rtol=1e-4, atol=1e-3)
    del ctx


def test_ckpt_planner_picks_checkpoints(tmp_graphs, monkeypatch):
    """With a budget that holds the checkpointed alpha but not the full spill, CTC_CRF_LOSS runs checkpointed (no hook) and
    matches the unconstrained call."""
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C, _lib
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 24, 60
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=71)
    yt = torch.tensor(y, device="cuda")
    full = _loss(monkeypatch, yt, labels, lens, ly, 0.05, None)
    L = _lib.lib()
    k = _C.ckpt_interval(T)
    rest = int(L.ccb_den_aux_bytes(N, T)) + int(L.ccb_ctc_workspace_bytes(N, T, int(ly.max())))
    budget = int(L.ccb_den_ckpt_alpha_floats(N, T, k)) * 4 + rest
    assert budget < int(L.ccb_den_alpha_floats(N, T)) * 4 + rest
    monkeypatch.setattr(_C, "_scratch_budget", lambda dev, need=0: budget)
    assert [s[4] for s in _C._plan_slices(L, torch.tensor(lens), torch.tensor(ly), N, V, yt.device)] == [k]
    logits = yt.clone().requires_grad_(True)
    loss = ctc_crf.CTC_CRF_LOSS(lamb=0.05)(logits, torch.tensor(labels), torch.tensor(lens), torch.tensor(ly))
    loss.backward()
    _close(float(loss.item()), full[0], 1e-6)
    assert np.abs(logits.grad.cpu().numpy() - full[1]).max() < 1e-5
    del ctx
