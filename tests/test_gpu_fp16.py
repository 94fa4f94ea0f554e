"""fp16 logits on the GPU: CTC_CRF_LOSS (log-probs and raw logits), WARP_CTC_LOSS and ctc_align take torch.float16 as they
take bfloat16, reading each element in place and converting it to fp32 at the load.

The central check: an fp16 input gives what an fp32 input of the same (upcast) values gives, `x.half()` against
`x.half().float()` -- loss and logZ to 1e-6 relative (the den passes sum with atomics, so not bit for bit), logp_ctc bit for
bit, gradients to 1e-6 absolute.  Once per group the fp64 oracle, fed the fp16-rounded values, at the north_star tolerances:
loss 1e-4 relative, gradients 1e-3 absolute.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3
SAME_RTOL = 1e-6      # fp16 input against its fp32 upcast: den atomics only
SAME_GRAD = 1e-6


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32)


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _close(a, b, rtol):
    """(A length-0 utterance that cannot reach a final state has logZ = -inf and makes the batch loss NaN on both inputs.)"""
    if not np.isfinite(b):
        assert np.isnan(a) if np.isnan(b) else a == b, (a, b)
        return
    assert abs(a - b) <= rtol * max(1.0, abs(b)), (a, b)


def _edge_lens(N, T, seed):
    """Lengths T, 0 and 1 first, the rest random in [1, T]."""
    lens = np.random.default_rng(seed).integers(1, T + 1, size=N).astype(np.int32)
    lens[:min(N, 3)] = [T, 0, 1][:N]
    return lens


def _inputs(N, T, V, seed, lens, from_logits):
    """(fp16 logits on the GPU, labels, lens, ly): log-probs of the oracle's synthetic batch, or raw encoder-like outputs
    4 randn + 7 (far from normalised, so the raw entry's log-normaliser matters)."""
    from oracle import oracle
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=seed, lens=lens)
    if from_logits:
        y = (4.0 * np.random.default_rng(seed + 1).standard_normal((N, T, V)) + 7.0).astype(np.float32)
    return torch.tensor(y, device="cuda").half(), labels, lens, ly


def _fused(y, labels, lens, ly, lamb, from_logits):
    from cat_b200 import _C
    loss, grad, parts = _C.ctc_crf_loss_fwd(y, _i32(labels), _i32(lens), _i32(ly), lamb, True, want_parts=True,
                                            from_logits=from_logits)
    return float(loss.item()), grad.cpu().numpy(), parts.cpu().numpy()


def _same(h, f):
    """(loss, grad, parts) of the fp16 input against those of its fp32 upcast."""
    (l0, g0, p0), (l1, g1, p1) = f, h
    N = p0.size // 2
    _close(l1, l0, SAME_RTOL)
    for a, b in zip(p1[:N], p0[:N]):                        # logZ
        _close(float(a), float(b), SAME_RTOL)
    assert np.array_equal(p1[N:], p0[N:]), (p1[N:], p0[N:])   # logp_ctc, bit for bit
    if g0 is not None:
        assert g1.dtype == np.float32
        assert np.array_equal(np.isnan(g1), np.isnan(g0))
        np.testing.assert_allclose(g1, g0, rtol=0, atol=SAME_GRAD)


def _fused_pair(y16, labels, lens, ly, lamb, from_logits):
    h = _fused(y16, labels, lens, ly, lamb, from_logits)
    f = _fused(y16.float(), labels, lens, ly, lamb, from_logits)
    _same(h, f)
    return h


def _check_oracle(g, y16, labels, lens, ly, lamb, from_logits, got):
    """The fp64 oracle on the fp16-rounded values."""
    from oracle import oracle
    loss, grad, parts = got
    N = len(lens)
    y_used = y16.float().cpu().numpy()
    if from_logits:
        oloss, ograd, oparts = oracle.ctc_crf_from_logits(g, y_used, labels, lens, ly, lamb)
    else:
        oloss, ograd, oparts = oracle.ctc_crf(g, y_used, labels, lens, ly, lamb)
    if np.isfinite(oloss):
        _close(loss, oloss, LOSS_RTOL)
    else:
        assert not np.isfinite(loss), (loss, oloss)
    ok = np.isfinite(oparts["logz_alpha"])
    np.testing.assert_allclose(parts[:N][ok], oparts["logz_alpha"][ok], rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(parts[N:], oparts["logp_ctc"], rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(grad[ok] - ograd[ok]).max() < GRAD_ATOL      # (the rows of utterances with a finite logZ)


@pytest.mark.parametrize("from_logits", [False, True])
@pytest.mark.parametrize("name,N", [("tlm_small", 5), ("random_split", 5), ("tlm_mid", 40), ("tlm_mid", 64), ("tlm_mid", 130)])
def test_fused_fp16_equals_upcast(tmp_graphs, name, N, from_logits):
    """N = 5: small-batch rows (16 floats); 40 / 64: one / two utterances per lane; 130: three slices (64, 64, 2).
    Lengths 0, 1 and T."""
    path, g, V = tmp_graphs[name]
    ctx = _ctx(path)
    T = 23
    y16, labels, lens, ly = _inputs(N, T, V, 110 + N, _edge_lens(N, T, seed=N), from_logits)
    h = _fused_pair(y16, labels, lens, ly, 0.1, from_logits)
    if N == 40:
        _check_oracle(g, y16, labels, lens, ly, 0.1, from_logits, h)
    del ctx


@pytest.mark.parametrize("env", ["HUBS", "CCB_ARCS_IN_GLOBAL", "CCB_NO_TMA", "CCB_NO_PAIRS", "CCB_NO_MERGE", "CCB_NO_OWN"])
def test_fp16_tiers(tmp_graphs, monkeypatch, env):
    """Every den tier the test hooks select, with and without a gradient: hub rows accumulated from parts, arcs in global
    memory, register gathers instead of TMA staging, the un-paired plan, two segments per pair, no own-row terms."""
    from cat_b200 import _C
    if env == "HUBS":
        monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
        monkeypatch.setenv("CCB_PART_ARCS", "7")
    else:
        monkeypatch.setenv(env, "1")
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    T = 30
    for N in (40, 12, 130):
        from_logits = N != 40
        y16, labels, lens, ly = _inputs(N, T, V, 120 + N, _edge_lens(N, T, seed=N + 1), from_logits)
        h = _fused_pair(y16, labels, lens, ly, 0.05, from_logits)
        args = (_i32(labels), _i32(lens), _i32(ly), 0.05, True)
        fh = _C.ctc_crf_loss_fwd_only(y16, *args, want_parts=True, from_logits=from_logits)
        ff = _C.ctc_crf_loss_fwd_only(y16.float(), *args, want_parts=True, from_logits=from_logits)
        _same((float(fh[0].item()), None, fh[1].cpu().numpy()), (float(ff[0].item()), None, ff[1].cpu().numpy()))
        if N == 12:
            _check_oracle(g, y16, labels, lens, ly, 0.05, from_logits, h)
    del ctx


@pytest.mark.parametrize("from_logits", [False, True])
def test_fp16_checkpointed(tmp_graphs, monkeypatch, from_logits):
    """The checkpointed denominator (alpha on a ring, segments recomputed from checkpoints every K frames) on fp16 input."""
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 40, 30
    y16, labels, lens, ly = _inputs(N, T, V, 130, _edge_lens(N, T, seed=7), from_logits)
    monkeypatch.setattr(_C, "_ckpt_k_override", 4)
    h = _fused_pair(y16, labels, lens, ly, 0.1, from_logits)
    _check_oracle(g, y16, labels, lens, ly, 0.1, from_logits, h)
    monkeypatch.setattr(_C, "_ckpt_k_override", None)
    del ctx


def test_fp16_fwd_only_and_modules(tmp_graphs):
    """ctc_crf_loss_fwd_only on fp16, and CTC_CRF_LOSS on fp16 through the Modules: under torch.no_grad the loss of the
    upcast input; with grad mode on the gradient comes back as fp16 on both entries (the raw entry casts it, autograd casts
    it on the log-prob entry) and equals the upcast input's fp32 gradient rounded to fp16."""
    import ctc_crf
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 48, 40
    for from_logits in (False, True):
        y16, labels, lens, ly = _inputs(N, T, V, 140, None, from_logits)
        lab, lx, lyt = _i32(labels), _i32(lens), _i32(ly)
        args = (lab, lx, lyt, 0.1, True)
        fh = _C.ctc_crf_loss_fwd_only(y16, *args, want_parts=True, from_logits=from_logits)
        ff = _C.ctc_crf_loss_fwd_only(y16.float(), *args, want_parts=True, from_logits=from_logits)
        _same((float(fh[0].item()), None, fh[1].cpu().numpy()), (float(ff[0].item()), None, ff[1].cpu().numpy()))
        crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits)
        with torch.no_grad():
            e16, e32 = crit(y16, lab, lx, lyt), crit(y16.float(), lab, lx, lyt)
        _close(float(e16.item()), float(e32.item()), SAME_RTOL)
        x16 = y16.clone().requires_grad_(True)
        x32 = y16.float().requires_grad_(True)
        l16, l32 = crit(x16, lab, lx, lyt), crit(x32, lab, lx, lyt)
        (l16 * 2.0).backward()
        (l32 * 2.0).backward()
        _close(float(l16.item()), float(l32.item()), SAME_RTOL)
        _close(float(e16.item()), float(l16.item()), SAME_RTOL)
        assert x16.grad.dtype == torch.float16 and x32.grad.dtype == torch.float32
        g16, g32 = x16.grad.float().cpu().numpy(), x32.grad.cpu().numpy()
        # the fp32 gradient rounded once to fp16: half an fp16 ulp (2^-11 relative) above the atomics' spread
        assert (np.abs(g16 - g32) <= SAME_GRAD + 2.0 ** -11 * np.abs(g32)).all(), np.abs(g16 - g32).max()
    del ctx


def test_fp16_ctc_loss_and_warp_ctc():
    """ctc_loss_fwd / ctc_loss_fwd_only on fp16 against the upcast input (the numerator is deterministic: logp and loss bit
    for bit), WARP_CTC_LOSS with a backward pass (fp16 gradient) and under torch.no_grad, and the fp64 oracle."""
    import ctc_crf
    from cat_b200 import _C
    from oracle import oracle
    N, T, V = 24, 50, 30
    y16, labels, lens, ly = _inputs(N, T, V, 150, _edge_lens(N, T, seed=3), False)
    lab, lx, lyt = _i32(labels), _i32(lens), _i32(ly)
    l16, g16, p16 = _C.ctc_loss_fwd(y16, lab, lx, lyt, True)
    l32, g32, p32 = _C.ctc_loss_fwd(y16.float(), lab, lx, lyt, True)
    assert torch.equal(p16, p32) and torch.equal(l16, l32)
    assert g16.dtype == torch.float32
    np.testing.assert_allclose(g16.cpu().numpy(), g32.cpu().numpy(), rtol=0, atol=SAME_GRAD)
    f16, q16 = _C.ctc_loss_fwd_only(y16, lab, lx, lyt, True)
    assert torch.equal(q16, p16) and torch.equal(f16, l16)
    warp = ctc_crf.WARP_CTC_LOSS()
    x16 = y16.clone().requires_grad_(True)
    w16 = warp(x16, lab, lx, lyt)
    w16.backward()
    assert float(w16.item()) == float(l16.item())
    assert x16.grad.dtype == torch.float16
    gg, gr = x16.grad.float().cpu().numpy(), g32.cpu().numpy()
    assert (np.abs(gg - gr) <= SAME_GRAD + 2.0 ** -11 * np.abs(gr)).all(), np.abs(gg - gr).max()
    with torch.no_grad():
        assert float(warp(y16, lab, lx, lyt).item()) == float(l16.item())
    olp, og = oracle.ctc(y16.float().cpu().numpy(), labels, ly, lens)
    np.testing.assert_allclose(p16.cpu().numpy(), olp, rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(g16.cpu().numpy() * N + og).max() < GRAD_ATOL      # grad = -gamma_ctc / N


def test_fp16_ctc_align():
    """Best-path alignment of fp16 log-probs: the alignment of the upcast input, the score bit for bit."""
    import ctc_crf
    N, T, V = 20, 60, 25
    y16, labels, lens, ly = _inputs(N, T, V, 160, _edge_lens(N, T, seed=4), False)
    lab, lx, lyt = _i32(labels), _i32(lens), _i32(ly)
    a16, s16 = ctc_crf.ctc_align(y16, lab, lx, lyt)
    a32, s32 = ctc_crf.ctc_align(y16.float(), lab, lx, lyt)
    assert torch.equal(a16, a32)
    assert torch.equal(s16, s32)
    assert torch.isfinite(s16[0])


def test_config3_fp16_raw_logits(tmp_path):
    """At size: config 3's shape (V=72, N=64, T=1500, 1.02 M-arc den graph) with fp16 RAW logits, as an fp16 autocast encoder
    returns them: the upcast input's loss, parts and gradient, and the fp64 oracle on two utterances."""
    from cat_b200 import fst
    from oracle import oracle
    V, N, T, lamb = 72, 64, 1500, 0.01
    g = fst.make_synthetic_den(20000, 24, V, seed=7)
    path = str(tmp_path / "den_20000_72.fst")
    fst.write_fst(path, g)
    ctx = _ctx(path)
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=1234)
    shift = np.random.default_rng(9).standard_normal((N, T, 1)).astype(np.float32) * 3.0
    z16 = torch.tensor(y + shift, device="cuda").half()
    h = _fused_pair(z16, labels, lens, ly, lamb, True)
    loss, grad, parts = h
    assert np.isfinite(loss)
    sub = [0, N - 1]
    off = np.concatenate([[0], np.cumsum(ly)])
    sub_labels = np.concatenate([labels[off[i]:off[i + 1]] for i in sub])
    z_used = z16.float().cpu().numpy()[sub].astype(np.float64)
    y64 = z_used - np.log(np.exp(z_used - z_used.max(-1, keepdims=True)).sum(-1, keepdims=True)) - z_used.max(-1, keepdims=True)
    # (oracle.ctc_crf_from_logits composed with the scaled-linear fp64 den evaluation, which at-size tests use)
    _, og, oparts = oracle.ctc_crf(g, y64.astype(np.float32), sub_labels, lens[sub], ly[sub], lamb, size_average=False,
                                   nthreads=len(sub), fast=True)
    odz = og - np.exp(y64) * og.sum(-1, keepdims=True)
    d = np.abs(grad[sub] * N - odz).max()
    print("config 3 (fp16 raw logits) max |grad - oracle| (x N):", d)
    assert d < GRAD_ATOL
    np.testing.assert_allclose(parts[:N][sub], oparts["logz_alpha"], rtol=LOSS_RTOL)
    np.testing.assert_allclose(parts[N:][sub], oparts["logp_ctc"], rtol=LOSS_RTOL)
    del ctx
