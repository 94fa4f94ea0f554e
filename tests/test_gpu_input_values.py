"""GPU: what the kernels read and what they do with -inf, on every entry.

An encoder hands the loss two kinds of values the rest of the suite never feeds it:

a. junk in the padding.  A key-padding-masked attention layer gives NaN in padded frames (a softmax over no keys is 0/0),
   and fp16 activations there can overflow to +-inf.  Nothing at t >= lx[n], and nothing outside the (N,T,V) block, may
   be read: each entry runs on a clean batch and on copies whose padding is NaN, +inf or -inf, with the logits placed in
   the middle of a buffer whose guard bands before and after hold NaN.  Every output must be what the clean run gives
   (to 1e-6, gradients to 1e-6 plus 32 fp32 ulps: the runs differ only in the order of the den's atomic sums, see
   SAME_ULPS), finite where it is finite, and the gradient rows at t >= lx[n] of every run exactly zero.  The clean run is also checked against the fp64 oracle.
b. -inf log-probabilities in valid frames.  Vocabulary masks, blank suppression and masked_fill(mask, -inf) before
   log_softmax give exact -inf entries, and raw logits can hold -inf too.  Costs, gradients, zero_infinity and the
   alignment against the fp64 oracle (pinned against path enumeration in tests/test_oracle.py) and torch's fp64 ctc_loss.
c. large finite raw logits (fp32 offset by 1e4, fp16 near +-6e4 with a frame's logits within the den's range), against
   the oracle's fp64 log_softmax.

Tolerances against the oracle are the suite's: loss 1e-4 relative, gradients 1e-3 absolute (plus half an ulp of a
16-bit gradient).
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3
SAME_TOL = 1e-6       # poisoned against clean: relative for losses and log-likelihoods, absolute for gradients ...
SAME_ULPS = 32        # ... plus this many fp32 ulps of the value for gradients.  The den normalises each gradient row by a
                      # sum of occupancies accumulated with fp32 atomics in no fixed order, so two runs on the same input
                      # differ by a few ulps RELATIVE to each entry: 20 repeated clean runs of _C.gpu_den on an H100 (tlm_mid,
                      # T = 20) gave at most 5.4e-7 / 7.2e-7 / 1.01e-6 absolute and 8.9e-7 / 8.3e-7 / 1.28e-6 relative
                      # (11 ulps) at N = 12 / 40 / 130, so 1e-6 absolute alone fails now and then at N = 130
LAMB = 0.1
GUARD = 4096          # NaN elements before and after the logits
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
POISONS = (math.nan, math.inf, -math.inf)


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32)


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _guarded(y, fill=math.nan):
    """y (a CUDA tensor) copied into the contiguous middle of a buffer whose GUARD elements on each side hold `fill`."""
    buf = torch.full((y.numel() + 2 * GUARD,), fill, dtype=y.dtype, device="cuda")
    v = buf[GUARD:GUARD + y.numel()].view(y.shape)
    v.copy_(y)
    return v


def _past(lens, T, device="cuda"):
    return torch.arange(T, device=device)[None, :] >= torch.tensor(np.asarray(lens), device=device)[:, None]


def _poisoned(y, lens, value):
    p = y.clone()
    p[_past(lens, y.shape[1])] = value
    return p


def _same(clean, got, what):
    """Every output of a poisoned run against the clean run: the same non-finite values (NaN, +inf, -inf) at the same
    places, finite values within SAME_TOL (gradients absolute plus SAME_ULPS fp32 ulps and one ulp of a 16-bit gradient;
    the rest relative),
    alignments identical."""
    for k, a in clean.items():
        if k.startswith("_"):
            continue
        b = got[k]
        if k == "align":
            assert np.array_equal(a, b), (what, k)
            continue
        fa, fb = np.isfinite(a), np.isfinite(b)
        assert np.array_equal(fa, fb), (what, k, a[fa != fb], b[fa != fb])
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~fa & ~np.isnan(a)], b[~fb & ~np.isnan(b)]), \
            (what, k)
        if k.startswith("grad"):
            tol = SAME_TOL + (SAME_ULPS * float(np.finfo(np.float32).eps) + got["_eps"]) * np.abs(a[fa])
        else:
            tol = SAME_TOL * np.maximum(1.0, np.abs(a[fa]))
        assert np.all(np.abs(a[fa] - b[fa]) <= tol), (what, k, np.abs(a[fa] - b[fa]).max())


def _weights(N):
    """Weights of the per-utterance costs, |w| <= 1 so that a weighted gradient keeps the 1e-6 of an unweighted one."""
    return np.linspace(-1.0, 0.9, N).astype(np.float32)


def _np(out, dtype):
    """CUDA results -> float64 numpy; `_eps` is one ulp of the dtype gradients come back in."""
    r = {k: (v.detach().cpu().numpy() if k == "align" else v.detach().float().cpu().numpy().astype(np.float64))
         for k, v in out.items()}
    r["_eps"] = float(torch.finfo(dtype).eps) if dtype != torch.float32 else 0.0
    return r


# ---------------------------------------------------------------------------------------------------------------------
# the entries, each returning its outputs
# ---------------------------------------------------------------------------------------------------------------------
def _crf_autograd(x, labels, lens, ly, fl):
    """CTC_CRF_LOSS through autograd (the scalar of size_average) and the parts of the same native call."""
    import ctc_crf
    from cat_b200 import _C
    a = (_i32(labels), _i32(lens), _i32(ly))
    x.requires_grad_(True)
    loss = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, from_logits=fl)(x, *a)
    (g,) = torch.autograd.grad(loss, x)
    x.requires_grad_(False)
    _, _, parts = _C.ctc_crf_loss_fwd(x, *a, LAMB, True, want_parts=True, from_logits=fl)
    return dict(loss=loss, grad=g, parts=parts)


def _crf_no_grad(x, labels, lens, ly, fl):
    import ctc_crf
    from cat_b200 import _C
    a = (_i32(labels), _i32(lens), _i32(ly))
    with torch.no_grad():
        loss = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, from_logits=fl)(x, *a)
    _, parts = _C.ctc_crf_loss_fwd_only(x, *a, LAMB, True, want_parts=True, from_logits=fl)
    return dict(loss_eval=loss, parts_eval=parts)


def _crf_costs(x, labels, lens, ly, fl, zero_infinity=True):
    """reduction='none' (with zero_infinity): the costs, the gradient of a weighted sum of them, the no_grad costs."""
    import ctc_crf
    a = (_i32(labels), _i32(lens), _i32(ly))
    crit = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, from_logits=fl, reduction="none", zero_infinity=zero_infinity)
    w = torch.tensor(_weights(x.shape[0]), device="cuda")
    x.requires_grad_(True)
    costs = crit(x, *a)
    (g,) = torch.autograd.grad((costs * w).sum(), x)
    x.requires_grad_(False)
    with torch.no_grad():
        ev = crit(x, *a)
    return dict(costs=costs, grad_costs=g, costs_eval=ev)


def _crf_native(x, labels, lens, ly, fl):
    """_C.ctc_crf_loss_fwd and _C.ctc_crf_loss_fwd_only with parts: the calls the host paths (slices, checkpoints) make."""
    from cat_b200 import _C
    a = (_i32(labels), _i32(lens), _i32(ly))
    loss, grad, parts = _C.ctc_crf_loss_fwd(x, *a, LAMB, True, want_parts=True, from_logits=fl)
    _, parts_ev = _C.ctc_crf_loss_fwd_only(x, *a, LAMB, True, want_parts=True, from_logits=fl)
    return dict(loss=loss, grad=grad, parts=parts, parts_eval=parts_ev)


def _warp(x, labels, lens, ly):
    import ctc_crf
    a = (_i32(labels), _i32(lens), _i32(ly))
    x.requires_grad_(True)
    loss = ctc_crf.WARP_CTC_LOSS()(x, *a)
    (g,) = torch.autograd.grad(loss, x)
    crit = ctc_crf.WARP_CTC_LOSS(reduction="none", zero_infinity=True)
    costs = crit(x, *a)
    (gc,) = torch.autograd.grad(costs.sum(), x)
    x.requires_grad_(False)
    with torch.no_grad():
        ev = ctc_crf.WARP_CTC_LOSS()(x, *a)
    return dict(ctc_loss=loss, grad_ctc=g, ctc_costs=costs, grad_ctc_costs=gc, ctc_loss_eval=ev)


def _align(x, labels, lens, ly):
    import ctc_crf
    align, score = ctc_crf.ctc_align(x, _i32(labels), _i32(lens), _i32(ly))
    return dict(align=align, score=score)


def _gpu_den(x, lens, sentinel=1234.5):
    """_C.gpu_den (fp32, reference signature) with grad_net pre-zeroed inside a sentinel-filled buffer: the sentinels must
    survive."""
    from cat_b200 import _C
    N = x.shape[0]
    gbuf = torch.full((x.numel() + 2 * GUARD,), sentinel, device="cuda")
    grad = gbuf[GUARD:GUARD + x.numel()].view(x.shape)
    grad.zero_()
    ca, cb = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    _C.gpu_den(x, grad, _i32(lens).cuda(), ca, cb)
    torch.cuda.synchronize()
    assert bool((gbuf[:GUARD] == sentinel).all()) and bool((gbuf[-GUARD:] == sentinel).all())
    return dict(den_logz_alpha=ca, den_logz_beta=cb, grad_den=grad)


def _check_padding(run, y, lens, dtype):
    """`run(x)` on the clean guarded batch and on its NaN / +inf / -inf padded copies.  Returns the clean outputs."""
    clean = _np(run(_guarded(y)), dtype)
    _padding_rows_zero(clean, lens, "clean")
    for value in POISONS:
        got = _np(run(_guarded(_poisoned(y, lens, value))), dtype)
        _padding_rows_zero(got, lens, value)
        _same(clean, got, value)
    return clean


def _padding_rows_zero(out, lens, what):
    """Every gradient row at t >= lx[n] of one run is exactly zero."""
    for k, v in out.items():
        if k.startswith("grad"):
            assert not v[_past(lens, v.shape[1], "cpu").numpy()].any(), (what, k)


# ---------------------------------------------------------------------------------------------------------------------
# a. padding is never read
# ---------------------------------------------------------------------------------------------------------------------
def _ragged_batch(layout, V, seed=17, N=9):
    """Lengths 0, 1 and the longest in a ragged batch.  'full': the longest utterances fill all T frames, the last one
    included, so a read past its last frame leaves the tensor; 'tail': T = max(lx) + 5, the padding a length-sorted
    batch carries past its longest utterance."""
    from oracle import oracle
    lens = np.array([24, 0, 13, 1, 20, 7, 24, 16, 24][:N], np.int32)
    T = 24 if layout == "full" else 29
    if layout == "tail":
        lens[-1] = 22
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=seed, lens=lens)
    return y, labels, lens, ly


def _without_empty(y, labels, lens, ly):
    """The batch without its length-0 utterances (log p = logZ = -inf there, so they make a batch loss NaN)."""
    keep = lens > 0
    off = np.concatenate([[0], np.cumsum(ly)])
    lab = np.concatenate([labels[off[n]:off[n + 1]] for n in np.flatnonzero(keep)]).astype(np.int32)
    return y[keep], lab, lens[keep], ly[keep]


def _raw(y, seed):
    """Unnormalised logits: log-probs shifted by a per-frame constant."""
    return (y + 3.0 * np.random.default_rng(seed).standard_normal(y.shape[:2] + (1,)) + 5.0).astype(np.float32)


def _crf_vs_oracle(g, clean, y_used, labels, lens, ly, fl, dtype):
    """The clean outputs of _crf_autograd / _crf_native against the oracle, utterances of finite cost only."""
    from oracle import oracle
    fn = oracle.ctc_crf_from_logits if fl else oracle.ctc_crf
    _, ograd, op = fn(g, y_used, labels, lens, ly, LAMB, size_average=True)
    N = len(lens)
    ok = np.isfinite(op["logz_alpha"]) & np.isfinite(op["logp_ctc"])
    assert ok.all()
    np.testing.assert_allclose(clean["parts"][:N][ok], op["logz_alpha"][ok], rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(clean["parts"][N:][ok], op["logp_ctc"][ok], rtol=LOSS_RTOL, atol=1e-4)
    ref = ograd[ok]
    assert np.all(np.abs(clean["grad"][ok] - ref) <= GRAD_ATOL + 0.5 * clean["_eps"] * np.abs(ref))


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("layout", ["full", "tail"])
def test_padding_never_read_fused_entries(tmp_graphs, layout, dtype):
    """CTC_CRF_LOSS on log-probs and on raw logits: reduction='none' with zero_infinity and ctc_align on the whole batch;
    the scalar losses (autograd, no_grad, WARP_CTC_LOSS with and without grad) on the batch without its length-0 utterance,
    so that the scalars compared are finite."""
    path, g, V = tmp_graphs["tlm_mid"]
    dt = DTYPES[dtype]
    y, labels, lens, ly = _ragged_batch(layout, V)
    ye, labe, lense, lye = _without_empty(y, labels, lens, ly)
    ctx = _ctx(path)
    for fl in (False, True):
        yt = torch.tensor(_raw(y, 3) if fl else y, device="cuda").to(dt)
        yte = torch.tensor(_raw(y, 3)[lens > 0] if fl else ye, device="cuda").to(dt)

        def run_all(x):
            out = _crf_costs(x, labels, lens, ly, fl)
            if not fl:
                out.update(_align(x, labels, lens, ly))
            return out

        def run_scalars(x):
            out = _crf_autograd(x, labe, lense, lye, fl)
            out.update(_crf_no_grad(x, labe, lense, lye, fl))
            if not fl:
                out.update(_warp(x, labe, lense, lye))
            return out

        clean = _check_padding(run_all, yt, lens, dt)
        assert np.isfinite(clean["costs"]).all()
        clean = _check_padding(run_scalars, yte, lense, dt)
        for k in ("loss", "loss_eval", "ctc_loss", "ctc_loss_eval"):
            assert k not in clean or np.isfinite(clean[k]).all(), k
        _crf_vs_oracle(g, clean, yte.float().cpu().numpy(), labe, lense, lye, fl, dt)
    del ctx


@pytest.mark.parametrize("path_kind", ["ckpt", "slices"])
def test_padding_never_read_host_paths(tmp_graphs, monkeypatch, path_kind):
    """Checkpointed alpha (every 3 frames) and a batch cut into slices of 4 utterances, each walking its own max(lx)."""
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    if path_kind == "ckpt":
        monkeypatch.setattr(_C, "_ckpt_k_override", 3)
    else:
        monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 4)
    y, labels, lens, ly = _ragged_batch("tail", V, seed=23)
    ye, labe, lense, lye = _without_empty(y, labels, lens, ly)
    ctx = _ctx(path)
    for fl in (False, True):
        yt = torch.tensor(_raw(y, 4) if fl else y, device="cuda")
        yte = torch.tensor(_raw(y, 4)[lens > 0] if fl else ye, device="cuda")
        _check_padding(lambda x: _crf_costs(x, labels, lens, ly, fl), yt, lens, torch.float32)
        clean = _check_padding(lambda x: _crf_native(x, labe, lense, lye, fl), yte, lense, torch.float32)
        assert np.isfinite(clean["loss"]).all()
        _crf_vs_oracle(g, clean, yte.cpu().numpy(), labe, lense, lye, fl, torch.float32)
    del ctx


def _den_case(g, path, N, V, T=20, seed=31, fused=True):
    """gpu_den (sentinel-guarded gradient) and, if `fused`, the fused loss, on a ragged batch of N with padding poisoned;
    the clean den against oracle.den."""
    from oracle import oracle
    from cat_b200 import _C
    lens = np.random.default_rng(seed).integers(2, T + 1, size=N).astype(np.int32)
    lens[0], lens[1], lens[N // 2], lens[N - 1] = T - 3, 0, 1, T
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=seed, lens=lens)
    yt = torch.tensor(y, device="cuda")
    clean = _check_padding(lambda x: _gpu_den(x, lens), yt, lens, torch.float32)
    sub = np.array(sorted({0, 1, N // 2, N - 1, 2}))
    la, lb, gd = oracle.den(g, y[sub], lens[sub], fast=True)
    fin = np.isfinite(la)
    np.testing.assert_allclose(clean["den_logz_alpha"][sub][fin], la[fin], rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(clean["den_logz_beta"][sub][fin], lb[fin], rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(clean["grad_den"][sub] - gd).max() < GRAD_ATOL
    if fused:
        ye, labe, lense, lye = _without_empty(y, labels, lens, ly)
        clean = _check_padding(lambda x: _crf_native(x, labe, lense, lye, False), torch.tensor(ye, device="cuda"), lense,
                               torch.float32)
        assert np.isfinite(clean["loss"]).all()


@pytest.mark.parametrize("tier", ["hub_parts", "arcs_in_global", "no_tma", "small_batch", "n130"])
def test_padding_never_read_den_tiers(tmp_graphs, monkeypatch, tier):
    """The den launches the Init-time hooks reach: hub rows summed in parts (CCB_HUB_IN_ARCS / CCB_PART_ARCS), arc tiles
    from global memory (CCB_ARCS_IN_GLOBAL), rows loaded without TMA (CCB_NO_TMA), the small-batch kernels (N <= 16) and
    130 utterances in one call (four per lane forwards)."""
    from cat_b200 import _C
    env = {"hub_parts": {"CCB_HUB_IN_ARCS": "10", "CCB_PART_ARCS": "7"}, "arcs_in_global": {"CCB_ARCS_IN_GLOBAL": "1"},
           "no_tma": {"CCB_NO_TMA": "1"}}.get(tier, {})
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    if tier == "n130":
        monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 512)
    _den_case(g, path, 130 if tier == "n130" else 12 if tier == "small_batch" else 40, V)
    del ctx


def test_padding_never_read_streamed_backward(monkeypatch, tmp_path):
    """The 1.02 M-arc benchmark graph on a 4-CTA plan at N = 12: the backward pass streams its arcs with TMA row staging
    (tests/test_gpu_grids.py pins the tier)."""
    from cat_b200 import fst
    from test_gpu_grids import TIER_STREAMED, _Plan
    g = fst.make_synthetic_den(20000, 24, 218, seed=7)
    path = str(tmp_path / "headline.fst")
    fst.write_fst(path, g)
    plan = _Plan(path, 4)
    try:
        assert plan.launch(12, True)["tier"] == TIER_STREAMED
    finally:
        plan.close()
    monkeypatch.setenv("CCB_DEN_CTAS", "4")
    ctx = _ctx(path)
    _den_case(g, path, 12, 218, T=16)
    del ctx


def test_padding_never_read_gpu_ctc():
    """_C.gpu_ctc in its (T,N,V) layout: padding frames t >= lx[n] of each utterance interleave with the others' valid
    frames.  Costs and the pre-zeroed gradient (inside a sentinel buffer) against the clean run and oracle.ctc."""
    from oracle import oracle
    from cat_b200 import _C
    N, T, V = 6, 30, 23
    lens = np.array([30, 0, 1, 17, 25, 30], np.int32)
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=41, lens=lens)
    labels[0] = labels[1]                       # a repeat
    yt = torch.tensor(y, device="cuda").transpose(0, 1).contiguous()      # (T, N, V)

    def run(x):
        gbuf = torch.full((x.numel() + 2 * GUARD,), 77.0, device="cuda")
        grads = gbuf[GUARD:GUARD + x.numel()].view(x.shape)
        grads.zero_()
        costs = torch.zeros(N)
        _C.gpu_ctc(x, grads, _i32(labels), _i32(ly), _i32(lens), N, costs, 0)
        torch.cuda.synchronize()
        assert bool((gbuf[:GUARD] == 77.0).all()) and bool((gbuf[-GUARD:] == 77.0).all())
        return dict(logp=costs, grad=grads.transpose(0, 1))

    def poison(value):
        p = yt.clone()
        p[_past(lens, T).transpose(0, 1)] = value
        return p

    clean = _np(run(_guarded(yt)), torch.float32)
    for value in POISONS:
        _same(clean, _np(run(_guarded(poison(value))), torch.float32), value)
    assert not clean["grad"][_past(lens, T, "cpu").numpy()].any()
    lp, gc = oracle.ctc(y, labels, ly, lens)
    assert np.array_equal(np.isfinite(clean["logp"]), np.isfinite(lp))
    fin = np.isfinite(lp)
    np.testing.assert_allclose(clean["logp"][fin], lp[fin], rtol=LOSS_RTOL)
    assert np.abs(clean["grad"] - gc).max() < GRAD_ATOL


# ---------------------------------------------------------------------------------------------------------------------
# b. -inf emissions against the oracle
# ---------------------------------------------------------------------------------------------------------------------
MASK_V = 48           # logits wider than tlm_mid's 40 den labels
GOOD, KILLED, DEN_DEAD, DEAD_FRAME = (0, 1, 2, 3, 6), 4, 5, 7


def _masked_batch(seed=53):
    """Eight utterances over V = 48 classes, of which tlm_mid's den graph uses the first 40:
      0 nothing masked                          4 a frame keeps only tokens off the transcript: log p = -inf, cost +inf
      1 every token off the transcript masked   5 a frame keeps only token 44 (in the transcript, not in the den graph):
      2 blank masked at every third frame         logZ = -inf, log p finite, cost -inf
      3 a label masked at frames where other    6 length 1, blank-only transcript, tokens 20.. masked
        alignments remain                       7 one valid frame entirely -inf: cost not finite (NaN)
    Returns (raw scores z, mask, labels, lens, ly)."""
    rng = np.random.default_rng(seed)
    N, T, V = 8, 30, MASK_V
    lens = np.array([30, 26, 30, 22, 30, 28, 1, 25], np.int32)
    ly = np.array([5, 4, 6, 5, 4, 5, 0, 4], np.int32)
    labs = [list(rng.integers(1, 40, size=int(n))) for n in ly]
    labs[5][2] = 44
    mask = np.zeros((N, T, V), bool)
    mask[1, :, [k for k in range(1, V) if k not in labs[1]]] = True
    mask[2, 1::3, 0] = True
    mask[3, 1:4, labs[3][0]] = True           # the first label can still come at frame 0 or from frame 4 on
    mask[3, 15:19, labs[3][-1]] = True        # the last label anywhere in frames 4..21 but these
    mask[4, 10, [0] + labs[4]] = True
    mask[5, 12, [k for k in range(V) if k != 44]] = True
    mask[6, :, 20:] = True
    mask[7, 5, :] = True
    z = 3.0 * rng.standard_normal((N, T, V))
    return z, mask, np.concatenate(labs).astype(np.int32), lens, ly


def _masked_inputs(fl, dtype):
    """Raw logits z.masked_fill(mask, -inf) (fl) or log_softmax of them, in `dtype` on the device, and the fp32 values
    the kernels read."""
    z, mask, labels, lens, ly = _masked_batch()
    zt = torch.tensor(z).masked_fill(torch.tensor(mask), -math.inf)
    if fl:
        x = zt + 2.0
    else:
        x = zt.log_softmax(-1)
        x[torch.tensor(mask.all(-1))] = -math.inf      # log_softmax of an all -inf row is NaN; as log-probs it is -inf
    x = x.float().cuda().to(dtype)
    return x, x.float().cpu().numpy(), labels, lens, ly


def _oracle_costs(g, y_used, labels, lens, ly, fl):
    from oracle import oracle
    fn = oracle.ctc_crf_from_logits if fl else oracle.ctc_crf
    _, ograd, op = fn(g, y_used, labels, lens, ly, LAMB, size_average=False)
    with np.errstate(invalid="ignore"):
        return op["logz_alpha"] - (1.0 + LAMB) * op["logp_ctc"], ograd, op


def _check_costs(costs, grad, ocost, ograd, w, dtype, zero_infinity):
    good = list(GOOD)
    np.testing.assert_allclose(costs[good], ocost[good], rtol=LOSS_RTOL, atol=LOSS_RTOL)
    ref = w[good, None, None] * ograd[good]
    assert np.all(np.abs(grad[good] - ref) <= GRAD_ATOL + 0.5 * float(torch.finfo(dtype).eps) * np.abs(ref))
    bad = [KILLED, DEN_DEAD, DEAD_FRAME]
    if zero_infinity:
        assert (costs[bad] == 0).all(), costs
        assert np.isfinite(grad).all() and not grad[bad].any()
    else:
        assert costs[KILLED] == np.inf and costs[DEN_DEAD] == -np.inf and not np.isfinite(costs[DEAD_FRAME]), costs


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("fl", [False, True], ids=["logprobs", "logits"])
def test_neg_inf_emissions_vs_oracle(tmp_graphs, monkeypatch, fl, dtype):
    """The fused loss (costs, weighted gradient, zero_infinity, no_grad, checkpointed alpha, the scalar) on masked inputs
    against the oracle.  The oracle's costs have the expected signs: +inf, -inf and NaN for utterances 4, 5, 7."""
    import ctc_crf
    from cat_b200 import _C
    path, g, _ = tmp_graphs["tlm_mid"]
    dt = DTYPES[dtype]
    x, y_used, labels, lens, ly = _masked_inputs(fl, dt)
    ocost, ograd, op = _oracle_costs(g, y_used, labels, lens, ly, fl)
    assert np.isfinite(ocost[list(GOOD)]).all()
    assert ocost[KILLED] == np.inf and ocost[DEN_DEAD] == -np.inf and np.isnan(ocost[DEAD_FRAME])
    assert (np.isinf(y_used[list(GOOD)][:, :, :]).sum(-1) > 0).any()
    N = len(lens)
    w_np = _weights(N).astype(np.float64)
    a = (_i32(labels), _i32(lens), _i32(ly))
    ctx = _ctx(path)
    for zi in (False, True):
        out = _np(_crf_costs(x, labels, lens, ly, fl, zero_infinity=zi), dt)
        _check_costs(out["costs"], out["grad_costs"], ocost, ograd, w_np, dt, zi)
        same = np.isfinite(out["costs"])
        np.testing.assert_allclose(out["costs_eval"][same], out["costs"][same], rtol=SAME_TOL)
        assert np.array_equal(np.isnan(out["costs_eval"]), np.isnan(out["costs"]))
        # checkpointed alpha, every 4 frames
        monkeypatch.setattr(_C, "_ckpt_k_override", 4)
        ck, ckg, ckp = _C.ctc_crf_loss_fwd(x, *a, LAMB, True, want_parts=True, from_logits=fl, reduction="none",
                                           zero_infinity=zi)
        monkeypatch.setattr(_C, "_ckpt_k_override", None)
        _check_costs(ck.cpu().numpy(), ckg.cpu().numpy(), ocost, ograd, np.ones(N), torch.float32, zi)
        ckp = ckp.cpu().numpy()
        assert ckp[DEN_DEAD] == -np.inf and ckp[N + KILLED] == -np.inf
        np.testing.assert_allclose(ckp[list(GOOD)], op["logz_alpha"][list(GOOD)], rtol=LOSS_RTOL, atol=1e-4)
    # the scalar with zero_infinity: the mean of the finite costs over all N
    x.requires_grad_(True)
    loss = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, from_logits=fl, zero_infinity=True)(x, *a)
    (gs,) = torch.autograd.grad(loss, x)
    x.requires_grad_(False)
    assert abs(float(loss) - ocost[list(GOOD)].sum() / N) <= LOSS_RTOL * max(1.0, abs(ocost[list(GOOD)].sum() / N))
    gs = gs.float().cpu().numpy()
    assert np.isfinite(gs).all() and not gs[[KILLED, DEN_DEAD, DEAD_FRAME]].any()
    del ctx


def test_neg_inf_emissions_warp_ctc(tmp_graphs):
    """WARP_CTC_LOSS on the masked log-probs: costs against oracle.ctc and torch's fp64 ctc_loss forward, the gradient
    against the oracle's occupancies, zero_infinity masking the two utterances of log p = -inf, no_grad equal."""
    import ctc_crf
    from oracle import oracle
    x, y, labels, lens, ly = _masked_inputs(False, torch.float32)
    lp, gc = oracle.ctc(y, labels, ly, lens)
    nll = torch.nn.functional.ctc_loss(torch.tensor(y, dtype=torch.float64).transpose(0, 1), torch.tensor(labels).long(),
                                       torch.tensor(lens).long(), torch.tensor(ly).long(), reduction="none").numpy()
    fin = np.isfinite(lp)
    assert list(np.flatnonzero(~fin)) == [KILLED, DEAD_FRAME] and np.isinf(nll[~fin]).all()
    z, mask, _, _, _ = _masked_batch()         # utterance 3's masked labels carry occupancy without the mask
    off = np.concatenate([[0], np.cumsum(ly)])
    y3 = torch.tensor(z[3:4]).log_softmax(-1).float().numpy()
    _, g3 = oracle.ctc(y3, labels[off[3]:off[4]], ly[3:4], lens[3:4])
    assert (g3[0][mask[3]] > 0).all()
    np.testing.assert_allclose(-lp[fin], nll[fin], rtol=1e-9)
    a = (_i32(labels), _i32(lens), _i32(ly))
    for zi in (False, True):
        crit = ctc_crf.WARP_CTC_LOSS(reduction="none", zero_infinity=zi)
        x.requires_grad_(True)
        costs = crit(x, *a)
        (g,) = torch.autograd.grad(costs[torch.tensor(fin, device="cuda")].sum(), x)
        x.requires_grad_(False)
        costs, g = costs.detach().cpu().numpy(), g.cpu().numpy()
        np.testing.assert_allclose(costs[fin], nll[fin], rtol=LOSS_RTOL)
        assert np.abs(g[fin] + gc[fin]).max() < GRAD_ATOL and np.isfinite(g).all()
        assert (costs[~fin] == 0).all() if zi else (costs[~fin] == np.inf).all()
        with torch.no_grad():
            ev = crit(x, *a).cpu().numpy()
        assert np.array_equal(ev, costs)


@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_neg_inf_emissions_align(dtype):
    """ctc_align on the masked log-probs against the vectorised fp64 Viterbi: the score of the best finite path, a row
    that collapses to the labels, and for an utterance every path of which crosses a -inf emission a score of -inf and
    an all -1 row."""
    import ctc_crf
    from test_gpu_regimes import _viterbi_np
    x, y, labels, lens, ly = _masked_inputs(False, DTYPES[dtype])
    align, score = ctc_crf.ctc_align(_guarded(x), _i32(labels), _i32(lens), _i32(ly))
    align, score = align.cpu().numpy(), score.cpu().numpy()
    off = np.concatenate([[0], np.cumsum(ly)])
    for n in range(len(lens)):
        lab = labels[off[n]:off[n + 1]]
        yn = y[n, :lens[n]].astype(np.float64)
        ref, sc = _viterbi_np(yn, lab)
        assert (align[n, lens[n]:] == -1).all()
        if sc == -np.inf:
            assert n in (KILLED, DEAD_FRAME)
            assert score[n] == -np.inf and (align[n] == -1).all(), (n, align[n])
            continue
        assert abs(float(score[n]) - sc) <= LOSS_RTOL * max(1.0, abs(sc)), (n, score[n], sc)
        got = align[n, :lens[n]]
        assert abs(yn[np.arange(lens[n]), got].sum() - sc) <= LOSS_RTOL * max(1.0, abs(sc))
        collapsed = [int(k) for i, k in enumerate(got) if k != 0 and (i == 0 or got[i - 1] != k)]
        assert collapsed == [int(k) for k in lab], n


# ---------------------------------------------------------------------------------------------------------------------
# c. large finite raw logits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["fp32_1e4", "fp16_6e4"])
def test_large_raw_logits_vs_oracle(tmp_graphs, case):
    """Raw logits far from 0: fp32 offset by 1e4; fp16 at +-59 008 and 32 or 64 below it (fp16's ulp there is 32), so
    that a frame's logits stay within the den's range of about 140 nats below the frame's mass (INTEGRATION.md section
    1, 'range'; a wider spread flushes paths to zero by design).  The den and numerator shift each
    frame by its max, so their occupancies are exact; what the magnitude costs is the frame log-normaliser lz, which the
    kernels round to fp32 per frame: |error| <= ulp_fp32(|lz|) / 2 (2^-11 at 1e4, 2^-9 at 6e4) plus logf's few ulp of a
    number <= log V.  Summed over an utterance's Tn frames that moves logZ and log p by up to Tn of it each, the cost
    (= logZ_raw - (1+lamb) log p_raw + lamb * sum lz) by lamb times that, and a gradient entry by
    softmax_k * |sum_j g_j| * that per frame (under 1e-3).  The tolerances add this bound to the suite's."""
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    N, T = 6, 30
    lens = np.array([30, 24, 17, 30, 9, 1], np.int32)
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=59, lens=lens)
    rng = np.random.default_rng(59)
    if case == "fp32_1e4":
        zt = torch.tensor(y + 1e4 + rng.standard_normal((N, T, 1)).astype(np.float32), device="cuda")
    else:
        sign = np.where(rng.random((N, T, 1)) < 0.5, -1.0, 1.0)
        zt = torch.tensor(sign * 59008.0 - 32.0 * rng.integers(0, 3, size=(N, T, V)), device="cuda").half()
    z_used = zt.float().cpu().numpy()
    _, ograd, op = oracle.ctc_crf_from_logits(g, z_used, labels, lens, ly, LAMB, size_average=False)
    ocost = op["logz_alpha"] - (1.0 + LAMB) * op["logp_ctc"]
    assert np.isfinite(ocost).all()
    if case == "fp16_6e4":
        assert np.abs(z_used).max() > 5.9e4 and np.ptp(z_used, axis=-1).max() <= 64.0
    zmax = np.abs(z_used).max() + math.log(V)
    lz_err = float(np.spacing(np.float32(zmax))) / 2 + 1e-6
    bound = lens * lz_err
    ctx = _ctx(path)
    crit = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, from_logits=True, reduction="none")
    x = zt.clone().requires_grad_(True)
    costs = crit(x, _i32(labels), _i32(lens), _i32(ly))
    w = torch.linspace(0.5, 1.5, N, device="cuda")
    (gz,) = torch.autograd.grad((costs * w).sum(), x)
    costs, gz = costs.detach().cpu().numpy().astype(np.float64), gz.float().cpu().numpy()
    assert np.all(np.abs(costs - ocost) <= LOSS_RTOL * np.maximum(1.0, np.abs(ocost)) + LAMB * bound), (costs, ocost)
    ref = w.cpu().numpy()[:, None, None] * ograd
    assert np.all(np.abs(gz - ref) <= GRAD_ATOL + 0.5 * float(torch.finfo(zt.dtype).eps) * np.abs(ref))
    _, _, parts = _C.ctc_crf_loss_fwd(zt, _i32(labels), _i32(lens), _i32(ly), LAMB, False, want_parts=True,
                                      from_logits=True)
    parts = parts.cpu().numpy().astype(np.float64)
    for got, ref_p in ((parts[:N], op["logz_alpha"]), (parts[N:], op["logp_ctc"])):
        assert np.all(np.abs(got - ref_p) <= LOSS_RTOL * np.maximum(1.0, np.abs(ref_p)) + bound), (got, ref_p)
    del ctx
