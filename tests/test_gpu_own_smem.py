"""GPU: the den kernels with each warp's own rows kept on chip (DenLaunch::own_smem) against the same calls with them re-read
from L2 (the Init-time hook CCB_OWN_IN_L2=1), and against the fp64 oracle.

Each case runs twice, in fresh contexts, with and without the hook, and checks through ccb_plan_launch_own that the first
run keeps the own rows in shared memory and the second does not.  The two runs read the same bits from a different place,
so they agree to the bound two clean runs of the same call keep (tests/test_gpu_input_values.py: the den's atomic sums
land in no fixed order): 1e-6 relative for losses and costs, 1e-6 absolute plus 32 fp32 ulps for gradients.  The on-chip
run also matches the oracle at the suite's tolerances: loss 1e-4 relative, gradients 1e-3 absolute.
"""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3
SAME_TOL = 1e-6
SAME_ULPS = 32
LAMB = 0.1
OWN_IN_L2 = 8   # ccb_plan_launch hooks bit


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32)


def _own_smem(path, N, n_ctas=None, hooks=0):
    """(forward, backward) of ccb_plan_launch_own for N utterances on this device's plan (or one cut for n_ctas CTAs)."""
    from cat_b200 import _lib
    L = _lib.lib()
    props = torch.cuda.get_device_properties(0)
    h = L.ccb_plan_create(path.encode(), n_ctas or props.multi_processor_count, 16)
    assert h, _lib.last_error()
    try:
        out = []
        for backward in (0, 1):
            o = (C.c_long * 2)()
            assert L.ccb_plan_launch_own(h, N, backward, props.shared_memory_per_block_optin, hooks, o) == 0, _lib.last_error()
            out.append(bool(o[0]))
        return tuple(out)
    finally:
        L.ccb_plan_destroy(h)


def _np(out):
    return {k: v.detach().float().cpu().numpy().astype(np.float64) for k, v in out.items()}


def _both(monkeypatch, path, run, widths, n_ctas=None, own=(True, True)):
    """run() in a fresh context with the own rows on chip, then in one with CCB_OWN_IN_L2=1; the outputs of both.  `widths`:
    the batch widths of the den calls run() makes, whose launches must keep the own rows on chip (`own`: per pass)."""
    import ctc_crf
    if n_ctas is not None:
        if n_ctas > torch.cuda.get_device_properties(0).multi_processor_count:
            pytest.skip(f"{n_ctas} CTAs need at least as many SMs")
        monkeypatch.setenv("CCB_DEN_CTAS", str(n_ctas))
    res = []
    for in_l2 in (False, True):
        for N in widths:
            want = (False, False) if in_l2 else own
            assert _own_smem(path, N, n_ctas, OWN_IN_L2 if in_l2 else 0) == want, (N, in_l2)
        if in_l2:
            monkeypatch.setenv("CCB_OWN_IN_L2", "1")
        else:
            monkeypatch.delenv("CCB_OWN_IN_L2", raising=False)
        ctx = ctc_crf.CRFContext(path, gpus=0)
        try:
            res.append(_np(run()))
        finally:
            del ctx
    monkeypatch.delenv("CCB_OWN_IN_L2", raising=False)
    on_chip, in_l2 = res
    for k, a in on_chip.items():
        b = in_l2[k]
        fa = np.isfinite(a)
        assert np.array_equal(fa, np.isfinite(b)), k
        assert np.array_equal(a[~fa], b[~fa]) or np.array_equal(np.isnan(a[~fa]), np.isnan(b[~fa])), k
        if k.startswith("grad"):
            tol = SAME_TOL + SAME_ULPS * float(np.finfo(np.float32).eps) * np.abs(a[fa])
        else:
            tol = SAME_TOL * np.maximum(1.0, np.abs(a[fa]))
        assert np.all(np.abs(a[fa] - b[fa]) <= tol), (k, np.abs(a[fa] - b[fa]).max())
    return on_chip


def _ragged(N, T, seed, zero):
    """Lengths in [2, T]: T first, then 0 (or 2) and 1 at fixed places, the last one T - 1."""
    lens = np.random.default_rng(seed).integers(2, T + 1, size=N).astype(np.int32)
    lens[0], lens[1], lens[N // 2], lens[N - 1] = T, 0 if zero else 2, 1, T - 1
    return lens


def _batch(V, N, T, seed, zero=False):
    from oracle import oracle
    return oracle.synth_batch(N, T, V, seed=seed, lens=_ragged(N, T, seed, zero))


def _loss_run(y, labels, lens, ly, dtype=torch.float32):
    import ctc_crf
    x = torch.tensor(y, device="cuda", dtype=dtype).requires_grad_(True)
    loss = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, size_average=False)(x, _i32(labels), _i32(lens), _i32(ly))
    (g,) = torch.autograd.grad(loss, x)
    return dict(loss=loss, grad=g)


def _loss_vs_oracle(g, out, y, labels, lens, ly):
    from oracle import oracle
    oloss, ograd, _ = oracle.ctc_crf(g, y, labels, lens, ly, LAMB, size_average=False, fast=True)
    assert abs(out["loss"].item() - oloss) <= LOSS_RTOL * max(1.0, abs(oloss)), (out["loss"].item(), oloss)
    assert np.abs(out["grad"] - ograd).max() < GRAD_ATOL


# ---------------------------------------------------------------------------------------------------------------------
# the fused loss and its entries on tlm_mid
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [33, 64, 100, 130])
def test_fused_loss(tmp_graphs, monkeypatch, N):
    """CTC_CRF_LOSS through autograd, lengths 1, 2, T - 1 and T among them: two and four utterances per lane forwards,
    two lane groups backwards at N = 100 and 130."""
    path, g, V = tmp_graphs["tlm_mid"]
    T = 30
    y, labels, lens, ly = _batch(V, N, T, seed=N)
    out = _both(monkeypatch, path, lambda: _loss_run(y, labels, lens, ly), [N])
    _loss_vs_oracle(g, out, y, labels, lens, ly)
    assert not out["grad"][np.arange(T)[None, :] >= lens[:, None]].any()


def test_entries(tmp_graphs, monkeypatch):
    """N = 40 with lengths 0, 1 and T, and the 39 utterances of nonzero length: forward-only under torch.no_grad (alpha on
    the frame ring), checkpointed alpha every 4 frames (several segment launches in each pass), the batch sliced into calls
    of 20 and 19 utterances (slices of 16 or fewer run the small-batch kernels, which keep nothing on chip), fp16 raw
    logits, reduction='none' with zero_infinity (the length-0 utterance's cost is 0) and _C.gpu_den."""
    import ctc_crf
    from cat_b200 import _C
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_mid"]
    N, T = 40, 28
    y, labels, lens, ly = _batch(V, N, T, seed=5, zero=True)
    keep = lens > 0
    off = np.concatenate([[0], np.cumsum(ly)])
    lab_k = np.concatenate([labels[off[n]:off[n + 1]] for n in np.flatnonzero(keep)]).astype(np.int32)
    yk, lensk, lyk = y[keep], lens[keep], ly[keep]
    zk = (yk + 3.0 * np.random.default_rng(1).standard_normal((lensk.size, T, 1)) + 5.0).astype(np.float32)
    w = np.linspace(-1.0, 0.9, N).astype(np.float32)

    def run():
        a = (_i32(labels), _i32(lens), _i32(ly))
        ak = (_i32(lab_k), _i32(lensk), _i32(lyk))
        out = {}
        xk = torch.tensor(yk, device="cuda")
        with torch.no_grad():
            out["loss_eval"] = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, size_average=False)(xk, *ak)
        monkeypatch.setattr(_C, "_ckpt_k_override", 4)
        try:
            out["loss_ckpt"], out["grad_ckpt"], _ = _C.ctc_crf_loss_fwd(xk, *ak, LAMB, False, want_parts=True)
        finally:
            monkeypatch.setattr(_C, "_ckpt_k_override", None)
        monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 20)
        try:
            r = _loss_run(yk, lab_k, lensk, lyk)
        finally:
            monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 512)
        out["loss_sliced"], out["grad_sliced"] = r["loss"], r["grad"]
        zt = torch.tensor(zk, device="cuda").half()
        out["loss_fp16"], gz, _ = _C.ctc_crf_loss_fwd(zt, *ak, LAMB, False, want_parts=True, from_logits=True)
        out["grad_fp16"] = gz.float()
        x = torch.tensor(y, device="cuda").requires_grad_(True)
        costs = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, reduction="none", zero_infinity=True)(x, *a)
        (out["grad_costs"],) = torch.autograd.grad((costs * torch.tensor(w, device="cuda")).sum(), x)
        out["costs"] = costs
        xd = torch.tensor(y, device="cuda")
        grad = torch.zeros_like(xd)
        ca, cb = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
        _C.gpu_den(xd, grad, _i32(lens).cuda(), ca, cb)
        out.update(den_logz_alpha=ca, den_logz_beta=cb, grad_den=grad)
        return out

    out = _both(monkeypatch, path, run, [N, lensk.size, 20, lensk.size - 20])
    oloss, ograd, oparts = oracle.ctc_crf(g, yk, lab_k, lensk, lyk, LAMB, size_average=False, fast=True)
    for k in ("loss_eval", "loss_ckpt", "loss_sliced"):
        assert abs(out[k].item() - oloss) <= LOSS_RTOL * max(1.0, abs(oloss)), (k, out[k].item(), oloss)
    for k in ("grad_ckpt", "grad_sliced"):
        assert np.abs(out[k] - ograd).max() < GRAD_ATOL, k
    zl, zg, _ = oracle.ctc_crf_from_logits(g, torch.tensor(zk).half().float().numpy(), lab_k, lensk, lyk, LAMB,
                                           size_average=False)
    assert abs(out["loss_fp16"].item() - zl) <= LOSS_RTOL * max(1.0, abs(zl))
    assert np.abs(out["grad_fp16"] - zg).max() < GRAD_ATOL
    ocost = oparts["logz_alpha"] - (1.0 + LAMB) * oparts["logp_ctc"]
    np.testing.assert_allclose(out["costs"][keep], ocost, rtol=LOSS_RTOL, atol=1e-4)
    assert not out["costs"][~keep].any() and not out["grad_costs"][~keep].any()
    assert np.abs(out["grad_costs"][keep] - w[keep][:, None, None] * ograd).max() < GRAD_ATOL
    la, lb, gd = oracle.den(g, y[keep], lens[keep], fast=True)
    np.testing.assert_allclose(out["den_logz_alpha"][keep], la, rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(out["den_logz_beta"][keep], lb, rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(out["grad_den"][keep] - gd).max() < GRAD_ATOL


# ---------------------------------------------------------------------------------------------------------------------
# plans the hooks change, other grids, the headline shape
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hook,own", [("CCB_NO_MERGE", False), ("CCB_NO_OWN", False), ("HUBS", False), ("CCB_NO_PAIRS", True)])
def test_plans_the_hooks_build(tmp_graphs, monkeypatch, hook, own):
    """Plans without own-row terms (unmerged pairs, the hook, hub rows summed in parts) keep nothing on chip, and
    CCB_OWN_IN_L2 changes nothing there; without pairs the own-row terms are the rows' self loops, kept on chip."""
    if hook == "HUBS":
        monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
        monkeypatch.setenv("CCB_PART_ARCS", "7")
    else:
        monkeypatch.setenv(hook, "1")
    path, g, V = tmp_graphs["tlm_mid"]
    N = 40
    y, labels, lens, ly = _batch(V, N, 20, seed=9)
    out = _both(monkeypatch, path, lambda: _loss_run(y, labels, lens, ly), [N], own=(own, own))
    _loss_vs_oracle(g, out, y, labels, lens, ly)


@pytest.mark.parametrize("n_ctas", [78, 4])
def test_other_grids(tmp_graphs, monkeypatch, n_ctas):
    """tlm_mid's plans at 78 and 4 CTAs (larger tiles than the 132-CTA plan's), N = 40 and 100 (Npad = 128: on 4 CTAs the
    tile's own rows fit up to that width)."""
    path, g, V = tmp_graphs["tlm_mid"]
    for N in (40, 100):
        y, labels, lens, ly = _batch(V, N, 20, seed=N + n_ctas)
        out = _both(monkeypatch, path, lambda: _loss_run(y, labels, lens, ly), [N], n_ctas=n_ctas)
        _loss_vs_oracle(g, out, y, labels, lens, ly)


def test_headline_shape(tmp_path_factory, monkeypatch):
    """The benchmark's 1.02 M-arc graph at N = 64, T = 1500 (bench.py's workload, its seed aside): loss and gradient on chip
    against L2, logZ from alpha and from beta equal, the occupancies of every frame summing to 1, and the first, the
    length-1 and the last utterance against the oracle over 300 frames."""
    from cat_b200 import _C, fst
    from oracle import oracle
    path = str(tmp_path_factory.mktemp("own_headline") / "den_20000_218.fst")
    g = fst.make_synthetic_den(20000, 24, 218, seed=7)
    fst.write_fst(path, g)
    N, T, V = 64, 1500, 218
    y, labels, lens, ly = _batch(V, N, T, seed=3)
    ys, lens_s = y[:, :300], np.minimum(lens, 300)

    def run():
        out = _loss_run(y, labels, lens, ly)
        xd = torch.tensor(ys, device="cuda")
        grad = torch.zeros_like(xd)
        ca, cb = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
        _C.gpu_den(xd, grad, _i32(lens_s).cuda(), ca, cb)
        out.update(den_logz_alpha=ca, den_logz_beta=cb, grad_den=grad)
        return out

    out = _both(monkeypatch, path, run, [N])
    np.testing.assert_allclose(out["den_logz_alpha"], out["den_logz_beta"], rtol=1e-5)
    rows = out["grad_den"].sum(-1)
    inside = np.arange(300)[None, :] < lens_s[:, None]
    assert np.abs(rows[inside] - 1.0).max() < 1e-4
    sub = np.array([0, N // 2, N - 1])
    la, lb, gd = oracle.den(g, ys[sub], lens_s[sub], fast=True)
    np.testing.assert_allclose(out["den_logz_alpha"][sub], la, rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(out["grad_den"][sub] - gd).max() < GRAD_ATOL
