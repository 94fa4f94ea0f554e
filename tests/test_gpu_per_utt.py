"""Per-utterance costs (`reduction='none'`) and `zero_infinity` of CTC_CRF_LOSS and WARP_CTC_LOSS on the GPU.

Costs against the fp64 oracle per utterance (1e-4 relative), the gradient of a weighted sum of the costs against the oracle's
per-utterance gradients (1e-3 absolute, plus the rounding of a 16-bit result), every host path that splits a batch, the mask
of utterances whose cost is not finite, the forward-only entries, and WARP_CTC_LOSS against torch's fp64 ctc_loss.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32)


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _close(a, b, rtol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.all(np.abs(a - b) <= rtol * np.maximum(1.0, np.abs(b))), (a, b)


def _grad_tol(ref, dtype):
    """1e-3, plus half an ulp of the dtype the gradient is returned in."""
    return GRAD_ATOL + 0.5 * torch.finfo(dtype).eps * np.abs(ref)


def _oracle(g, y_used, labels, lens, ly, lamb, from_logits):
    """Per-utterance costs and the unscaled per-utterance gradients of the fp64 oracle."""
    from oracle import oracle
    if from_logits:
        _, grad, parts = oracle.ctc_crf_from_logits(g, y_used, labels, lens, ly, lamb, size_average=False)
    else:
        _, grad, parts = oracle.ctc_crf(g, y_used, labels, lens, ly, lamb, size_average=False)
    return parts["logz_alpha"] - (1.0 + lamb) * parts["logp_ctc"], grad


def _inputs(N, T, V, seed, lens, dtype, from_logits):
    """(logits on the GPU in `dtype`, the fp32 values the kernels see, labels, lens, ly)."""
    from oracle import oracle
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=seed, lens=lens)
    if from_logits:
        y = y + 3.0 * np.random.default_rng(seed).standard_normal((N, T, 1)).astype(np.float32) + 5.0   # unnormalised
    yt = torch.tensor(y, device="cuda").to(dtype).contiguous()
    return yt, yt.float().cpu().numpy(), labels, lens, ly


def _costs_and_grad(crit, yt, labels, lens, ly, w):
    y = yt.clone().requires_grad_(True)
    costs = crit(y, _i32(labels), _i32(lens), _i32(ly))
    (g,) = torch.autograd.grad(costs.mul(w).sum(), y)
    return costs.detach(), g


def _check_against_oracle(g_graph, crit, yt, y_used, labels, lens, ly, lamb, from_logits, seed=0):
    N = yt.shape[0]
    w = torch.tensor(np.random.default_rng(seed).uniform(-2.0, 2.0, N).astype(np.float32), device="cuda")
    costs, grad = _costs_and_grad(crit, yt, labels, lens, ly, w)
    assert costs.shape == (N,) and costs.dtype == torch.float32 and costs.is_cuda
    assert grad.dtype == yt.dtype
    ocost, ograd = _oracle(g_graph, y_used, labels, lens, ly, lamb, from_logits)
    _close(costs.cpu().numpy(), ocost, LOSS_RTOL)
    ref = w.cpu().numpy()[:, None, None] * ograd
    assert np.all(np.abs(grad.float().cpu().numpy() - ref) <= _grad_tol(ref, yt.dtype)), \
        np.abs(grad.float().cpu().numpy() - ref).max()
    for n in range(N):
        assert not grad[n, int(lens[n]):].any()
    return costs


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("from_logits", [False, True])
@pytest.mark.parametrize("name", ["fixture", "tlm_small", "tlm_mid"])
def test_costs_and_weighted_grad_vs_oracle(tmp_graphs, fixture_fst, fixture_inputs, name, from_logits, dtype):
    """reduction='none' per utterance against the oracle; costs.sum()/N is the default reduction's loss."""
    import ctc_crf
    from cat_b200 import fst
    dt = DTYPES[dtype]
    if name == "fixture":
        fi = fixture_inputs
        path, g = fixture_fst, fst.read_fst(fixture_fst)
        yt = torch.tensor(fi["y"], device="cuda").to(dt).contiguous()
        y_used, labels, lens, ly, lamb = yt.float().cpu().numpy(), fi["labels"], fi["lx"], fi["ly"], fi["lamb"]
    else:
        path, g, V = tmp_graphs[name]
        N, T = (6, 30) if name == "tlm_small" else (9, 40)
        lamb = 0.1
        yt, y_used, labels, lens, ly = _inputs(N, T, V, 11, np.linspace(T, 4, N).astype(np.int32), dt, from_logits)
    ctx = _ctx(path)
    crit = ctc_crf.CTC_CRF_LOSS(lamb=lamb, from_logits=from_logits, reduction="none")
    costs = _check_against_oracle(g, crit, yt, y_used, labels, lens, ly, lamb, from_logits)
    N = yt.shape[0]
    mean = ctc_crf.CTC_CRF_LOSS(lamb=lamb, from_logits=from_logits)(yt.clone().requires_grad_(True), _i32(labels),
                                                                    _i32(lens), _i32(ly))
    _close(float(costs.double().sum()) / N, float(mean.item()), 1e-6)
    del ctx


@pytest.mark.parametrize("path_kind", ["slices", "ckpt", "sorted_padded"])
def test_host_paths_write_every_cost_in_place(tmp_graphs, monkeypatch, path_kind):
    """More than 64 utterances (two native calls), slices forced to checkpointed alpha, and a length-sorted batch padded
    past its longest utterance: every utterance's cost lands at its own index."""
    import ctc_crf
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    if path_kind == "slices":
        N, T = 70, 16
        lens = np.maximum(1, T - (np.arange(N) * 5) % T).astype(np.int32)
    elif path_kind == "ckpt":
        monkeypatch.setattr(_C, "_ckpt_k_override", 3)
        monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 4)
        N, T = 10, 30
        lens = np.maximum(1, T - (np.arange(N) * 7) % T).astype(np.int32)
    else:
        N, T = 12, 48
        lens = np.sort(np.random.default_rng(3).integers(1, 37, size=N))[::-1].astype(np.int32)
    for from_logits in (False, True):
        yt, y_used, labels, lens, ly = _inputs(N, T, V, 5 + N, lens, torch.float32, from_logits)
        crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits, reduction="none")
        _check_against_oracle(g, crit, yt, y_used, labels, lens, ly, 0.1, from_logits, seed=N)
    del ctx


def _bad_batch(V, seed):
    """Nine utterances; index 2 is infeasible (more labels than frames, log p = -inf, cost +inf), index 5 has length 0
    (logZ = -inf and log p = -inf on these graphs, cost NaN).  Returns the batch and the indices of the good ones."""
    from oracle import oracle
    N, T = 9, 30
    lens = np.array([30, 28, 6, 25, 20, 0, 17, 9, 30], np.int32)
    y, _, lens, ly = oracle.synth_batch(N, T, V, seed=seed, lens=lens)
    ly[2] = 9
    labels = np.random.default_rng(seed).integers(1, V, size=int(ly.sum())).astype(np.int32)
    return y, labels, lens, ly, [n for n in range(N) if n not in (2, 5)]


def _subset(labels, ly, keep):
    off = np.concatenate([[0], np.cumsum(ly)])
    return np.concatenate([labels[off[n]:off[n + 1]] for n in keep]).astype(np.int32), ly[keep]


@pytest.mark.parametrize("path_kind", ["one_call", "slices", "ckpt"])
@pytest.mark.parametrize("from_logits", [False, True])
def test_zero_infinity_masks_bad_utterances(tmp_graphs, monkeypatch, path_kind, from_logits):
    import ctc_crf
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    if path_kind == "slices":
        monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 4)
    elif path_kind == "ckpt":
        monkeypatch.setattr(_C, "_ckpt_k_override", 4)
    y, labels, lens, ly, good = _bad_batch(V, seed=61)
    yt = torch.tensor(y, device="cuda")
    N = len(lens)
    w = torch.tensor(np.random.default_rng(2).uniform(0.5, 2.0, N).astype(np.float32), device="cuda")
    crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits, reduction="none", zero_infinity=True)
    costs, grad = _costs_and_grad(crit, yt, labels, lens, ly, w)
    costs, grad = costs.cpu().numpy(), grad.cpu().numpy()
    assert costs[2] == 0.0 and costs[5] == 0.0
    assert not grad[2].any() and not grad[5].any()
    # every other utterance: the costs and gradient of the batch without the two bad ones
    sub_labels, sub_ly = _subset(labels, ly, good)
    ref = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits, reduction="none")
    rc, rg = _costs_and_grad(ref, yt[good].contiguous(), sub_labels, lens[good], sub_ly, w[good])
    _close(costs[good], rc.cpu().numpy(), 1e-6)
    assert np.abs(grad[good] - rg.cpu().numpy()).max() <= 1e-6
    # the scalar loss is finite, the divisor stays N
    for sa in (True, False):
        yg = yt.clone().requires_grad_(True)
        loss = ctc_crf.CTC_CRF_LOSS(lamb=0.1, size_average=sa, from_logits=from_logits, zero_infinity=True)(
            yg, _i32(labels), _i32(lens), _i32(ly))
        loss.backward()
        assert np.isfinite(float(loss.item()))
        _close(float(loss.item()), float(rc.double().sum()) / (N if sa else 1), 1e-6)
        gs = yg.grad.cpu().numpy()
        assert not gs[2].any() and not gs[5].any() and np.isfinite(gs).all()
    # zero_infinity=False: today's inf / NaN
    raw = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits, reduction="none")(
        yt.clone().requires_grad_(True), _i32(labels), _i32(lens), _i32(ly)).detach().cpu().numpy()
    assert raw[2] == np.inf and not np.isfinite(raw[5])
    loss = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits)(yt.clone().requires_grad_(True), _i32(labels),
                                                                   _i32(lens), _i32(ly))
    assert not np.isfinite(float(loss.item()))
    # forward only: the same masked costs
    with torch.no_grad():
        ev = crit(yt, _i32(labels), _i32(lens), _i32(ly)).cpu().numpy()
    assert ev[2] == 0.0 and ev[5] == 0.0
    _close(ev[good], costs[good], 1e-6)
    del ctx


@pytest.fixture(scope="module")
def few_finals_graph(tmp_path_factory):
    """A 40k-state den graph of which only 6 states are final: no path of 2 frames ends in one of them."""
    from cat_b200 import fst
    g = fst.make_synthetic_den(20000, 24, 218, seed=7)
    keep = np.flatnonzero(~np.isinf(g.final))[::max(1, (2 * 20000 - 1) // 6)][:6]
    fin = np.full_like(g.final, np.inf)
    fin[keep] = g.final[keep]
    g.final = fin
    path = str(tmp_path_factory.mktemp("few_finals") / "den_few_finals.fst")
    fst.write_fst(path, g)
    return path, g


@pytest.mark.parametrize("from_logits", [False, True])
def test_zero_infinity_masks_unreachable_final_state(few_finals_graph, from_logits):
    """An utterance WITH frames whose logZ is -inf while its log p is finite: the den half of the mask in the occupancy
    kernel.  Unmasked its rows hold the numerator occupancies (cost -inf); masked they are zeros and its cost 0, and the
    other utterances get what they get in a batch without it."""
    import ctc_crf
    from cat_b200 import _C
    from oracle import oracle
    path, g = few_finals_graph
    ctx = _ctx(path)
    V, lamb = 218, 0.01
    lens = np.array([40, 2, 37], np.int32)
    y, labels, lens, ly = oracle.synth_batch(3, 40, V, seed=79, lens=lens, scale=8.0)
    assert ly[1] == 0                                   # all-blank: log p finite
    yt = torch.tensor(y, device="cuda")
    if from_logits:
        yt = yt + 2.0
    lab, lx, lyt = _i32(labels), _i32(lens), _i32(ly)
    _, _, parts = _C.ctc_crf_loss_fwd(yt, lab, lx, lyt, lamb, True, want_parts=True, from_logits=from_logits)
    parts = parts.cpu().numpy()
    assert parts[1] == -np.inf and np.isfinite(parts[3 + 1])
    w = torch.tensor([0.7, 1.3, -0.9], device="cuda")
    plain = ctc_crf.CTC_CRF_LOSS(lamb=lamb, from_logits=from_logits, reduction="none")
    c0, g0 = _costs_and_grad(plain, yt, labels, lens, ly, w)
    assert float(c0[1]) == -np.inf and not bool((g0[1, :2] == 0).all())
    crit = ctc_crf.CTC_CRF_LOSS(lamb=lamb, from_logits=from_logits, reduction="none", zero_infinity=True)
    c1, g1 = _costs_and_grad(crit, yt, labels, lens, ly, w)
    c1, g1 = c1.cpu().numpy(), g1.cpu().numpy()
    assert c1[1] == 0.0 and not g1[1].any()
    good = [0, 2]
    sub_labels, sub_ly = _subset(labels, ly, good)
    rc, rg = _costs_and_grad(plain, yt[good].contiguous(), sub_labels, lens[good], sub_ly, w[good])
    _close(c1[good], rc.cpu().numpy(), 1e-6)
    assert np.abs(g1[good] - rg.cpu().numpy()).max() <= 1e-6
    with torch.no_grad():
        ev = crit(yt, lab, lx, lyt).cpu().numpy()
    assert ev[1] == 0.0
    _close(ev[good], c1[good], 1e-6)
    del ctx


def test_forward_only_costs_and_launches(tmp_graphs):
    """Under torch.no_grad the 'none' costs are the grad-mode costs: log p bit for bit, logZ to fp32 rounding.  The
    forward of 'none' runs the launches of the default reduction; its backward is one launch."""
    import ctc_crf
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 20, 36
    for from_logits in (False, True):
        yt, _, labels, lens, ly = _inputs(N, T, V, 77, np.linspace(T, 1, N).astype(np.int32), torch.float32, from_logits)
        args = (yt, _i32(labels), _i32(lens), _i32(ly), 0.1, True)
        c0, _, p0 = _C.ctc_crf_loss_fwd(*args, want_parts=True, from_logits=from_logits, reduction="none")
        c1, p1 = _C.ctc_crf_loss_fwd_only(*args, want_parts=True, from_logits=from_logits, reduction="none")
        p0, p1 = p0.cpu().numpy(), p1.cpu().numpy()
        assert np.array_equal(p0[N:], p1[N:])
        _close(p1[:N], p0[:N], 1e-6)
        _close(c1.cpu().numpy(), c0.cpu().numpy(), 1e-6)
        crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits, reduction="none")
        with torch.no_grad():
            ev = crit(yt, _i32(labels), _i32(lens), _i32(ly))
        _close(ev.cpu().numpy(), c0.cpu().numpy(), 1e-6)
        counts = {}
        for red in (None, "none"):
            y = yt.clone().requires_grad_(True)
            k0 = _C.launch_count()
            out = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits, reduction=red)(y, _i32(labels), _i32(lens),
                                                                                         _i32(ly))
            k1 = _C.launch_count()
            out.sum().backward()
            counts[red] = (k1 - k0, _C.launch_count() - k1)
        assert counts["none"] == (counts[None][0], 1), counts
    del ctx


@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_grad_rows_scale_stays_in_its_rows(dtype):
    """ccb_grad_rows_scale writes exactly the N*T*V elements of `out`: guard regions on both sides keep their sentinel.
    Valid rows are w[n]*G rounded once to the dtype (as torch rounds the fp32 product), rows t >= len are zeros even where
    G holds NaN, and an unknown dtype code is refused before any launch."""
    from cat_b200 import _C, _lib
    L = _lib.lib()
    dt = DTYPES[dtype]
    N, T, V, pad = 5, 13, 37, 64
    gen = torch.Generator(device="cuda").manual_seed(3)
    G = torch.randn(N, T, V, device="cuda", generator=gen)
    lens = torch.tensor([13, 0, 7, 1, 12], dtype=torch.int32, device="cuda")
    valid = torch.arange(T, device="cuda")[None, :, None] < lens[:, None, None].long()
    G = torch.where(valid, G, torch.full_like(G, float("nan")))          # never read: zeros come out regardless
    w = torch.randn(N, device="cuda", generator=gen)
    buf = torch.full((N * T * V + 2 * pad,), 7.0, dtype=dt, device="cuda")
    out = buf[pad:pad + N * T * V]
    stream = _C._stream(G.device)
    assert L.ccb_grad_rows_scale(G.data_ptr(), w.data_ptr(), lens.data_ptr(), N, T, V, out.data_ptr(), _C._DTYPES[dt],
                                 stream) == 0
    torch.cuda.synchronize()
    assert bool((buf[:pad] == 7).all()) and bool((buf[-pad:] == 7).all())
    ref = torch.where(valid, w[:, None, None] * G, torch.zeros_like(G)).to(dt)
    assert torch.equal(out.view(N, T, V), ref)
    k0 = _C.launch_count()
    assert L.ccb_grad_rows_scale(G.data_ptr(), w.data_ptr(), lens.data_ptr(), N, T, V, out.data_ptr(), 7, stream) != 0
    assert "dtype" in _lib.last_error() and _C.launch_count() == k0


def _torch_ctc(y, labels, lens, ly, w, zero_infinity):
    """torch's fp64 ctc_loss (reduction='none') and the gradient of sum_n w[n] cost[n] in the convention of
    WARP_CTC_LOSS: d(-log p)/dy with y taken as free variables.  torch's gradient assumes log-softmax inputs and carries an
    extra exp(y) * w[n] on every valid row of an utterance it does not zero; it is removed here."""
    lp = torch.tensor(y, dtype=torch.float64).transpose(0, 1).contiguous().requires_grad_(True)
    costs = torch.nn.functional.ctc_loss(lp, torch.tensor(labels, dtype=torch.long), torch.tensor(lens, dtype=torch.long),
                                         torch.tensor(ly, dtype=torch.long), blank=0, reduction="none",
                                         zero_infinity=zero_infinity)
    wd = torch.tensor(w, dtype=torch.float64)
    (g,) = torch.autograd.grad((costs * wd).sum(), lp)
    g = g.transpose(0, 1).numpy().copy()
    c = costs.detach().numpy()
    for n in range(len(lens)):     # (meaningful for the feasible utterances only, the ones compared)
        g[n, :lens[n]] -= np.exp(y[n, :lens[n]].astype(np.float64)) * w[n]
    return c, g


@pytest.mark.parametrize("zero_infinity", [False, True])
def test_warp_ctc_costs_vs_torch(zero_infinity):
    import ctc_crf
    from oracle import oracle
    N, T, V = 7, 40, 15
    lens = np.array([40, 37, 30, 22, 12, 6, 40], np.int32)
    y, _, lens, ly = oracle.synth_batch(N, T, V, seed=13, lens=lens)
    ly = np.array([8, 5, 0, 7, 4, 9, 12], np.int32)            # L = 0, and 9 labels in 6 frames: infeasible
    labels = np.random.default_rng(4).integers(1, V, size=int(ly.sum())).astype(np.int32)
    labels[1] = labels[0]                                         # a repeat
    w = np.random.default_rng(6).uniform(-2.0, 2.0, N).astype(np.float32)
    crit = ctc_crf.WARP_CTC_LOSS(reduction="none", zero_infinity=zero_infinity)
    costs, grad = _costs_and_grad(crit, torch.tensor(y, device="cuda"), labels, lens, ly, torch.tensor(w, device="cuda"))
    costs, grad = costs.cpu().numpy(), grad.cpu().numpy()
    tc, tg = _torch_ctc(y, labels, lens, ly, w, zero_infinity)
    if zero_infinity:
        assert costs[5] == 0.0 and tc[5] == 0.0 and not grad[5].any()
    else:
        assert costs[5] == np.inf and tc[5] == np.inf
    ok = [n for n in range(N) if np.isfinite(tc[n]) and n != 5]
    _close(costs[ok], tc[ok], LOSS_RTOL)
    for n in ok:
        assert np.abs(grad[n, :lens[n]] - tg[n, :lens[n]]).max() < GRAD_ATOL, n
        assert not grad[n, lens[n]:].any()
    # forward only
    with torch.no_grad():
        ev = crit(torch.tensor(y, device="cuda"), _i32(labels), _i32(lens), _i32(ly)).cpu().numpy()
    assert np.array_equal(ev, costs)
    # the scalar with zero_infinity: finite, and the mean over all N
    if zero_infinity:
        loss = ctc_crf.WARP_CTC_LOSS(zero_infinity=True)(torch.tensor(y, device="cuda"), _i32(labels), _i32(lens), _i32(ly))
        _close(float(loss.item()), float(costs.astype(np.float64).sum()) / N, 1e-6)
