"""GPU: ``warp_ctct.ctct_loss`` and ``ctct_simple_loss``, the CTC-T loss of CAT's ``topo: ctct`` transducers, against the
fp64 restatement (tests/ctct_oracle.py).

Bounds.  The oracle runs on the inputs as given, upcast to fp64.  Costs must agree to 1e-5 (1 + |ref|); for fp32 log-prob
input the row terms are the input bits and the lattice is fp64, so the cost is one fp32 rounding of an fp64 value that
differs from the oracle's by far less than an fp32 ulp: within 2 fp32 ulps.  Raw logits add the row logsumexp (__expf /
__logf, a few ulp of |lse| per row, summed over T rows).  Gradients agree to 1e-4 (1 + |ref|) elementwise, plus half an
output ulp for 16-bit gradients: each element is a posterior (fp64 lattice, one fp32 rounding) times w, or softmax times
the occupancy in fp32.
"""
import gc

import numpy as np
import pytest
import torch

import ctct_oracle as O
from test_scratch_proxy import ScratchProxy

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _return_cached_memory():
    """Each test hands the device memory it cached back when it ends.  The CAT-sized cases leave ~13 GB in torch's
    caching allocator, and later tests allocate outside it (the den context's stream-ordered scratch, the profiler's
    activity buffers): they must not find the device held by blocks nothing uses."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
IDS = ["f32", "bf16", "f16"]
HALF_ULP = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
TINY16 = {torch.float32: 0.0, torch.bfloat16: 0.0, torch.float16: 2.0 ** -25}


def _loss():
    from warp_ctct import ctct_loss
    return ctct_loss


def _batch(lx, ly, V, blank=0, seed=0, Tmax=None, Umax=None, scale=2.0, repeats=0.3):
    """Padded joint (N, Tmax, Umax+1, V) fp64 on the CPU, labels (N, Umax) int32 other than blank with some adjacent
    repeats, lengths int32."""
    rng = np.random.default_rng(seed)
    lx, ly = np.asarray(lx), np.asarray(ly)
    N, Tmax, Umax = len(lx), Tmax or int(lx.max()), Umax if Umax is not None else int(ly.max())
    z = rng.standard_normal((N, Tmax, Umax + 1, V)) * scale
    y = rng.integers(0, V - 1, (N, Umax))
    y = np.where(y >= blank, y + 1, y)
    rep = rng.random((N, Umax)) < repeats
    for u in range(1, Umax):
        y[:, u] = np.where(rep[:, u], y[:, u - 1], y[:, u])
    return (torch.tensor(z), torch.tensor(y, dtype=torch.int32), torch.tensor(lx, dtype=torch.int32),
            torch.tensor(ly, dtype=torch.int32))


def _compact(x, y, lx, ly):
    V = x.shape[-1]
    rows = torch.cat([x[n, :lx[n], :ly[n] + 1].reshape(-1, V) for n in range(len(lx))])
    return rows, torch.cat([y[n, :ly[n]] for n in range(len(lx))])


def _uncompact(g, lx, ly, like):
    out, o = torch.zeros_like(like), 0
    for n, (T, U) in enumerate(zip(lx.tolist(), ly.tolist())):
        out[n, :T, :U + 1] = g[o:o + T * (U + 1)].reshape(T, U + 1, -1)
        o += T * (U + 1)
    return out


def _log_probs(z, from_logits, dtype):
    x = z if from_logits else z.log_softmax(-1)
    return x.to(dtype)


def _run(x, y, lx, ly, compact, from_logits, reduction="none", blank=0, w=None):
    xd = x.detach().cuda().requires_grad_(True)
    c = _loss()(xd, y, lx, ly, reduction=reduction, blank=blank, compact=compact, from_logits=from_logits)
    c.backward(None if c.dim() == 0 else (torch.ones_like(c) if w is None else w))
    torch.cuda.synchronize()
    return c.detach(), xd.grad


def _assert_cost(c, ref, ulps=None):
    c = c.double().cpu().numpy()
    assert np.array_equal(np.isinf(c), np.isinf(ref)) and not np.isnan(c).any()
    f = np.isfinite(ref)
    err = np.abs(c[f] - ref[f])
    assert np.all(err <= 1e-5 * (1 + np.abs(ref[f]))), err.max()
    if ulps is not None:
        assert np.all(err <= ulps * np.spacing(np.abs(ref[f]).astype(np.float32)).astype(np.float64)), err.max()


def _assert_grad(gr, ref, dtype):
    gr = gr.double().cpu().numpy()
    bound = 1e-4 * (1 + np.abs(ref)) + HALF_ULP[dtype] * np.abs(ref) + TINY16[dtype]
    err = np.abs(gr - ref)
    assert np.all(err <= bound), (err.max(), (err / bound).max())


# ---------------------------------------------------------------------------------------------------
# oracle parity
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [37, 64])
@pytest.mark.parametrize("compact", [False, True], ids=["padded", "compact"])
@pytest.mark.parametrize("from_logits", [False, True], ids=["logprobs", "logits"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_oracle_parity(dtype, from_logits, compact, V):
    """Ragged lengths with T_n = 1 and U_n = 0 among them, adjacent repeats, blank 0 and blank != 0."""
    lx, ly = [9, 1, 6, 7, 4, 1, 2], [5, 0, 3, 0, 2, 1, 3]
    for blank in (0, V // 2):
        z, y, lxt, lyt = _batch(lx, ly, V, blank, seed=V + blank)
        x = _log_probs(z, from_logits, dtype)
        xr = x.double().numpy()
        oc, og = O.ctct_loss(xr, y.numpy(), lx, ly, blank=blank, from_logits=from_logits)
        assert np.isinf(oc[-1]) and np.isfinite(oc[:-1]).all()      # the last needs at least 3 frames
        if compact:
            xc, yc = _compact(x, y, lxt, lyt)
            c, g = _run(xc, yc, lxt, lyt, True, from_logits, blank=blank)
            g = _uncompact(g.cpu(), lxt, lyt, x)
        else:
            c, g = _run(x, y, lxt, lyt, False, from_logits, blank=blank)
        _assert_cost(c, oc, 2 if dtype == torch.float32 and not from_logits else None)
        _assert_grad(g, og, dtype)
        assert g.dtype == dtype


def test_adjacent_repeats():
    """[3, 3, 3, 5, 5] in 10 frames, and the same labels without repeats allowed to skip."""
    y = torch.tensor([[3, 3, 3, 5, 5]], dtype=torch.int32)
    for T in (8, 10, 14):
        z = torch.randn(1, T, 6, 11, dtype=torch.float64, generator=torch.Generator().manual_seed(T)) * 2
        lx, ly = torch.tensor([T], dtype=torch.int32), torch.tensor([5], dtype=torch.int32)
        for fl in (False, True):
            x = _log_probs(z, fl, torch.float32)
            oc, og = O.ctct_loss(x.double().numpy(), y.numpy(), lx, ly, from_logits=fl)
            c, g = _run(x, y, lx, ly, False, fl)
            _assert_cost(c, oc)
            _assert_grad(g, og, torch.float32)


def test_single_path():
    """T = U + repeats: exactly one alignment, 3 b 3 b 3 5 b 5 for [3, 3, 3, 5, 5] in 8 frames.  The cost is -sum lp along
    it and the log-prob gradient is exactly -w on its entries and 0 elsewhere."""
    y = torch.tensor([[3, 3, 3, 5, 5]], dtype=torch.int32)
    z = torch.randn(1, 8, 6, 9, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    x = z.log_softmax(-1).float()
    path = [(0, 0, 3), (1, 1, 0), (2, 1, 3), (3, 2, 0), (4, 2, 3), (5, 3, 5), (6, 4, 0), (7, 4, 5)]
    want = -sum(float(x[0, t, u, k]) for t, u, k in path)
    lx, ly = torch.tensor([8], dtype=torch.int32), torch.tensor([5], dtype=torch.int32)
    for w in (1.0, 0.375):
        c, g = _run(x, y, lx, ly, False, False, w=torch.tensor([w], device="cuda"))
        assert abs(c.item() - want) <= 2 * np.spacing(np.float32(abs(want)))
        exp = torch.zeros_like(x)
        for t, u, k in path:
            exp[0, t, u, k] = -w
        assert torch.equal(g.cpu(), exp)


@pytest.mark.parametrize("compact", [False, True], ids=["padded", "compact"])
@pytest.mark.parametrize("from_logits", [False, True], ids=["logprobs", "logits"])
def test_infeasible(compact, from_logits):
    """T = U + repeats - 1: cost +inf, zero gradient rows, the other utterances' bits unchanged, no NaN anywhere."""
    V = 12
    z, y, lx, ly = _batch([7, 7, 5], [5, 5, 2], V, seed=3, repeats=0.0)
    y[1] = torch.tensor([3, 3, 3, 5, 5], dtype=torch.int32)
    x = _log_probs(z, from_logits, torch.float32)
    lx_bad = lx.clone()
    lx_bad[1] = 7                       # needs 8
    lx_ok = lx.clone()
    lx_ok[1] = 8
    x_ok = torch.cat([x, torch.zeros_like(x[:, :1])], 1)
    x_ok[1, 7] = x[1, 6]
    out = {}
    for name, xx, lxx in (("bad", torch.cat([x, x[:, :1]], 1), lx_bad), ("ok", x_ok, lx_ok)):
        if compact:
            xc, yc = _compact(xx, y, lxx, ly)
            c, g = _run(xc, yc, lxx, ly, True, from_logits)
            g = _uncompact(g.cpu(), lxx, ly, xx)
        else:
            c, g = _run(xx, y, lxx, ly, False, from_logits)
        out[name] = (c.cpu(), g.cpu())
    c, g = out["bad"]
    assert c[1] == float("inf") and not torch.isnan(c).any() and not torch.isnan(g).any()
    assert not g[1].any()
    co, go = out["ok"]
    assert torch.isfinite(co).all()
    assert torch.equal(c[[0, 2]], co[[0, 2]]) and torch.equal(g[[0, 2]], go[[0, 2]])


@pytest.mark.parametrize("compact", [False, True], ids=["padded", "compact"])
def test_frame_occupancy(compact):
    """Log-prob input, reduction='sum': every frame t < T_n emits exactly one symbol, so -sum_{u,k} grad[t,u,k] = 1."""
    z, y, lx, ly = _batch([30, 12, 25, 1], [8, 3, 12, 0], 29, seed=5)
    x = z.log_softmax(-1).float()
    if compact:
        xc, yc = _compact(x, y, lx, ly)
        _, g = _run(xc, yc, lx, ly, True, False, reduction="sum")
        g = _uncompact(g.cpu(), lx, ly, x)
    else:
        _, g = _run(x, y, lx, ly, False, False, reduction="sum")
    occ = -g.double().cpu().sum((2, 3))
    for n, T in enumerate(lx.tolist()):
        assert torch.all((occ[n, :T] - 1).abs() <= 1e-5), occ[n, :T]
        assert not occ[n, T:].any()


@pytest.mark.parametrize("from_logits", [False, True], ids=["logprobs", "logits"])
def test_alpha_beta_agree_and_layouts_bit_identical(from_logits):
    from cat_b200.ctct import ctct_costs_both_ways
    z, y, lx, ly = _batch([40, 17, 33, 1, 26], [12, 5, 0, 1, 20], 67, seed=8, repeats=0.2)
    x = _log_probs(z, from_logits, torch.float32)
    a, b = ctct_costs_both_ways(x.cuda(), y, lx, ly, from_logits=from_logits)
    fin = torch.isfinite(a)
    assert torch.equal(fin, torch.isfinite(b))
    assert torch.all((a[fin] - b[fin]).abs() <= 1e-6 * (1 + a[fin].abs()))
    cp, gp = _run(x, y, lx, ly, False, from_logits)
    xc, yc = _compact(x, y, lx, ly)
    cc, gc = _run(xc, yc, lx, ly, None, from_logits)          # compact inferred from the rank
    assert torch.equal(cp, cc)
    assert torch.equal(_compact(gp.cpu(), y, lx, ly)[0], gc.cpu())


# ---------------------------------------------------------------------------------------------------
# padding, -inf, device lengths, allocator, determinism, streams, no_grad, synchronisation
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("from_logits", [False, True], ids=["logprobs", "logits"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_padding_never_read(dtype, from_logits):
    z, y, lx, ly = _batch([11, 3, 9], [4, 2, 0], 37, seed=12, Tmax=13, Umax=6)
    x = _log_probs(z, from_logits, dtype)
    xn, yn = x.clone(), y.clone()
    for n in range(3):
        xn[n, lx[n]:] = float("nan")
        xn[n, :, ly[n] + 1:] = float("nan")
        yn[n, ly[n]:] = -1
    c, g = _run(x, y, lx, ly, False, from_logits)
    cn, gn = _run(xn, yn, lx, ly, False, from_logits)
    assert torch.equal(c, cn) and torch.equal(g, gn)
    for n in range(3):
        assert not g[n, lx[n]:].any() and not g[n, :, ly[n] + 1:].any()


def test_minus_inf_entries():
    """-inf at tokens that are neither blank nor a label, and at a label entry off the paths' rows: finite costs, the
    oracle's gradient, zeros at the -inf tokens."""
    z, y, lx, ly = _batch([9, 6], [3, 2], 31, seed=4, repeats=0.0)
    y = torch.where(y >= 25, torch.ones_like(y), y)
    z[:, :, :, 25:] = -float("inf")
    for fl in (False, True):
        x = z.clone() if fl else torch.cat([z[..., :25].log_softmax(-1), z[..., 25:]], -1)
        x = x.float()
        oc, og = O.ctct_loss(x.double().numpy(), y.numpy(), lx, ly, from_logits=fl)
        assert np.isfinite(oc).all()
        c, g = _run(x, y, lx, ly, False, fl)
        _assert_cost(c, oc)
        _assert_grad(g, og, torch.float32)
        assert not g[..., 25:].any()


def test_device_lengths_bad_utterance():
    """Device lengths: a label equal to blank, outside [0, V), or a length past the tensor makes utterance 1 bad (NaN cost,
    zero gradient) and leaves the others' bits as they are, without a host synchronisation."""
    V = 23
    z, y, lx, ly = _batch([8, 6, 7], [3, 2, 4], V, seed=6)
    x = z.log_softmax(-1).float()
    c0, g0 = _run(x, y, lx, ly, False, False)
    breaks = [lambda a, b, c: a.__setitem__((1, 0), 0), lambda a, b, c: a.__setitem__((1, 1), V),
              lambda a, b, c: b.__setitem__(1, 9), lambda a, b, c: c.__setitem__(1, 5),
              lambda a, b, c: b.__setitem__(1, 0)]
    for brk in breaks:
        a, b, c_ = y.clone(), lx.clone(), ly.clone()
        brk(a, b, c_)
        a, b, c_ = a.cuda(), b.cuda(), c_.cuda()
        xd = x.cuda().requires_grad_(True)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            cst = _loss()(xd, a, b, c_, reduction="none")
            cst.backward(torch.ones_like(cst))
        finally:
            torch.cuda.set_sync_debug_mode("default")
        cst = cst.detach()
        assert torch.isnan(cst[1]) and not xd.grad[1].any()
        assert torch.equal(cst[[0, 2]], c0[[0, 2]]) and torch.equal(xd.grad[[0, 2]], g0[[0, 2]])


def _bits(t):
    t = t.detach()
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16).cpu()


@pytest.mark.parametrize("compact", [False, True], ids=["padded", "compact"])
@pytest.mark.parametrize("fl", [False, True], ids=["logprobs", "logits"])
def test_poisoned_allocator(monkeypatch, compact, fl):
    """Every buffer the loss allocates (in cat_b200.rnnt, which runs both losses) filled with 0x00, 0xFF and 0x7F: the
    same bits out, including an infeasible utterance, a bad one (device lengths) and, compact, tail rows behind the last
    utterance, which get exact zeros."""
    import cat_b200.rnnt as R
    from cat_b200 import _lib
    proxy = ScratchProxy(0)
    monkeypatch.setattr(R, "torch", proxy)
    V, blank = 24, 5
    z, y, lx, ly = _batch([6, 4, 7, 3, 5], [3, 2, 4, 1, 2], V, blank, seed=9, Tmax=8, Umax=5)
    y[2] = torch.tensor([7, 7, 7, 7, 1], dtype=torch.int32)           # needs 7 frames: feasible; utterance 3: U = 1
    y[4, :2] = 9
    lx[4] = 2                                                         # needs 3 frames: infeasible
    x = _log_probs(z, fl, torch.float32)
    if compact:
        x, yt = _compact(x, y, lx, ly)
        x = torch.cat([x, torch.randn(9, V, dtype=x.dtype)])
        yt = yt.clone()
        yt[int(ly[0])] = blank
    else:
        yt = y.clone()
        yt[1, 0] = blank
    x = x.cuda()
    dev = [t.cuda() for t in (yt, lx, ly)]
    w = torch.tensor([0.5, 1.0, -2.0, 1.5, 0.25], device="cuda")

    def run():
        xg = x.detach().clone().requires_grad_(True)
        c = _loss()(xg, *dev, reduction="none", blank=blank, compact=compact, from_logits=fl)
        (g,) = torch.autograd.grad((c * w).nan_to_num(0.0, 0.0, 0.0).sum(), xg)
        with torch.no_grad():
            ce = _loss()(x, *dev, reduction="none", blank=blank, compact=compact, from_logits=fl)
        return dict(c=c, g=g, ce=ce)

    clean = {k: _bits(v) for k, v in run().items()}
    rows = x.shape[0] if compact else x[..., 0].numel()
    seen = {nb for nb, _, d in proxy.record if d.type == "cuda"}
    assert int(_lib.lib().ccb_ctct_workspace_bytes(len(lx), rows)) in seen, sorted(seen)
    c = clean["c"].view(torch.float32)
    assert torch.isnan(c[1]) and c[4] == float("inf") and torch.isfinite(c[[0, 2, 3]]).all()
    assert torch.equal(clean["c"], clean["ce"])
    if compact:
        assert not clean["g"].view(torch.float32)[-9:].any()
    for byte in (0xFF, 0x7F):
        proxy.byte = byte
        got = {k: _bits(v) for k, v in run().items()}
        for k in clean:
            assert torch.equal(got[k], clean[k]), (hex(byte), k)


def test_determinism_streams_no_grad_and_no_sync():
    z, y, lx, ly = _batch([50, 31, 44, 12], [14, 9, 20, 3], 129, seed=21)
    for fl in (False, True):
        x = _log_probs(z, fl, torch.float32)
        c1, g1 = _run(x, y, lx, ly, False, fl)
        c2, g2 = _run(x, y, lx, ly, False, fl)
        assert torch.equal(c1, c2) and torch.equal(g1, g2)
        xc = x.cuda()
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            xs = xc.clone().requires_grad_(True)
            c3 = _loss()(xs, y, lx, ly, reduction="none", from_logits=fl)
            c3.backward(torch.ones_like(c3))
        s.synchronize()
        assert torch.equal(c3.detach(), c1) and torch.equal(xs.grad, g1)
        with torch.no_grad():
            c4 = _loss()(xc.requires_grad_(), y, lx, ly, reduction="none", from_logits=fl)
        assert torch.equal(c4, c1)
        yd, lxd, lyd = y.cuda(), lx.cuda(), ly.cuda()
        xg = xc.detach().requires_grad_(True)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for yy, a, b in ((y, lx, ly), (yd, lxd, lyd)):
                loss = _loss()(xg, yy, a, b, from_logits=fl)
                loss.backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")


@pytest.mark.parametrize("shape", [(64, 150, 20, 4232), (32, 400, 120, 1024)], ids=["aishell", "librispeech"])
def test_cat_sized_shapes(shape):
    """Compact raw logits at CAT's sizes (uniform lengths, labels without adjacent repeats, so every utterance is feasible);
    the first and last utterances against the oracle."""
    N, T, U, V = shape
    gen = torch.Generator().manual_seed(T)
    gen_d = torch.Generator(device="cuda").manual_seed(T)
    lx = torch.full((N,), T, dtype=torch.int32)
    ly = torch.full((N,), U, dtype=torch.int32)
    y = torch.randint(1, V, (N, U), generator=gen, dtype=torch.int32)
    y[:, 1:] = torch.where(y[:, 1:] == y[:, :-1], (y[:, 1:] % (V - 1)) + 1, y[:, 1:])
    x = torch.randn(N * T * (U + 1), V, generator=gen_d, device="cuda")
    yc = y.reshape(-1)
    c, g = _run(x, yc, lx, ly, True, True)
    assert torch.isfinite(c).all()
    per = T * (U + 1)
    sub = {n: (x[n * per:(n + 1) * per].cpu(), g[n * per:(n + 1) * per].cpu()) for n in (0, N - 1)}
    del x, g                                                  # the oracle runs on the host: free the device first
    for n, (xn, gn) in sub.items():
        oc, og = O.ctct_loss(xn.double().numpy(), y[n].numpy(), [T], [U], compact=True, from_logits=True)
        _assert_cost(c[n:n + 1], oc)
        _assert_grad(gn, og, torch.float32)


# ---------------------------------------------------------------------------------------------------
# ctct_simple_loss
# ---------------------------------------------------------------------------------------------------
def _simple_inputs(rng, N, Tm, Um, V, dtype, lx, ly, blank=0):
    f = torch.tensor(rng.standard_normal((N, Tm, V)) * 2).to(dtype)
    g = torch.tensor(rng.standard_normal((N, Um + 1, V)) * 2).to(dtype)
    y = rng.integers(0, V - 1, (N, Um))
    y = np.where(y >= blank, y + 1, y)
    if V > 2:
        y[:, 1] = y[:, 0]                                     # an adjacent repeat in every utterance with U >= 2
    return f, g, torch.tensor(y, dtype=torch.int64), torch.tensor(lx), torch.tensor(ly)


def _run_simple(f, g, y, lx, ly, blank=0, reduction="none"):
    from warp_ctct import ctct_simple_loss
    ft, gt = f.cuda().requires_grad_(), g.cuda().requires_grad_()
    c = ctct_simple_loss(ft, gt, y, lx, ly, reduction=reduction, blank=blank)
    c.backward(torch.ones_like(c))
    torch.cuda.synchronize()
    return c.detach(), ft.grad, gt.grad


@pytest.mark.parametrize("V", [2, 7, 1023, 4233])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_simple_oracle_parity(dtype, V):
    """int64 lengths and labels on the device, T_n = 1, U_n = 0, an infeasible utterance, blank 0 and blank != 0."""
    rng = np.random.default_rng(V)
    lx, ly = [9, 1, 4, 7, 2], [5, 0, 3, 0, 2]
    for blank in (0, V - 1):
        f, g, y, lxt, lyt = _simple_inputs(rng, 5, 9, 5, V, dtype, lx, ly, blank)
        if V == 2:
            y[:] = 1 - blank                                  # one label: every utterance is all repeats
        rc, rgf, rgg = O.simple_batch(f.double().numpy(), g.double().numpy(), y.numpy(), lx, ly, blank)
        c, gf, gg = _run_simple(f, g, y.cuda(), lxt.cuda(), lyt.cuda(), blank)
        _assert_cost(c, rc)
        _assert_grad(gf, rgf, dtype)
        _assert_grad(gg, rgg, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_simple_peaked_all_flagged(dtype):
    """f[t] and g[u] peaked by 120 on different tokens: every cell's S underflows and takes the exact fix-up."""
    N, T, U, V = 2, 7, 4, 67
    gen = torch.Generator().manual_seed(2)
    f = torch.randn(N, T, V, dtype=torch.float64, generator=gen)
    g = torch.randn(N, U + 1, V, dtype=torch.float64, generator=gen)
    f[:, :, 40] += 120
    g[:, :, 50] += 120
    y = torch.tensor([[3, 3, 5, 6], [7, 8, 8, 2]], dtype=torch.int32)
    lx, ly = torch.tensor([7, 6], dtype=torch.int32), torch.tensor([4, 3], dtype=torch.int32)
    f, g = f.to(dtype), g.to(dtype)
    rc, rgf, rgg = O.simple_batch(f.double().numpy(), g.double().numpy(), y.numpy(), lx, ly)
    c, gf, gg = _run_simple(f, g, y, lx, ly)
    _assert_cost(c, rc)
    _assert_grad(gf, rgf, dtype)
    _assert_grad(gg, rgg, dtype)


@pytest.mark.parametrize("V", [7, 1023])
def test_simple_matches_materialised(V):
    from warp_ctct import ctct_loss
    rng = np.random.default_rng(11)
    f, g, y, lx, ly = _simple_inputs(rng, 3, 8, 5, V, torch.float32, [8, 5, 6], [5, 2, 3])
    c, gf, gg = _run_simple(f, g, y, lx, ly)
    ft, gt = f.cuda().requires_grad_(), g.cuda().requires_grad_()
    cm = ctct_loss((ft[:, :, None] + gt[:, None]).log_softmax(-1), y.int(), lx.int(), ly.int(), reduction="none")
    cm.backward(torch.ones_like(cm))
    rc = cm.detach().double().cpu().numpy()
    assert np.all(np.abs(c.double().cpu().numpy() - rc) <= 2e-5 * (1 + np.abs(rc)))
    for a, b in ((gf, ft.grad), (gg, gt.grad)):
        b = b.double().cpu().numpy()
        assert np.all(np.abs(a.double().cpu().numpy() - b) <= 2e-4 * (1 + np.abs(b)))


def test_simple_determinism_no_grad_and_bad_utterance():
    from warp_ctct import ctct_simple_loss
    rng = np.random.default_rng(29)
    f, g, y, lx, ly = _simple_inputs(rng, 4, 20, 8, 257, torch.float32, [20, 13, 17, 9], [8, 4, 6, 2])
    c1, gf1, gg1 = _run_simple(f, g, y, lx, ly)
    c2, gf2, gg2 = _run_simple(f, g, y, lx, ly)
    assert torch.equal(c1, c2) and torch.equal(gf1, gf2) and torch.equal(gg1, gg2)
    with torch.no_grad():
        c3 = ctct_simple_loss(f.cuda(), g.cuda(), y, lx, ly, reduction="none")
    assert torch.equal(c3, c1)
    yb = y.clone()
    yb[1, 0] = 0
    ft, gt = f.cuda().requires_grad_(), g.cuda().requires_grad_()
    yd, lxd, lyd = yb.cuda(), lx.cuda(), ly.cuda()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        c = ctct_simple_loss(ft, gt, yd, lxd, lyd, reduction="none")
        c.backward(torch.ones_like(c))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isnan(c[1]) and not ft.grad[1].any() and not gt.grad[1].any()
    keep = [0, 2, 3]
    assert torch.equal(c.detach()[keep], c1[keep]) and torch.equal(ft.grad[keep], gf1[keep])


# ---------------------------------------------------------------------------------------------------
# CAT's TransducerTrainer with topo = "ctct"
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("joiner", ["joint_compact", "joint_padded", "logadd"])
def test_cat_ctct_trainer_step(joiner):
    """TransducerTrainer.forward's topo="ctct" branches (cat/rnnt/train.py): warp_ctct.ctct_loss(xys, y, lsub, ly) on the
    JointNet output (the compact joiner's 2-D rows, or the padded 4-D tensor), and warp_ctct.ctct_simple_loss(enc_out,
    pred_out, y, lsub, ly) for LogAdd, with LongTensor labels and lengths as CAT passes them.  The loss falls under SGD."""
    import warp_ctct
    from cat_b200.rnnt import gather_sum
    torch.manual_seed(0)
    N, T, D, H, V, Um = 3, 14, 16, 24, 11, 5
    enc = torch.nn.Linear(D, H if joiner != "logadd" else V).cuda()
    pred = torch.nn.Embedding(V, H if joiner != "logadd" else V).cuda()
    out = torch.nn.Linear(H, V).cuda()
    x = torch.randn(N, T, D, device="cuda")
    lx = torch.tensor([14, 11, 8])
    ly = torch.tensor([5, 2, 3])
    y = torch.randint(1, V, (N, Um))
    y[0, 1] = y[0, 0]
    for n in range(N):
        y[n, ly[n]:] = 0
    params = list(enc.parameters()) + list(pred.parameters()) + list(out.parameters())
    opt = torch.optim.SGD(params, lr=0.1)
    losses = []
    for _ in range(5):
        enc_out, lsub = enc(x), lx.cuda()
        pred_out = pred(torch.cat([torch.zeros(N, 1, dtype=torch.long), y], 1).cuda())
        if joiner == "logadd":
            loss = warp_ctct.ctct_simple_loss(enc_out, pred_out, y, lsub, ly)
        elif joiner == "joint_padded":
            xys = out(torch.tanh(enc_out[:, :, None] + pred_out[:, None])).log_softmax(-1)
            loss = warp_ctct.ctct_loss(xys, y.int(), lsub.int(), ly.int())
        else:
            a = torch.cat([enc_out[n, :lx[n]] for n in range(N)])
            b = torch.cat([pred_out[n, :ly[n] + 1] for n in range(N)])
            xys = out(torch.tanh(gather_sum(a, b, lx.int(), (ly + 1).int()))).log_softmax(-1)
            yc = torch.cat([y[n, :ly[n]] for n in range(N)]).int()
            loss = warp_ctct.ctct_loss(xys, yc, lsub.int(), ly.int())
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
