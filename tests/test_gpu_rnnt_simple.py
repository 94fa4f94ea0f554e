"""GPU: ``warp_rnnt.rnnt_loss_simple``, the RNN-T loss of CAT's LogAdd joiner, against the fp64 restatement
(tests/rnnt_simple_oracle.py) and against the materialised joint through ``rnnt_loss``.

Bounds.  The oracle runs on the inputs as given, upcast to fp64.  Costs must agree to 1e-5 (1 + |ref|) and gradients to
1e-4 (1 + |ref|) elementwise, plus half an output ulp for 16-bit gradients.  Where they come from: Z = mf + mg + log S is
a few fp32 roundings of values of size |Z| (S from an fp32 sum of at most V products, each within ~2 ulp, so log S is
within ~V 2^-24 relative of S, well below 1e-5 for V <= 4233); each cost sums T + U such lp's, so its error is about
(T + U) 2^-22 |Z|, below 1e-5 |cost| here because |cost| grows with (T + U) |lp|.  The lattice is fp64.  A gradient
element is exp(f - mf) (sum_u W Eg) plus the fp32 sums of at most max(T, U+1) posteriors: a few ulp per term, far below
1e-4.
"""
import numpy as np
import pytest
import torch

from rnnt_simple_oracle import batch
from test_rnnt_simple_dispatch import simple_layout

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
HALF_ULP = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
TINY16 = {torch.float32: 0.0, torch.bfloat16: 0.0, torch.float16: 2.0 ** -25}


def _loss():
    from warp_rnnt import rnnt_loss_simple
    return rnnt_loss_simple


def _inputs(rng, N, Tm, Um, V, dtype, scale=2.0, lx=None, ly=None, blank=0):
    if lx is None:
        lx = rng.integers(1, Tm + 1, N)
        lx[0] = Tm
    if ly is None:
        ly = rng.integers(0, Um + 1, N)
        ly[-1] = Um
    f = (torch.randn(N, Tm, V, dtype=torch.float64, generator=torch.Generator().manual_seed(int(rng.integers(1 << 30))))
         * scale).to(dtype)
    g = (torch.randn(N, Um + 1, V, dtype=torch.float64, generator=torch.Generator().manual_seed(int(rng.integers(1 << 30))))
         * scale).to(dtype)
    y = rng.integers(0, V - 1, (N, Um))
    y = np.where(y >= blank, y + 1, y)              # labels in [0, V) other than blank
    return f, g, torch.tensor(y, dtype=torch.int32), torch.tensor(lx, dtype=torch.int32), torch.tensor(ly, dtype=torch.int32)


def _run(f, g, y, lx, ly, reduction="none", blank=0, weights=None):
    """Costs and the gradients on f and g (backward with the given weights, or ones), on the GPU."""
    ft = f.cuda().requires_grad_()
    gt = g.cuda().requires_grad_()
    c = _loss()(ft, gt, y, lx, ly, reduction=reduction, blank=blank)
    c.backward(None if c.dim() == 0 else (torch.ones_like(c) if weights is None else weights))
    torch.cuda.synchronize()
    return c.detach(), ft.grad, gt.grad


def _ref(f, g, y, lx, ly, blank=0):
    return batch(f.double().numpy(), g.double().numpy(), y.numpy(), lx.numpy(), ly.numpy(), blank)


def _assert_cost(c, ref):
    c = c.double().cpu().numpy()
    err = np.abs(c - ref)
    assert np.all(err <= 1e-5 * (1 + np.abs(ref))), (err.max(), (err / (1e-5 * (1 + np.abs(ref)))).max())


def _assert_grad(gr, ref, dtype, scale=1.0):
    gr = gr.double().cpu().numpy()
    ref = ref * scale
    bound = 1e-4 * (1 + np.abs(ref)) + HALF_ULP[dtype] * np.abs(ref) + TINY16[dtype]
    err = np.abs(gr - ref)
    assert np.all(err <= bound), (err.max(), (err / bound).max())


# ---------------------------------------------------------------------------------------------------
# oracle parity
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [2, 7, 1023, 4233])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
def test_oracle_parity(dtype, V):
    """Odd N with ragged lengths, T_n = 1 and U_n = 0 among them, blank 0 and blank != 0, all three reductions."""
    rng = np.random.default_rng(V)
    lx = np.array([9, 1, 4, 7, 1])
    ly = np.array([6, 0, 3, 0, 2])
    for blank in (0, V - 1, V // 2):
        f, g, y, lx_t, ly_t = _inputs(rng, 5, 9, 6, V, dtype, lx=lx, ly=ly, blank=blank)
        rc, rgf, rgg = _ref(f, g, y, lx_t, ly_t, blank)
        c, gf, gg = _run(f, g, y, lx_t, ly_t, "none", blank)
        _assert_cost(c, rc)
        _assert_grad(gf, rgf, dtype)
        _assert_grad(gg, rgg, dtype)
        assert gf.dtype == dtype and gg.dtype == dtype
        for red, s in (("sum", 1.0), ("mean", 1.0 / 5)):
            c, gf, gg = _run(f, g, y, lx_t, ly_t, red, blank)
            assert abs(c.item() - rc.sum() * s) <= 1e-5 * s * (1 + np.abs(rc)).sum()
            _assert_grad(gf, rgf, dtype, s)
            _assert_grad(gg, rgg, dtype, s)


def test_signed_weights_reduction_none():
    rng = np.random.default_rng(3)
    f, g, y, lx, ly = _inputs(rng, 4, 6, 5, 33, torch.float32)
    w = torch.tensor([0.5, -2.0, 0.0, 3.0], device="cuda")
    c, gf, gg = _run(f, g, y, lx, ly, "none", 0, w)
    rc, rgf, rgg = _ref(f, g, y, lx, ly)
    wn = w.cpu().double().numpy()
    _assert_grad(gf, rgf * wn[:, None, None], torch.float32)
    _assert_grad(gg, rgg * wn[:, None, None], torch.float32)
    assert torch.all(gf[2] == 0) and torch.all(gg[2] == 0)


# ---------------------------------------------------------------------------------------------------
# equivalence with the materialised LogAdd path
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [7, 1023])
def test_matches_materialised_logadd(V):
    from warp_rnnt import rnnt_loss
    rng = np.random.default_rng(11)
    f, g, y, lx, ly = _inputs(rng, 3, 8, 5, V, torch.float32)
    c, gf, gg = _run(f, g, y, lx, ly, "none")
    ft, gt = f.cuda().requires_grad_(), g.cuda().requires_grad_()
    cm = rnnt_loss((ft[:, :, None] + gt[:, None]).log_softmax(-1), y, lx, ly, reduction="none")
    cm.backward(torch.ones_like(cm))
    rc = cm.detach().double().cpu().numpy()
    assert np.all(np.abs(c.double().cpu().numpy() - rc) <= 2e-5 * (1 + np.abs(rc)))
    for a, b in ((gf, ft.grad), (gg, gt.grad)):
        b = b.double().cpu().numpy()
        assert np.all(np.abs(a.double().cpu().numpy() - b) <= 2e-4 * (1 + np.abs(b)))


# ---------------------------------------------------------------------------------------------------
# underflow: flagged cells and the exact fix-up
# ---------------------------------------------------------------------------------------------------
def _read_ws(ws, N, Tmax, Umax):
    lay, total = simple_layout(N, Tmax, Umax)
    raw = ws.cpu().numpy()
    assert raw.size == total
    return {k: raw[o:o + n * dt.itemsize].view(dt) for k, (o, n, dt) in lay.items()}


def _peaked(N, T, U, V, M, seed):
    """f[t] peaks at token a_t, g[u] at b_u (both away from blank and the labels) by M over N(0,1) entries: cells with
    a_t != b_u have S ~ 2 exp(-M), cells with a_t = b_u have S ~ 1."""
    gen = torch.Generator().manual_seed(seed)
    f = torch.randn(N, T, V, dtype=torch.float64, generator=gen)
    g = torch.randn(N, U + 1, V, dtype=torch.float64, generator=gen)
    peaks = torch.arange(V // 2, V)
    a = peaks[torch.randint(0, len(peaks), (N, T), generator=gen)]
    b = peaks[torch.randint(0, len(peaks), (N, U + 1), generator=gen)]
    b[:, ::3] = a[:, :1].expand(N, b[:, ::3].shape[1])   # some cells agree (row 0 of f with every third row of g)
    f.scatter_(2, a[..., None], M)
    g.scatter_(2, b[..., None], M)
    y = torch.randint(1, V // 2, (N, U), generator=gen, dtype=torch.int32)
    return f, g, y


@pytest.mark.parametrize("M", [60.0, 120.0])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
def test_underflow_flagged_cells(dtype, M):
    """M = 60 puts S near 2^-86 (below 2^-64, still a normal fp32); M = 120 flushes it to zero, so the GEMM's Z alone would
    be -inf.  The flagged cells are exactly those with S < 2^-64 in fp64, they carry the likely paths (their lp's are
    about -M where the agreeing cells' are about -2M), and costs and gradients still meet the oracle bounds."""
    from cat_b200.rnnt_simple import _forward, check_rnnt_simple_args
    N, T, U, V = 3, 7, 5, 67
    f, g, y = _peaked(N, T, U, V, M, seed=int(M))
    f, g = f.to(dtype), g.to(dtype)
    lx = torch.tensor([7, 5, 1], dtype=torch.int32)
    ly = torch.tensor([5, 2, 0], dtype=torch.int32)
    fc, gc = f.cuda(), g.cuda()
    shape = check_rnnt_simple_args(fc, gc, y, lx, ly, "none", 0)
    costs, ws, _ = _forward(fc, gc, y, lx, ly, 0, True, shape)
    W = _read_ws(ws, N, T, U)
    f64, g64 = f.double(), g.double()
    Ef = torch.exp(f64 - f64.amax(-1, keepdim=True))
    Eg = torch.exp(g64 - g64.amax(-1, keepdim=True))
    S64 = torch.einsum("ntk,nuk->ntu", Ef, Eg).numpy()
    S = W["S"].reshape(N, T, U + 1)
    n_flag = 0
    for n in range(N):
        live = S64[n, :lx[n], :ly[n] + 1]
        want = live < 2.0 ** -64
        assert np.all((live < 2.0 ** -70) | (live > 2.0 ** -58)), "a cell sits too near the threshold"
        got = ~(S[n, :lx[n], :ly[n] + 1] >= np.float32(2.0 ** -64))
        assert np.array_equal(got, want)
        n_flag += int(want.sum())
        if M > 100:     # the GEMM's own S is flushed to zero: its Z alone would be -inf
            assert np.all(S[n, :lx[n], :ly[n] + 1][want] == 0)
    assert n_flag > 0
    rc, rgf, rgg = _ref(f, g, y, lx, ly)
    _assert_cost(costs, rc)
    c, gf, gg = _run(f, g, y, lx, ly, "none")
    assert torch.equal(c, costs)
    _assert_cost(c, rc)
    _assert_grad(gf, rgf, dtype)
    _assert_grad(gg, rgg, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
def test_minus_inf_entries(dtype):
    """-inf in f or g at tokens that are neither blank nor a label: finite costs, zero gradient at those tokens."""
    rng = np.random.default_rng(5)
    V = 37
    f, g, y, lx, ly = _inputs(rng, 3, 6, 4, V, dtype)
    y = torch.where(y >= 30, torch.ones_like(y), y)
    f[:, :, 30] = -float("inf")
    f[0, :, 33] = -float("inf")
    g[:, :, 31] = -float("inf")
    g[:, 0, 34:] = -float("inf")
    rc, rgf, rgg = _ref(f, g, y, lx, ly)
    assert np.all(np.isfinite(rc))
    c, gf, gg = _run(f, g, y, lx, ly, "none")
    _assert_cost(c, rc)
    _assert_grad(gf, rgf, dtype)
    _assert_grad(gg, rgg, dtype)
    assert torch.all(gf[:, :, 30] == 0) and torch.all(gg[:, :, 31] == 0)


# ---------------------------------------------------------------------------------------------------
# padding, device lengths, determinism, streams
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
def test_padding_never_read(dtype):
    """NaN in every padded row of f and g and -1 in the padded labels: the costs and gradients are bit-identical to the
    same batch with zero padding and to each utterance called alone at its own size; padded gradient rows are exactly 0."""
    rng = np.random.default_rng(17)
    N, Tm, Um, V = 5, 70, 35, 129
    lx = np.array([70, 3, 66, 1, 40])
    ly = np.array([12, 35, 0, 4, 33])
    f, g, y, lx_t, ly_t = _inputs(rng, N, Tm, Um, V, dtype, lx=lx, ly=ly)
    fz, gz, yz = f.clone(), g.clone(), y.clone()
    for n in range(N):
        f[n, lx[n]:] = float("nan")
        g[n, ly[n] + 1:] = float("nan")
        y[n, ly[n]:] = -1
        fz[n, lx[n]:] = 0
        gz[n, ly[n] + 1:] = 0
        yz[n, ly[n]:] = 1
    c, gf, gg = _run(f, g, y, lx_t, ly_t)
    cz, gfz, ggz = _run(fz, gz, yz, lx_t, ly_t)
    assert torch.equal(c, cz) and torch.equal(gf, gfz) and torch.equal(gg, ggz)
    for n in range(N):
        T, U = int(lx[n]), int(ly[n])
        assert torch.all(gf[n, T:] == 0) and not torch.signbit(gf[n, T:]).any()
        assert torch.all(gg[n, U + 1:] == 0) and not torch.signbit(gg[n, U + 1:]).any()
        c1, gf1, gg1 = _run(f[n:n + 1, :T], g[n:n + 1, :U + 1], y[n:n + 1, :U], lx_t[n:n + 1], ly_t[n:n + 1])
        assert torch.equal(c1, c[n:n + 1]) and torch.equal(gf1[0], gf[n, :T]) and torch.equal(gg1[0], gg[n, :U + 1])


@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
def test_device_lengths_bad_utterance(idt):
    """Device lengths and labels, int32 or int64, no host synchronisation.  A bad utterance (a label equal to blank, a label
    outside [0, V), a length past Tmax or Umax, or an int64 value beyond the int32 range) has NaN cost and zero gradients,
    and every other utterance's results are bit-identical to a call in which it is valid."""
    rng = np.random.default_rng(23)
    N, Tm, Um, V = 4, 9, 6, 41
    f, g, y, lx, ly = _inputs(rng, N, Tm, Um, V, torch.float32, lx=np.array([9, 5, 7, 3]), ly=np.array([6, 4, 2, 5]))
    c0, gf0, gg0 = _run(f, g, y, lx, ly)
    yb, lxb, lyb = y.to(idt), lx.to(idt), ly.to(idt)
    breaks = [("label = blank", lambda a, b, c: a.__setitem__((2, 1), 0)),
              ("label = V", lambda a, b, c: a.__setitem__((2, 0), V)),
              ("T > Tmax", lambda a, b, c: b.__setitem__(2, Tm + 1)),
              ("U > Umax", lambda a, b, c: c.__setitem__(2, Um + 1)),
              ("T < 1", lambda a, b, c: b.__setitem__(2, 0))]
    if idt == torch.int64:
        breaks.append(("label wraps", lambda a, b, c: a.__setitem__((2, 0), 2 ** 32 + 1)))
        breaks.append(("T wraps", lambda a, b, c: b.__setitem__(2, 2 ** 32 + 3)))
    for what, brk in breaks:
        a, b, c_ = yb.clone(), lxb.clone(), lyb.clone()
        brk(a, b, c_)
        ft, gt = f.cuda().requires_grad_(), g.cuda().requires_grad_()
        a, b, c_ = a.cuda(), b.cuda(), c_.cuda()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            cst = _loss()(ft, gt, a, b, c_, reduction="none")
            cst.backward(torch.ones_like(cst))
        finally:
            torch.cuda.set_sync_debug_mode("default")
        cst = cst.detach()
        assert torch.isnan(cst[2]), what
        assert torch.all(ft.grad[2] == 0) and torch.all(gt.grad[2] == 0), what
        keep = [0, 1, 3]
        assert torch.equal(cst[keep], c0[keep]), what
        assert torch.equal(ft.grad[keep], gf0[keep]) and torch.equal(gt.grad[keep], gg0[keep]), what


def test_determinism_streams_and_no_grad():
    rng = np.random.default_rng(29)
    f, g, y, lx, ly = _inputs(rng, 6, 40, 15, 257, torch.float32)
    c1, gf1, gg1 = _run(f, g, y, lx, ly)
    c2, gf2, gg2 = _run(f, g, y, lx, ly)
    assert torch.equal(c1, c2) and torch.equal(gf1, gf2) and torch.equal(gg1, gg2)
    s = torch.cuda.Stream()
    fc, gc = f.cuda(), g.cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        ft, gt = fc.clone().requires_grad_(), gc.clone().requires_grad_()
        c3 = _loss()(ft, gt, y, lx, ly, reduction="none")
        c3.backward(torch.ones_like(c3))
    s.synchronize()
    assert torch.equal(c3.detach(), c1) and torch.equal(ft.grad, gf1) and torch.equal(gt.grad, gg1)
    with torch.no_grad():
        c4 = _loss()(fc.requires_grad_(), gc, y, lx, ly, reduction="none")
    assert torch.equal(c4, c1)
    c5 = _loss()(fc.detach(), gc, y, lx, ly, reduction="none")       # nothing requires grad: forward only
    assert torch.equal(c5, c1) and not c5.requires_grad


def test_one_input_requires_grad():
    rng = np.random.default_rng(31)
    f, g, y, lx, ly = _inputs(rng, 3, 5, 4, 19, torch.float32)
    _, gf, gg = _run(f, g, y, lx, ly)
    gt = g.cuda().requires_grad_()
    c = _loss()(f.cuda(), gt, y, lx, ly, reduction="none")
    c.backward(torch.ones_like(c))
    assert torch.equal(gt.grad, gg)


# ---------------------------------------------------------------------------------------------------
# CAT's call and CAT-sized shapes
# ---------------------------------------------------------------------------------------------------
def test_cat_logadd_branch():
    """TransducerTrainer.forward's LogAdd branch (cat/rnnt/train.py): a linear encoder and an embedding predictor,
    LongTensor y and ly on the CPU and lsub on the device, one SGD step through warp_rnnt.rnnt_loss_simple against one
    through the materialised LogAdd joint (joiner.LogAdd.forward) and warp_rnnt.rnnt_loss."""
    import warp_rnnt
    torch.manual_seed(0)
    N, T, D, V, Um = 3, 12, 16, 11, 5
    enc0 = torch.nn.Linear(D, V).cuda()
    pred0 = torch.nn.Embedding(V, V).cuda()
    x = torch.randn(N, T, D, device="cuda")
    lx = torch.tensor([12, 9, 4])
    ly = torch.tensor([5, 2, 3])
    y = torch.randint(1, V, (N, Um))
    for n in range(N):
        y[n, ly[n]:] = 0
    params = []
    for simple in (True, False):
        enc = torch.nn.Linear(D, V).cuda()
        pred = torch.nn.Embedding(V, V).cuda()
        enc.load_state_dict(enc0.state_dict())
        pred.load_state_dict(pred0.state_dict())
        opt = torch.optim.SGD(list(enc.parameters()) + list(pred.parameters()), lr=0.5)
        enc_out, lsub = enc(x), lx.cuda()
        pred_out = pred(torch.cat([torch.zeros(N, 1, dtype=torch.long), y], 1).cuda())
        if simple:
            loss = warp_rnnt.rnnt_loss_simple(enc_out, pred_out, y, lsub, ly)
        else:
            logp = (enc_out.unsqueeze(2) + pred_out.unsqueeze(1)).log_softmax(dim=-1)
            loss = warp_rnnt.rnnt_loss(logp, y.int(), lsub.int(), ly.int())
        opt.zero_grad()
        loss.backward()
        opt.step()
        params.append([p.detach().clone() for p in list(enc.parameters()) + list(pred.parameters())])
    for a, b in zip(*params):
        assert torch.all((a - b).abs() <= 0.5 * 2e-4 * (1 + b.abs())), (a - b).abs().max()


@pytest.mark.parametrize("shape", [(64, 150, 20, 4232), (32, 400, 120, 1024)], ids=["aishell", "librispeech"])
def test_cat_sized_shapes(shape):
    N, Tm, Um, V = shape
    rng = np.random.default_rng(Tm)
    f, g, y, lx, ly = _inputs(rng, N, Tm, Um, V, torch.float32, scale=1.0)
    c, gf, gg = _run(f, g, y, lx, ly)
    assert torch.isfinite(c).all()
    for n in (0, N - 1):
        T, U = int(lx[n]), int(ly[n])
        rc, rgf, rgg = _ref(f[n:n + 1, :T], g[n:n + 1, :U + 1], y[n:n + 1, :U], lx[n:n + 1], ly[n:n + 1])
        _assert_cost(c[n:n + 1], rc)
        _assert_grad(gf[n:n + 1, :T], rgf, torch.float32)
        _assert_grad(gg[n:n + 1, :U + 1], rgg, torch.float32)
