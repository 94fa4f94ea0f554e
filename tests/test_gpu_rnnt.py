"""GPU: the RNN-T loss (cat_b200.rnnt / warp_rnnt) and the joiner's gather.sum (gather) against the fp64 restatement
oracle/rnnt.py at the parity gate (loss 1e-4 relative, gradient 1e-3 absolute), and their invariants: layouts, input modes,
reductions, grad mode, padding, -inf, device lengths, determinism, streams, CAT-sized shapes."""
import numpy as np
import pytest
import torch

from oracle import rnnt as R

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def _case(N, Tm, Um, V, seed, dtype=torch.float32, scale=2.0):
    g = torch.Generator().manual_seed(seed)
    lx = torch.randint(1, Tm + 1, (N,), generator=g, dtype=torch.int32)
    ly = torch.randint(0, Um + 1, (N,), generator=g, dtype=torch.int32)
    lx[0], ly[-1] = Tm, Um
    z = (torch.randn(N, Tm, Um + 1, V, generator=g) * scale).to(dtype)
    y = torch.randint(1, V, (N, Um), generator=g, dtype=torch.int32)
    return z, y, lx, ly


def _compact(x, y, lx, ly):
    V = x.shape[-1]
    rows = torch.cat([x[n, :lx[n], :ly[n] + 1].reshape(-1, V) for n in range(len(lx))])
    return rows, torch.cat([y[n, :ly[n]] for n in range(len(lx))])


def _unpack(g, lx, ly):
    """Compact rows -> per-utterance blocks (list of (T, U+1, V))."""
    out, o = [], 0
    for T, U in zip(lx.tolist(), ly.tolist()):
        out.append(g[o:o + T * (U + 1)].reshape(T, U + 1, -1))
        o += T * (U + 1)
    return out


def _run(x, y, lx, ly, compact, from_logits, reduction="sum", dev="cuda", **kw):
    from warp_rnnt import rnnt_loss
    xd = x.to(dev).requires_grad_(True)
    loss = rnnt_loss(xd, y, lx, ly, reduction=reduction, compact=compact, from_logits=from_logits, **kw)
    (loss.sum() if reduction == "none" else loss).backward()
    return loss.detach(), xd.grad


# half an ulp of each gradient dtype, relative: the gradient is returned rounded to the input's dtype
HALF_ULP = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}


def _check(cost, grad, oc, og, mask=None):
    c = cost.double().cpu().numpy()
    assert np.all(np.abs(c - oc) <= 1e-4 * np.maximum(1.0, np.abs(oc))), (c, oc)
    gr = grad.double().cpu().numpy()
    if mask is not None:
        assert not gr[~mask].any()
        gr, og = gr[mask], og[mask]
    assert np.all(np.abs(gr - og) < 1e-3 + HALF_ULP[grad.dtype] * np.abs(og))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("from_logits", [False, True])
@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("V", [37, 64])        # 37: rows not a multiple of 16 bytes (element path); 64: 16-byte chunks
def test_matches_oracle(dtype, from_logits, compact, V):
    z, y, lx, ly = _case(5, 9, 6, V, seed=V + 3)
    x = z if from_logits else z.log_softmax(-1)
    x = x.to(dtype)
    xr = x.float().numpy()                           # the oracle is fed the rounded values
    oc, og = R.rnnt_loss(xr, y.numpy(), lx.numpy(), ly.numpy(), compact=False, from_logits=from_logits)
    mask = np.zeros(x.shape[:3], bool)
    for n in range(5):
        mask[n, :lx[n], :ly[n] + 1] = True
    if compact:
        xc, yc = _compact(x, y, lx, ly)
        cost, grad = _run(xc, yc, lx, ly, True, from_logits, reduction="none")
        assert grad.dtype == dtype
        ogc = np.concatenate([og[n][mask[n]].reshape(-1, V) for n in range(5)])
        _check(cost, grad, oc, ogc)
    else:
        cost, grad = _run(x, y, lx, ly, False, from_logits, reduction="none")
        assert grad.dtype == dtype
        _check(cost, grad, oc, og, mask[..., None].repeat(V, -1))


@pytest.mark.parametrize("from_logits", [False, True])
def test_compact_and_padded_bit_identical(from_logits):
    z, y, lx, ly = _case(6, 11, 7, 48, seed=11)
    x = z if from_logits else z.log_softmax(-1)
    pc, pg = _run(x, y, lx, ly, False, from_logits, reduction="none")
    xc, yc = _compact(x, y, lx, ly)
    cc, cg = _run(xc, yc, lx, ly, True, from_logits, reduction="none")
    assert torch.equal(pc, cc)
    for n, blk in enumerate(_unpack(cg, lx, ly)):
        assert torch.equal(pg[n, :lx[n], :ly[n] + 1], blk)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_raw_logits_match_log_softmax_chain(dtype):
    from warp_rnnt import rnnt_loss
    z, y, lx, ly = _case(4, 10, 5, 96, seed=5)
    xc, yc = _compact(z, y, lx, ly)
    zd = xc.to(dtype).cuda().requires_grad_(True)
    a = rnnt_loss(zd, yc, lx, ly, reduction="none", compact=True, from_logits=True)
    a.sum().backward()
    z2 = xc.to(dtype).cuda().requires_grad_(True)
    b = rnnt_loss(z2.float().log_softmax(-1), yc, lx, ly, reduction="none", compact=True)
    b.sum().backward()
    assert torch.allclose(a, b, rtol=1e-5, atol=0)
    assert (zd.grad.float() - z2.grad.float()).abs().max() < (1e-5 if dtype == torch.float32 else 2e-3)


def test_reductions_and_weights():
    z, y, lx, ly = _case(5, 8, 4, 32, seed=9)
    x = z.log_softmax(-1)
    xc, yc = _compact(x, y, lx, ly)
    costs, g1 = _run(xc, yc, lx, ly, True, False, reduction="none")
    w = torch.linspace(0.5, 2.0, 5, device="cuda")
    from warp_rnnt import rnnt_loss
    xd = xc.cuda().requires_grad_(True)
    (rnnt_loss(xd, yc, lx, ly, reduction="none", compact=True) * w).sum().backward()
    rows_w = torch.cat([w[n].expand(int(lx[n] * (ly[n] + 1))) for n in range(5)])
    assert torch.allclose(xd.grad, g1 * rows_w[:, None], rtol=1e-6, atol=1e-7)
    s, gs = _run(xc, yc, lx, ly, True, False, reduction="sum")
    m, gm = _run(xc, yc, lx, ly, True, False, reduction="mean")
    assert torch.allclose(s, costs.sum()) and torch.allclose(m, costs.mean())
    assert torch.equal(gs, g1)
    assert torch.allclose(gm, g1 / 5, rtol=1e-6, atol=1e-8)
    # the default is the batch mean, as CAT's Manager assumes
    from warp_rnnt import rnnt_loss as f
    assert torch.equal(f(xc.cuda(), yc, lx, ly, compact=True), m)


def test_no_grad_matches_grad_mode_bits():
    from warp_rnnt import rnnt_loss
    z, y, lx, ly = _case(7, 13, 9, 40, seed=2)
    xc, yc = _compact(z, y, lx, ly)
    for fl in (False, True):
        xd = (xc if fl else xc.log_softmax(-1)).cuda().requires_grad_(True)
        a = rnnt_loss(xd, yc, lx, ly, reduction="none", compact=True, from_logits=fl)
        with torch.no_grad():
            b = rnnt_loss(xd, yc, lx, ly, reduction="none", compact=True, from_logits=fl)
        assert torch.equal(a.detach(), b)


def test_padding_is_never_read():
    z, y, lx, ly = _case(4, 9, 5, 24, seed=4)
    for fl in (False, True):
        x = (z if fl else z.log_softmax(-1)).clone()
        ref_c, ref_g = _run(x, y, lx, ly, False, fl, reduction="none")
        for n in range(4):
            x[n, lx[n]:] = float("nan")
            x[n, :, ly[n] + 1:] = float("nan")
        c, g = _run(x, y, lx, ly, False, fl, reduction="none")
        assert torch.isfinite(c).all() and torch.isfinite(g).all()
        assert torch.equal(c, ref_c) and torch.equal(g, ref_g)
        for n in range(4):
            assert not g[n, lx[n]:].any() and not g[n, :, ly[n] + 1:].any()


def test_minus_inf_entries():
    z, y, lx, ly = _case(4, 8, 5, 20, seed=6)
    lp = z.log_softmax(-1)
    g = torch.Generator().manual_seed(1)
    hole = torch.rand(lp.shape, generator=g) < 0.2
    hole[..., 0] = False                         # blank stays finite: every utterance keeps a path
    for fl, x in ((False, lp.masked_fill(hole, float("-inf"))), (True, z.masked_fill(hole, float("-inf")))):
        oc, og = R.rnnt_loss(x.numpy(), y.numpy(), lx.numpy(), ly.numpy(), from_logits=fl)
        c, gr = _run(x, y, lx, ly, False, fl, reduction="none")
        fin = np.isfinite(oc)
        assert np.array_equal(np.isfinite(c.cpu().numpy()), fin)
        mask = np.zeros(x.shape, bool)
        for n in range(4):
            if fin[n]:
                mask[n, :lx[n], :ly[n] + 1] = True
        c2 = c.double().cpu().numpy()
        assert np.all(np.abs(c2[fin] - oc[fin]) <= 1e-4 * np.maximum(1, np.abs(oc[fin])))
        assert np.abs(gr.double().cpu().numpy()[mask] - og[mask]).max() < 1e-3


def test_device_lengths_and_bad_utterances():
    z, y, lx, ly = _case(5, 7, 4, 16, seed=8)
    x = z.log_softmax(-1)
    xc, yc = _compact(x, y, lx, ly)
    c_host, g_host = _run(xc, yc, lx, ly, True, False, reduction="none")
    c_dev, g_dev = _run(xc, yc.cuda(), lx.cuda(), ly.cuda(), True, False, reduction="none")
    assert torch.equal(c_host, c_dev) and torch.equal(g_host, g_dev)
    # a label equal to blank / out of range in utterance 1, lengths overrunning the tensor in the last utterance: NaN cost
    # and zero gradient rows for those, the others unchanged
    ly2 = ly.clone()
    ly2[1] = max(int(ly[1]), 1)
    x2, y2 = _compact(x, y, lx, ly2)
    y2 = y2.clone()
    y2[int(ly2[0])] = 0
    lx2 = lx.clone()
    lx2[-1] += 1
    c, g = _run(x2, y2.cuda(), lx2.cuda(), ly2.cuda(), True, False, reduction="none")
    assert torch.isnan(c[1]) and torch.isnan(c[-1]) and torch.isfinite(c[[0, 2, 3]]).all()
    blocks = _unpack(g, lx, ly2)
    assert not blocks[1].any() and not blocks[-1].any()
    y3 = y2.clone()
    y3[int(ly2[0])] = 999
    c3, _ = _run(x2, y3.cuda(), lx.cuda(), ly2.cuda(), True, False, reduction="none")
    assert torch.isnan(c3[1]) and torch.isfinite(c3[[0, 2, 3, 4]]).all()
    assert torch.equal(c3[[0, 2, 3]], c[[0, 2, 3]])


def test_deterministic_and_side_stream():
    z, y, lx, ly = _case(8, 20, 10, 128, seed=12)
    xc, yc = _compact(z, y, lx, ly)
    a = _run(xc, yc, lx, ly, True, True, reduction="none")
    b = _run(xc, yc, lx, ly, True, True, reduction="none")
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    s = torch.cuda.Stream()
    xd = xc.cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        c = _run(xd, yc, lx, ly, True, True, reduction="none")
    s.synchronize()
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


def _oracle_rows(xc, yc, lx, ly, from_logits, rows, blank=0):
    """Costs of every utterance and gradient rows `rows` of a large compact case: the row terms in fp64 on the GPU, the
    lattice in fp64 on the host (the full fp64 gradient would not fit host memory)."""
    V = xc.shape[1]
    R_ = xc.shape[0]
    lse = torch.empty(R_, dtype=torch.float64, device=xc.device)
    for i in range(0, R_, 1 << 16):
        blk = xc[i:i + (1 << 16)].double()
        lse[i:i + (1 << 16)] = torch.logsumexp(blk, -1) if from_logits else 0.0
    lab_row = torch.full((R_,), blank, dtype=torch.long)
    o = lo = 0
    uidx = []
    for T, U in zip(lx.tolist(), ly.tolist()):
        r = torch.arange(T * (U + 1))
        u = r % (U + 1)
        lab = torch.cat([yc[lo:lo + U].long(), torch.tensor([blank])])
        lab_row[o:o + T * (U + 1)] = lab[u]
        uidx.append((o, T, U))
        o += T * (U + 1)
        lo += U
    ar = torch.arange(R_, device=xc.device)
    lpb = (xc[ar, blank].double() - lse).cpu().numpy()
    lpl = (xc[ar, lab_row.to(xc.device)].double() - lse).cpu().numpy()
    costs, pbs, pls = [], np.zeros(R_), np.zeros(R_)
    for o, T, U in uidx:
        lp, _, pb, pl = R.lattice(lpb[o:o + T * (U + 1)].reshape(T, U + 1), lpl[o:o + T * (U + 1)].reshape(T, U + 1)[:, :U])
        costs.append(-lp)
        pbs[o:o + T * (U + 1)] = pb.reshape(-1)
        pls[o:o + T * (U + 1)] = np.pad(pl, ((0, 0), (0, 1))).reshape(-1)
    xr = xc[rows.to(xc.device)].double().cpu().numpy()
    g = np.exp(xr - lse[rows.to(xc.device)].cpu().numpy()[:, None]) * (pbs[rows] + pls[rows])[:, None] if from_logits \
        else np.zeros_like(xr)
    g[np.arange(len(rows)), blank] -= pbs[rows]
    lr = lab_row[rows].numpy()
    has = pls[rows] != 0
    g[np.arange(len(rows))[has], lr[has]] -= pls[rows][has]
    return np.array(costs), g


@pytest.mark.parametrize("shape,from_logits,dtype", [
    ((64, 150, 20, 4232), False, torch.float32),     # aishell-like, CAT's log-prob path
    ((64, 150, 20, 4232), True, torch.float16),      # ... raw fp16 joiner output
    ((32, 400, 120, 1024), False, torch.float32),    # Librispeech-like
    ((32, 400, 120, 1024), True, torch.float32),
])
def test_cat_sized(shape, from_logits, dtype):
    from warp_rnnt import rnnt_loss
    N, T, U, V = shape
    g = torch.Generator(device="cuda").manual_seed(N + T)
    lx = torch.full((N,), T, dtype=torch.int32)
    lx[1::2] = T - T // 5
    ly = torch.full((N,), U, dtype=torch.int32)
    ly[1::3] = U // 2
    rows = int((lx.long() * (ly.long() + 1)).sum())
    x = (torch.randn(rows, V, device="cuda", generator=g) * 2).to(dtype)
    if not from_logits:
        x = x.float().log_softmax(-1).to(dtype)
    yc = torch.randint(1, V, (int(ly.sum()),), dtype=torch.int32, device="cuda", generator=g)
    xd = x.requires_grad_(True)
    cost = rnnt_loss(xd, yc, lx.cuda(), ly.cuda(), reduction="none", compact=True, from_logits=from_logits)
    cost.sum().backward()
    pick = torch.randint(0, rows, (2000,), generator=torch.Generator().manual_seed(3))
    oc, og = _oracle_rows(x.detach().float() if dtype != torch.float32 else x.detach(), yc.cpu(), lx, ly, from_logits, pick)
    c = cost.detach().double().cpu().numpy()
    assert np.all(np.abs(c - oc) <= 1e-4 * np.abs(oc)), np.abs(c - oc).max()
    assert np.all(np.abs(xd.grad[pick.cuda()].double().cpu().numpy() - og) < 1e-3 + HALF_ULP[dtype] * np.abs(og))


@pytest.mark.parametrize("shape", [(2, 50, 400, 32), (3, 9, 450, 8), (512, 20, 5, 16)])
def test_long_labels_and_large_batch(shape):
    N, T, U, V = shape
    z, y, lx, ly = _case(N, T, U, V, seed=21, scale=1.0)
    for fl in (False, True):
        x = z if fl else z.log_softmax(-1)
        xc, yc = _compact(x, y, lx, ly)
        oc, og = R.rnnt_loss(xc.numpy(), yc.numpy(), lx.numpy(), ly.numpy(), compact=True, from_logits=fl)
        c, g = _run(xc, yc, lx, ly, True, fl, reduction="none")
        _check(c, g, oc, og)


def test_alpha_and_beta_agree():
    from cat_b200.rnnt import rnnt_costs_both_ways
    z, y, lx, ly = _case(16, 60, 40, 64, seed=31)
    xc, yc = _compact(z, y, lx, ly)
    a, b = rnnt_costs_both_ways(xc.cuda(), yc, lx, ly, compact=True, from_logits=True)
    assert torch.allclose(a, b, rtol=1e-6, atol=0)


# ---------------------------------------------------------------------------------------------------
# gather.sum
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_gather_sum(dtype):
    import gather
    N, Tm, Um, H = 6, 17, 9, 80
    g = torch.Generator().manual_seed(0)
    la = torch.randint(1, Tm + 1, (N,), generator=g)
    lb = torch.randint(1, Um + 1, (N,), generator=g)
    la[2] = 0
    ea = torch.randn(N, Tm, H, generator=g).to(dtype).cuda()
    eb = torch.randn(N, Um, H, generator=g).to(dtype).cuda()
    a = gather.cat(ea, la).requires_grad_(True)
    b = gather.cat(eb, lb.cuda()).requires_grad_(True)
    out = gather.sum(a, b, la.cuda(), lb.cuda())
    ref = torch.cat([(ea[n, :la[n], None, :] + eb[n, None, :lb[n], :]).reshape(-1, H) for n in range(N)])
    assert out.dtype == dtype and torch.equal(out, ref)
    go = torch.randn(out.shape, generator=g).to(dtype).cuda()
    out.backward(go)
    # torch's broadcast-sum backward in fp32 as the reference
    ta = torch.cat([ea.float()[n, :la[n]] for n in range(N)]).requires_grad_(True)
    tb = torch.cat([eb.float()[n, :lb[n]] for n in range(N)]).requires_grad_(True)
    oa = ob = 0
    parts = []
    for n in range(N):
        parts.append((ta[oa:oa + la[n], None, :] + tb[None, ob:ob + lb[n], :]).reshape(-1, H))
        oa += int(la[n])
        ob += int(lb[n])
    torch.cat(parts).backward(go.float())
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    assert (a.grad.float() - ta.grad).abs().max() <= tol * max(1.0, float(ta.grad.abs().max()))
    assert (b.grad.float() - tb.grad).abs().max() <= tol * max(1.0, float(tb.grad.abs().max()))
    a3, b3 = a.detach().requires_grad_(True), b.detach().requires_grad_(True)
    gather.sum(a3, b3, la, lb).backward(go)
    assert torch.equal(a3.grad, a.grad) and torch.equal(b3.grad, b.grad)


def test_cat_joiner_training_step():
    """CAT's TransducerTrainer.compute_join + JointNet(compact=True) + warp_rnnt.rnnt_loss, restated on tiny sizes through
    the shim packages, against the same model built padded and scored by the fp64 restatement."""
    import gather
    import warp_rnnt
    torch.manual_seed(0)
    N, T, U, H, V = 4, 7, 5, 16, 11
    fc_enc, fc_dec = torch.nn.Linear(H, H).cuda(), torch.nn.Linear(H, H).cuda()
    fc = torch.nn.Sequential(torch.nn.Tanh(), torch.nn.Linear(H, V)).cuda()
    params = list(fc_enc.parameters()) + list(fc_dec.parameters()) + list(fc.parameters())
    enc = torch.randn(N, T, H, device="cuda")
    pred = torch.randn(N, U + 1, H, device="cuda")
    lsub = torch.tensor([7, 5, 6, 3], dtype=torch.int32)
    ly = torch.tensor([5, 2, 0, 3], dtype=torch.int32)
    y = torch.randint(1, V, (N, U), dtype=torch.int32)

    # compute_join (cat/rnnt/train.py:168-186) + JointNet.forward in "add" mode with the compact layout (joiner.py:102-122)
    lsub_d, ly_d, y_d = lsub.cuda(), ly.cuda(), y.cuda()
    yc = gather.cat(y_d, ly_d)
    e = gather.cat(enc, lsub_d)
    p = gather.cat(pred, ly_d + 1)
    xys = fc(gather.sum(fc_enc(e), fc_dec(p), lsub_d, ly_d + 1)).log_softmax(-1)
    loss = warp_rnnt.rnnt_loss(xys, yc, lsub_d, ly_d, compact=True)
    loss.backward()
    got = [q.grad.clone() for q in params]
    for q in params:
        q.grad = None

    # the padded model, scored by the restatement and chained through autograd
    xp = fc(fc_enc(enc)[:, :, None, :] + fc_dec(pred)[:, None, :, :]).log_softmax(-1)
    oc, og = R.rnnt_loss(xp.detach().cpu().numpy(), y.numpy(), lsub.numpy(), ly.numpy())
    xp.backward(torch.tensor(og / N, dtype=torch.float32, device="cuda"))
    assert abs(loss.item() - oc.mean()) <= 1e-5 * abs(oc.mean())
    for a, b in zip(got, [q.grad for q in params]):
        assert (a - b).abs().max() < 1e-4
