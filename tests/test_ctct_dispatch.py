"""CPU: the fp64 restatement of the CTC-T loss (tests/ctct_oracle.py) against brute-force enumeration of every frame path
and against torch's CTC loss on u-independent log-probs; the LogAdd restatement against the materialised joint; the
argument checks of ``warp_ctct.ctct_loss`` and ``ctct_simple_loss``; and the workspace sizes the library asks for."""
import itertools

import numpy as np
import pytest
import torch

import ctct_oracle as O
from test_rnnt_simple_dispatch import simple_layout
from test_rnnt_workspace import META_DTYPE


def brute_force(lp, y, blank=0):
    """Every one of the V^T frame paths of one utterance, collapsed by the CTC-T rule: blank keeps u and moves to the blank
    state, y_u from the label state repeats, y_{u+1} emits a new label (from the label state only when y_{u+1} != y_u); any
    other symbol, or a path that does not end at u = U, has no alignment.  Returns (log P, d cost / d lp)."""
    T, U1, V = lp.shape
    U = U1 - 1
    P, post = 0.0, np.zeros_like(lp)
    for path in itertools.product(range(V), repeat=T):
        u, last_l, score, cells = 0, False, 0.0, []
        for t, k in enumerate(path):
            cells.append((t, u, k))
            score += lp[t, u, k]
            if k == blank:
                last_l = False
            elif last_l and k == y[u - 1]:
                pass
            elif u < U and k == y[u] and not (last_l and y[u] == y[u - 1]):
                u, last_l = u + 1, True
            else:
                break
        else:
            if u == U:
                p = np.exp(score)
                P += p
                for c in cells:
                    post[c] += p
    if P == 0.0:
        return -np.inf, np.zeros_like(lp)
    return np.log(P), -post / P


LABELS = [[], [1], [2, 2], [1, 2], [3, 3, 3], [1, 2, 1], [2, 3, 3], [1, 1, 2, 2]]


@pytest.mark.parametrize("y", LABELS, ids=lambda y: "y" + "".join(map(str, y)) if y else "empty")
@pytest.mark.parametrize("T", [1, 2, 4, 6])
def test_oracle_matches_brute_force(T, y):
    V = 4
    if V ** T > 4096:
        pytest.skip("enumeration too large")
    rng = np.random.default_rng(T * 100 + len(y))
    y = np.array(y, np.int64)
    for blank in (0, 2) if 2 not in y else (0,):
        z = rng.standard_normal((T, len(y) + 1, V)) * 1.5
        lp = z - np.log(np.exp(z).sum(-1, keepdims=True))
        yb = np.where(y >= blank, y + (blank > 0), y) if blank else y
        yb = np.minimum(yb, V - 1)
        if blank and np.any(yb == blank):
            continue
        ref_lp, ref_g = brute_force(lp, yb, blank)
        logp, logp_b, g, _ = O.utterance(lp, yb, blank)
        reps = int(np.sum(yb[1:] == yb[:-1])) if len(yb) else 0
        assert np.isfinite(ref_lp) == (T >= len(yb) + reps)
        if np.isfinite(ref_lp):
            assert np.isclose(logp, ref_lp, rtol=1e-12, atol=1e-12) and np.isclose(logp_b, ref_lp, rtol=1e-12, atol=1e-12)
            assert np.allclose(g, ref_g, rtol=0, atol=1e-12)
            occ = -g.sum((1, 2))
            assert np.allclose(occ, 1.0, atol=1e-12)
        else:
            assert logp == -np.inf and logp_b == -np.inf and not g.any()


def _ctc_case(rng, N, Tm, Um, V, infeasible=False):
    lx = rng.integers(1, Tm + 1, N)
    lx[0] = Tm
    ly = np.minimum(rng.integers(0, Um + 1, N), lx)
    y = rng.integers(1, V, (N, Um))
    y[:, 1::3] = y[:, 0::3][:, :y[:, 1::3].shape[1]]       # some adjacent repeats
    if infeasible:
        ly[-1] = min(Um, Tm)
        y[-1, :] = 1                                        # all repeats: needs 2U - 1 frames
        lx[-1] = max(1, 2 * ly[-1] - 2)
    return lx, ly, y


@pytest.mark.parametrize("seed", range(4))
def test_u_independent_is_ctc(seed):
    """lp(t,u,k) = c(t,k) for every u: the cost is torch's CTC cost in fp64 (+inf for an infeasible utterance), and the
    raw-logit gradient summed over u is torch's gradient of ctc_loss(log_softmax(c)) with respect to c."""
    rng = np.random.default_rng(seed)
    N, Tm, Um, V = 5, 9, 5, 6
    lx, ly, y = _ctc_case(rng, N, Tm, Um, V, infeasible=seed % 2 == 1)
    c = rng.standard_normal((N, Tm, V)) * 2
    x = np.broadcast_to(c[:, :, None, :], (N, Tm, Um + 1, V)).copy()
    costs, grad = O.ctct_loss(x, y, lx, ly, from_logits=True)
    ct = torch.tensor(c, requires_grad=True)
    ref = torch.nn.functional.ctc_loss(ct.log_softmax(-1).transpose(0, 1), torch.tensor(y), torch.tensor(lx),
                                       torch.tensor(ly), blank=0, reduction="none", zero_infinity=False)
    r = ref.detach().numpy()
    assert np.array_equal(np.isinf(costs), np.isinf(r))
    fin = np.isfinite(r)
    assert np.allclose(costs[fin], r[fin], rtol=1e-10, atol=1e-10)
    ref[torch.tensor(fin)].sum().backward()
    gsum = grad.sum(2)
    assert np.allclose(gsum[fin], ct.grad.numpy()[fin], rtol=0, atol=1e-10)
    assert not grad[~fin].any()
    # log-prob input: the same costs
    lpc = c - np.log(np.exp(c).sum(-1, keepdims=True))
    costs_lp, _ = O.ctct_loss(np.broadcast_to(lpc[:, :, None, :], x.shape), y, lx, ly)
    assert np.allclose(costs_lp[fin], r[fin], rtol=1e-10, atol=1e-10) and np.all(np.isinf(costs_lp[~fin]))


def test_layouts_and_input_modes_agree():
    rng = np.random.default_rng(7)
    N, Tm, Um, V = 3, 6, 4, 5
    lx, ly, y = np.array([6, 3, 5]), np.array([4, 0, 2]), rng.integers(1, V, (N, Um))
    z = rng.standard_normal((N, Tm, Um + 1, V))
    cp, gp = O.ctct_loss(z, y, lx, ly, from_logits=True)
    rows = np.concatenate([z[n, :lx[n], :ly[n] + 1].reshape(-1, V) for n in range(N)])
    lab = np.concatenate([y[n, :ly[n]] for n in range(N)])
    cc, gc = O.ctct_loss(rows, lab, lx, ly, compact=True, from_logits=True)
    assert np.array_equal(cp, cc)
    assert np.array_equal(np.concatenate([gp[n, :lx[n], :ly[n] + 1].reshape(-1, V) for n in range(N)]), gc)
    lp = z - np.log(np.exp(z).sum(-1, keepdims=True))
    cl, gl = O.ctct_loss(lp, y, lx, ly)
    assert np.allclose(cl, cp, rtol=1e-12)
    # chain rule through log_softmax: raw gradient = gl - softmax * sum_k gl
    assert np.allclose(gp, gl - np.exp(lp) * gl.sum(-1, keepdims=True), atol=1e-12)


@pytest.mark.parametrize("case", range(4))
def test_simple_matches_materialised_joint(case):
    rng = np.random.default_rng(500 + case)
    N, Tm, Um, V = [(2, 5, 3, 4), (3, 7, 4, 7), (1, 1, 0, 3), (3, 6, 5, 9)][case]
    lx = rng.integers(1, Tm + 1, N)
    ly = rng.integers(0, Um + 1, N)
    lx[0], ly[-1] = Tm, Um
    f = rng.standard_normal((N, Tm, V)) * 2
    g = rng.standard_normal((N, Um + 1, V)) * 2
    y = rng.integers(1, V, (N, Um))
    c, gf, gg = O.simple_batch(f, g, y, lx, ly)
    jc, jg = O.ctct_loss(f[:, :, None] + g[:, None], y, lx, ly, from_logits=True)
    fin = np.isfinite(jc)
    assert np.array_equal(np.isinf(c), ~fin)
    assert np.allclose(c[fin], jc[fin], rtol=1e-12)
    assert np.allclose(gf, jg.sum(2), atol=1e-12) and np.allclose(gg, jg.sum(1), atol=1e-12)


# ---------------------------------------------------------------------------------------------------
# argument checks (no device needed)
# ---------------------------------------------------------------------------------------------------
def _args(compact=False):
    if compact:
        x = torch.zeros(3 * 3 + 2 * 2, 5)
        y = torch.tensor([1, 2, 3], dtype=torch.int32)
    else:
        x = torch.zeros(2, 3, 3, 5)
        y = torch.tensor([[1, 2], [3, 0]], dtype=torch.int32)
    return x, y, torch.tensor([3, 2], dtype=torch.int32), torch.tensor([2, 1], dtype=torch.int32)


def test_compact_inferred_from_rank():
    from warp_ctct import ctct_loss
    for compact in (True, False):
        x, y, lx, ly = _args(compact)
        with pytest.raises(ValueError, match="CUDA"):        # valid: stops at the device check
            ctct_loss(x, y, lx, ly)
        with pytest.raises(ValueError, match="CUDA"):
            ctct_loss(x, y, lx, ly, compact=compact)
        with pytest.raises(ValueError, match="ctct_loss"):   # an explicit flag that disagrees with the shape
            ctct_loss(x, y, lx, ly, compact=not compact)
    x, y, lx, ly = _args()
    with pytest.raises(ValueError, match="compact"):
        ctct_loss(x[0], y, lx, ly)


def test_ctct_checks():
    from warp_ctct import ctct_loss
    x, y, lx, ly = _args()
    with pytest.raises(AssertionError):
        ctct_loss(x.double(), y, lx, ly)
    with pytest.raises(AssertionError):
        ctct_loss(x, y.long(), lx, ly)
    with pytest.raises(ValueError, match="ctct_loss: reduction"):
        ctct_loss(x, y, lx, ly, reduction="avg")
    for blank in (-1, 5, True):
        with pytest.raises(ValueError, match="blank"):
            ctct_loss(x, y, lx, ly, blank=blank)
    with pytest.raises(ValueError, match="overrun"):
        ctct_loss(x, y, torch.tensor([4, 2], dtype=torch.int32), ly)
    with pytest.raises(ValueError, match=">= 1"):
        ctct_loss(x, y, torch.tensor([0, 2], dtype=torch.int32), ly)
    with pytest.raises(ValueError, match="differ from blank"):
        ctct_loss(x, torch.tensor([[1, 0], [3, 0]], dtype=torch.int32), lx, ly)
    xc, yc, lxc, lyc = _args(True)
    with pytest.raises(ValueError, match="rows"):
        ctct_loss(xc[:-1], yc, lxc, lyc)
    with pytest.raises(ValueError, match="label lengths"):
        ctct_loss(xc, yc[:2], lxc, lyc)


@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
def test_ctct_simple_checks(idt):
    from warp_ctct import ctct_simple_loss
    f, g = torch.zeros(2, 3, 5), torch.zeros(2, 3, 5)
    y = torch.tensor([[1, 2], [3, 0]], dtype=idt)
    lx, ly = torch.tensor([3, 2], dtype=idt), torch.tensor([2, 1], dtype=idt)
    with pytest.raises(AssertionError):
        ctct_simple_loss(f, g.half(), y, lx, ly)
    with pytest.raises(ValueError, match="ctct_simple_loss: reduction"):
        ctct_simple_loss(f, g, y, lx, ly, reduction="avg")
    with pytest.raises(ValueError, match="overrun"):
        ctct_simple_loss(f, g, y, lx, torch.tensor([3, 0], dtype=idt))
    with pytest.raises(ValueError, match="differ from blank"):
        ctct_simple_loss(f, g, y, lx, ly, blank=2)
    with pytest.raises(ValueError, match="CUDA"):
        ctct_simple_loss(f, g, y, lx, ly)


def test_checks_need_no_device(monkeypatch):
    from cat_b200 import _lib
    from warp_ctct import ctct_loss, ctct_simple_loss

    def no_lib():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "lib", no_lib)
    x, y, lx, ly = _args()
    with pytest.raises(ValueError, match="CUDA"):
        ctct_loss(x, y, lx, ly)
    with pytest.raises(ValueError, match="CUDA"):
        ctct_simple_loss(torch.zeros(2, 3, 5), torch.zeros(2, 3, 5), y, lx, ly)


# ---------------------------------------------------------------------------------------------------
# workspace: meta, tail, logp; alpha and beta with two fp64 cells per row; lpb, lpl, lpr, lse (fp32 per row), each aligned
# to 256 bytes.  The simple loss: that layout over the N Tmax (Umax+1) padded cells, then the LogAdd blocks and PR.
# ---------------------------------------------------------------------------------------------------
def _align256(b):
    return (b + 255) // 256 * 256


def ctct_layout(N, rows):
    """{block: (byte offset, element count, numpy dtype)} of the CTC-T loss's workspace, and its total."""
    blocks = [("meta", N, META_DTYPE), ("tail", 1, np.dtype("<i8")), ("logp", 2 * N, np.dtype(np.float64)),
              ("alpha", 2 * rows, np.dtype(np.float64)), ("beta", 2 * rows, np.dtype(np.float64))]
    blocks += [(name, rows, np.dtype(np.float32)) for name in ("lpb", "lpl", "lpr", "lse")]
    out, o = {}, 0
    for name, count, dt in blocks:
        out[name] = (o, count, dt)
        o += 256 if name == "tail" else _align256(count * dt.itemsize)
    return out, o


def ctct_simple_layout(N, Tmax, Umax):
    cells = N * Tmax * (Umax + 1)
    out, o = ctct_layout(N, cells)
    rn, rn_total = simple_layout(N, Tmax, Umax)
    base = rn["mf"][0]                       # the LogAdd blocks follow the lattice blocks in the same order
    for name in ("mf", "mg", "ff", "fg", "S", "W", "PB", "PL"):
        off, count, dt = rn[name]
        out[name] = (o + off - base, count, dt)
    o += rn_total - base
    out["PR"] = (o, cells, np.dtype(np.float32))
    return out, o + _align256(4 * cells)


@pytest.mark.parametrize("N", [1, 2, 7, 256, 257, 4097])
def test_ctct_workspace_bytes(N):
    from cat_b200 import _lib
    L = _lib.lib()
    for rows in (0, 1, 7, 33, 255, 256, 12345, 600_000, 3_000_000_017):
        lay, total = ctct_layout(N, rows)
        assert int(L.ccb_ctct_workspace_bytes(N, rows)) == total, (N, rows)
        offs = sorted(o for o, _, _ in lay.values())
        assert all(o % 256 == 0 for o in offs)
        # 48 bytes per row, 56 per utterance, at most 255 bytes of padding per block
        assert 48 * rows + 56 * N <= total <= 48 * rows + 56 * N + 256 + 9 * 255
    assert int(L.ccb_ctct_workspace_bytes(0, 10)) == 0 and int(L.ccb_ctct_workspace_bytes(2, -1)) == 0


@pytest.mark.parametrize("N,Tmax,Umax", [(1, 1, 0), (3, 5, 0), (5, 33, 17), (64, 150, 20), (32, 400, 120), (257, 61, 9)])
def test_ctct_simple_workspace_bytes(N, Tmax, Umax):
    from cat_b200 import _lib
    L = _lib.lib()
    lay, total = ctct_simple_layout(N, Tmax, Umax)
    assert int(L.ccb_ctct_simple_workspace_bytes(N, Tmax, Umax)) == total
    assert all(o % 256 == 0 for o, _, _ in lay.values())
    cells = N * Tmax * (Umax + 1)
    base = 68 * cells + 8 * (N * Tmax + N * (Umax + 1)) + 56 * N
    assert base <= total <= base + 256 + 18 * 255
    for args in ((0, 3, 2), (2, 0, 2), (2, 3, -1)):
        assert int(L.ccb_ctct_simple_workspace_bytes(*args)) == 0
