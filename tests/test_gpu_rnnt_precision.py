"""GPU: the RNN-T loss and gather.sum stage by stage, each stage against an fp64 recomputation from its own inputs, at the
precision the kernels deliver rather than at the parity gate of tests/test_gpu_rnnt.py.

The forward leaves its stages in the workspace (tests/test_rnnt_workspace.py restates the layout): per-utterance meta, the
row terms lpb / lpl (and lse for raw logits), the fp64 cells alpha / beta and log P from both.  Each is checked against
  - meta: the host's own offsets in both layouts, and `bad` exactly for the utterances the device lengths make bad;
  - lpb / lpl: the input bits for log-probs; for raw logits lse within `lse_bound`, and lpb = fl(x_blank - lse) exactly;
  - alpha, beta, log P: `oracle.rnnt.cells` run on the kernel's own lpb / lpl, within `lattice_bound`;
  - costs: exactly fp32(-log P) of the workspace;
  - gradient: pb / pl recomputed in fp64 from the workspace's alpha, beta, lpb, lpl and log P, within `grad_bound_prob`
    (and, for raw logits, the `__expf` term of the softmax part, derived where `stages` builds it).
End to end, with no workspace involved, the costs (and log-prob gradients) are held to `oracle/rnnt.py` within bounds built
from the same terms.  Every bound is derived in its function's docstring.  The largest error / bound seen per stage and
dtype is printed at the end of the module (run with -s to see it).
"""

import numpy as np
import pytest
import torch

from oracle import rnnt as R
from test_rnnt_workspace import read_workspace
from test_scratch_proxy import ScratchProxy

pytestmark = pytest.mark.gpu

DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
U32 = 2.0 ** -24                    # fp32 unit roundoff
ULP32 = 2.0 ** -23                  # fp32 ulp relative to the value, at most
# half an ulp of each output dtype, relative; and half its smallest subnormal, absolute
HALF_ULP = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
HALF_SUB = {torch.float32: 2.0 ** -150, torch.bfloat16: 2.0 ** -134, torch.float16: 2.0 ** -25}

RATIOS = {}


def _ratio(stage, dtype, err, bound):
    """Record max(err / bound) for the table, and assert err <= bound everywhere.  err, bound: same-shape arrays."""
    err, bound = np.asarray(err, np.float64).reshape(-1), np.asarray(bound, np.float64).reshape(-1)
    if err.size == 0:
        return
    assert np.all(np.isfinite(err)), (stage, dtype)
    worst = int(np.argmax(err - bound))
    assert err[worst] <= bound[worst], (stage, dtype, worst, err[worst], bound[worst])
    key = (stage, str(dtype).replace("torch.", ""))
    r = float(np.max(err / bound))
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _ratio_table():
    yield
    if RATIOS:
        print("\nlargest observed error / bound")
        for (stage, dt), r in sorted(RATIOS.items()):
            print(f"  {stage:14s} {dt:9s} {r:.3g}")


def _gamma(k):
    return k * U32 / (1.0 - k * U32)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _batch(lx, ly, V, blank, seed, Tmax=None, Umax=None, scale=2.0, shift=0.0):
    """Padded inputs (z (N, Tmax, Umax+1, V) fp64 raw logits, labels (N, Umax) int32 avoiding blank) for the lengths."""
    lx, ly = np.asarray(lx, np.int32), np.asarray(ly, np.int32)
    N = len(lx)
    Tmax = int(lx.max()) if Tmax is None else Tmax
    Umax = int(ly.max()) if Umax is None else Umax
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((N, Tmax, Umax + 1, V)) * scale
    if shift:
        z += rng.choice([-shift, shift], (N, Tmax, Umax + 1, 1))
    others = np.array([k for k in range(V) if k != blank], np.int32)
    y = rng.choice(others, (N, Umax)).astype(np.int32) if len(others) and Umax else np.zeros((N, Umax), np.int32)
    return z, y, lx, ly


def _inputs(z, y, lx, ly, compact, from_logits, dtype):
    """(x on the GPU in dtype, labels, lx, ly on the host) of the layout and input mode; log-probs are made in fp64."""
    with np.errstate(invalid="ignore"):          # NaN padding stays NaN
        x = z if from_logits else z - np.logaddexp.reduce(z, axis=-1, keepdims=True)
    x = torch.tensor(x, dtype=torch.float64).to(dtype)
    y_t, lx_t, ly_t = torch.tensor(y), torch.tensor(lx), torch.tensor(ly)
    if compact:
        V = x.shape[-1]
        x = torch.cat([x[n, :lx[n], :ly[n] + 1].reshape(-1, V) for n in range(len(lx))])
        y_t = torch.cat([y_t[n, :ly[n]] for n in range(len(lx))])
    return x.cuda(), y_t, lx_t, ly_t


def _layout(lx, ly, compact, Tmax, Umax):
    """Host restatement of the offsets: per utterance (roff, loff, ts, span), and the tail."""
    out, r, l = [], 0, 0
    for n, (T, U) in enumerate(zip(lx.tolist(), ly.tolist())):
        if compact:
            out.append((r, l, U + 1, T * (U + 1)))
            r += T * (U + 1)
            l += U
        else:
            out.append((n * Tmax * (Umax + 1), n * Umax, Umax + 1, Tmax * (Umax + 1)))
    return out, (r if compact else len(lx) * Tmax * (Umax + 1))


# ---------------------------------------------------------------------------------------------------------------------
# bounds
# ---------------------------------------------------------------------------------------------------------------------
def lse_bound(xr, V):
    """Per row, a bound on |lse_kernel - lse| for the raw-logit row pass (fp32 rows xr on the GPU), and the fp64 lse.

    The kernel keeps per lane an online (max m, sum s) over its chunks, with s += __expf(v - m) per element and
    s *= __expf(m_old - m_new) when the maximum grows, merges the 32 lanes in 5 shuffle rounds
    (s = s __expf(m - mm) + s' __expf(m' - mm)), and returns l = m + __logf(s).  With M the row maximum, t_i = exp(v_i - M)
    and S = sum t_i:
      - Term i passes through its own __expf, at most C - 1 rescales (C = ceil(V / 32) chunks per lane on the element
        path, more than on the vector path) and 5 merges: at most C + 5 calls.  The CUDA Programming Guide gives __expf
        2 + floor(1.173 |x|) ulp, and the arguments along the chain add up to v_i - M (each rescale moves the running
        maximum), so the calls cost at most 2 (C + 5) + 1.173 (M - v_i) ulp; each argument is one fp32 subtraction, whose
        rounding is at most u |x|, another 0.5 (M - v_i) ulp.  One ulp is at most 2^-23 of the value.
      - fp32 adds and multiplies on term i's path: at most ceil(V / 32) + 8 in-lane adds, C rescale multiplies and 3 per
        merge: gamma_m with m = ceil(V / 32) + 8 + C + 15.
      - __expf flushes results below 2^-126 to zero: at most V 2^-126 against S >= 1.
    All terms are positive, so the relative error of s is at most the t-weighted mean of the terms' errors:
      eps_s = 2^-23 (2 (C + 6) + 1.673 mean_t(M - v)) + gamma_m + V 2^-126.
    Then |log s_kernel - log S| <= eps_s / (1 - eps_s); __logf adds 2^-21.41 absolute on [0.5, 2] and 3 ulp of its result
    elsewhere (the larger of the two is taken, as s may sit on either side of 2); the final add m + log s rounds by
    u |l| <= u (|lse| + 1)."""
    xd = xr.double()
    M = xd.max(-1, keepdim=True).values
    t = torch.exp(xd - M)
    S = t.sum(-1)
    gap = torch.where(t > 0, t * (M - xd), torch.zeros_like(t)).sum(-1) / S
    lse = M[:, 0] + torch.log(S)
    C = -(-V // 32)
    m = C + 8 + C + 15
    eps = ULP32 * (2 * (C + 6) + 1.673 * gap) + _gamma(m) + V * 2.0 ** -126
    logs = torch.log(S)
    elog = torch.clamp(3 * ULP32 * logs.abs(), min=2.0 ** -21.41)      # either regime: s_kernel may sit across 2
    bound = eps / (1 - eps) + elog + U32 * (lse.abs() + 1)
    return lse, bound


def lattice_bound(steps, big):
    """|alpha_kernel - alpha_oracle| (and beta, log P) for a cell `steps` recursion steps from the start.

    Both sides are fp64 and run the same recursion x = logaddexp(c1 + l1, c2 + l2); they differ only in their rounding.  One
    step of either side rounds the two adds (2^-53 |x| each), |c1 + l1 - c2 - l2| (whose effect through exp(-d), log1p is
    at most 2^-53 d e^-d <= 2^-53), exp and log1p (an ulp each of values <= 1 and <= ln 2) and the final add (2^-53 |x|):
    at most 2^-51 (1 + |x|) per side, 2^-50 (1 + |x|) for the difference.  logaddexp is 1-Lipschitz in the max norm of its
    inputs (its weights sum to 1), so differences do not grow along the path, they only add up: with |x| <= big for every
    cell and term of the utterance, steps 2^-50 (1 + big)."""
    return steps * 2.0 ** -50 * (1.0 + big)


def grad_bound_prob(ref, S):
    """|pb_kernel - pb| for pb = w exp(alpha + lpb + beta' - log P) recomputed in fp64 from the kernel's own cells.

    The kernel sums the exponent in fp64 (3 adds, each rounded by 2^-53 of a partial sum <= S = |alpha| + |lp| + |beta'| +
    |log P|), takes the fp64 exp (1 ulp), rounds to fp32 and multiplies by w in fp32: relative (1 + u)^2 (1 + 2^-51 (S + 1))
    - 1, plus 2^-149 absolute where the results are fp32 subnormals."""
    rel = (1 + U32) ** 2 * (1 + 2.0 ** -51 * (S + 1)) - 1
    return rel * np.abs(ref) + 2.0 ** -149


# ---------------------------------------------------------------------------------------------------------------------
# the stage check
# ---------------------------------------------------------------------------------------------------------------------
def _live(lx, ly, lay):
    """Per live row: (global row, n, t, u), host int64 arrays."""
    rows, ns, ts, us = [], [], [], []
    for n, ((roff, _, tsz, _), T, U) in enumerate(zip(lay, lx.tolist(), ly.tolist())):
        t, u = np.meshgrid(np.arange(T), np.arange(U + 1), indexing="ij")
        rows.append((roff + t * tsz + u).reshape(-1))
        ns.append(np.full(T * (U + 1), n))
        ts.append(t.reshape(-1))
        us.append(u.reshape(-1))
    return [np.concatenate(a).astype(np.int64) for a in (rows, ns, ts, us)]


def stages(x, y, lx, ly, blank, compact, from_logits, w=None):
    """Run the forward through `_forward` and the loss through autograd on x (GPU, the layout's shape) and check every
    stage; returns (costs, grad)."""
    from cat_b200.rnnt import _forward, check_rnnt_args, rnnt_loss
    dtype = x.dtype
    shape = check_rnnt_args(x, y, lx, ly, "none", blank, compact)
    N, rows, V, Tmax, Umax = shape
    costs, costs_b, ws, _ = _forward(x, y, lx, ly, blank, compact, from_logits, True, shape)
    W = read_workspace(ws.cpu().numpy(), N, rows)
    lay, tail = _layout(lx, ly, compact, Tmax, Umax)

    # meta
    meta = W["meta"]
    assert meta["roff"].tolist() == [a[0] for a in lay] and meta["loff"].tolist() == [a[1] for a in lay]
    assert meta["ts"].tolist() == [a[2] for a in lay] and meta["span"].tolist() == [a[3] for a in lay]
    assert meta["T"].tolist() == lx.tolist() and meta["U"].tolist() == ly.tolist() and not meta["bad"].any()
    assert int(W["tail"][0]) == tail

    # row terms
    row, un, tt, uu = _live(lx, ly, lay)
    yc = y.reshape(-1).numpy().astype(np.int64)
    lab = np.where(uu < ly.numpy()[un], yc[np.minimum(meta["loff"][un] + uu, max(len(yc) - 1, 0))] if len(yc) else blank,
                   blank)
    has_l = uu < ly.numpy()[un]
    xr = x.reshape(rows, V)
    row_d, lab_d = torch.tensor(row, device="cuda"), torch.tensor(lab, device="cuda")
    xb32 = xr[row_d, blank].float().cpu().numpy()
    xl32 = xr[row_d, lab_d].float().cpu().numpy()
    lpb, lpl = W["lpb"][row], W["lpl"][row]
    if from_logits:
        lse64, dl = (v.cpu().numpy() for v in lse_bound(xr[row_d].float(), V))
        l32 = W["lse"][row]
        _ratio("lse", dtype, np.abs(l32.astype(np.float64) - lse64), dl)
        assert np.array_equal(lpb, xb32 - l32)
        assert np.array_equal(lpl[has_l], (xl32 - l32)[has_l])
    else:
        assert np.array_equal(lpb.view(np.int32), xb32.view(np.int32))
        assert np.array_equal(lpl[has_l].view(np.int32), xl32[has_l].view(np.int32))

    # lattice, per utterance, on the kernel's own row terms
    lpb64 = lpb.astype(np.float64)
    lpl64 = np.where(has_l, lpl, np.float32(0)).astype(np.float64)     # lpl at u = U is never written
    alpha, beta = W["alpha"][row], W["beta"][row]
    logp = W["logp"]
    a_o, b_o = np.empty(len(row)), np.empty(len(row))
    lp_o, big = np.empty(N), np.empty(N)
    starts = np.concatenate([[0], np.cumsum((lx.numpy().astype(np.int64)) * (ly.numpy() + 1))])
    for n in range(N):
        T, U = int(lx[n]), int(ly[n])
        s = slice(starts[n], starts[n + 1])
        pb_, pl_ = lpb64[s].reshape(T, U + 1), lpl64[s].reshape(T, U + 1)[:, :U]
        a, b = R.cells(pb_, pl_)
        a_o[s], b_o[s] = a.reshape(-1), b.reshape(-1)
        lp_o[n] = a[T - 1, U] + pb_[T - 1, U]
        fin = [np.abs(v[np.isfinite(v)]) for v in (a, b, pb_, pl_)]
        # every cell, term and sum c + l of the recursion is at most twice the largest of them in magnitude
        big[n] = max([float(v.max()) for v in fin if v.size] + [abs(lp_o[n])]) * 2
    for name, got, ref, steps in (("alpha", alpha, a_o, tt + uu + 1),
                                  ("beta", beta, b_o, (lx.numpy()[un] - 1 - tt) + (ly.numpy()[un] - uu) + 1)):
        fin = np.isfinite(ref)
        assert np.array_equal(fin, np.isfinite(got)) and np.array_equal(got[~fin], ref[~fin]), name
        _ratio(name, dtype, np.abs(got - ref)[fin], lattice_bound(steps, big[un])[fin])
    lsteps = lx.numpy() + ly.numpy() + 1
    _ratio("logP", dtype, np.abs(logp[:N] - lp_o), lattice_bound(lsteps, big))
    _ratio("logP", dtype, np.abs(logp[N:] - b_o[starts[:-1]]), lattice_bound(lsteps, big))

    # costs: one rounding of the fp64 log P
    assert np.array_equal(costs.cpu().numpy(), (-logp[:N]).astype(np.float32))
    assert np.array_equal(costs_b.cpu().numpy(), (-logp[N:]).astype(np.float32))

    # gradient through autograd on the same inputs
    w_t = torch.ones(N, device="cuda") if w is None else torch.tensor(w, dtype=torch.float32, device="cuda")
    xg = x.detach().requires_grad_(True)          # x's own storage: a misaligned base stays misaligned
    c2 = rnnt_loss(xg, y, lx, ly, reduction="none", blank=blank, compact=compact, from_logits=from_logits)
    assert torch.equal(c2.detach(), costs)
    (g,) = torch.autograd.grad((c2 * w_t).sum(), xg)
    assert g.dtype == dtype and g.shape == x.shape
    g = g.reshape(rows, V)
    wn = w_t.cpu().numpy().astype(np.float64)[un]
    Tn, Un = lx.numpy()[un], ly.numpy()[un]
    lP = logp[un]
    nxt_b = np.where(tt < Tn - 1, W["beta"][np.minimum(row + meta["ts"][un], rows - 1)], np.where(uu == Un, 0.0, -np.inf))
    nxt_l = np.where(has_l, W["beta"][np.minimum(row + 1, rows - 1)], -np.inf)
    with np.errstate(invalid="ignore", over="ignore"):
        pb = np.exp(alpha + lpb64 + nxt_b - lP)
        pl = np.where(has_l, np.exp(alpha + lpl64 + nxt_l - lP), 0.0)
    S_b = np.abs(alpha) + np.abs(lpb64) + np.where(np.isfinite(nxt_b), np.abs(nxt_b), 0) + np.abs(lP)
    S_l = np.abs(alpha) + np.abs(lpl64) + np.where(np.isfinite(nxt_l), np.abs(nxt_l), 0) + np.abs(lP)
    pbw, plw = pb * wn, pl * wn
    dpb, dpl = grad_bound_prob(pbw, S_b), np.where(has_l, grad_bound_prob(plw, S_l), 0.0)

    live = torch.zeros(rows, dtype=torch.bool, device="cuda")
    live[row_d] = True
    dead = g[~live]
    assert not dead.view(torch.int16 if dtype != torch.float32 else torch.int32).any(), "padding rows are not exactly 0.0"
    gl = g[row_d].double()
    ref = torch.zeros(len(row), V, dtype=torch.float64, device="cuda")
    bnd = torch.zeros_like(ref)
    ar = torch.arange(len(row), device="cuda")
    pbw_d, plw_d = torch.tensor(pbw, device="cuda"), torch.tensor(plw, device="cuda")
    if from_logits:
        # grad_bound_raw: e_k = exp(x_k - lse) with the kernel's lse; the kernel computes fl(__expf(fl(x_k - l)) occ) with
        # occ = fl(pb + pl): __expf 2 + 1.173 |x| ulp plus u |x| for the argument's rounding, occ carries the two terms'
        # bounds plus u |occ|, the product rounds by u; FTZ of __expf costs 2^-126 occ
        l_d = torch.tensor(W["lse"][row].astype(np.float64), device="cuda")
        arg = xr[row_d].double() - l_d[:, None]
        e = torch.exp(arg)
        occ = pbw_d + plw_d
        docc = torch.tensor(dpb + dpl, device="cuda") + U32 * occ.abs()
        erel = ULP32 * (2 + 1.173 * arg.abs() * (1 + U32)) + U32 * arg.abs() + U32
        ref += e * occ[:, None]
        bnd += e * docc[:, None] + e * occ.abs()[:, None] * erel + 2.0 ** -126 * occ.abs()[:, None]
    ref[ar, blank] -= pbw_d
    bnd[ar, blank] += torch.tensor(dpb, device="cuda")
    hl = torch.tensor(has_l, device="cuda")
    ref[ar[hl], lab_d[hl]] -= plw_d[hl]
    bnd[ar[hl], lab_d[hl]] += torch.tensor(dpl, device="cuda")[hl]
    if from_logits:
        bnd += U32 * ref.abs() + 2.0 ** -149       # the subtraction of pb or pl
    bnd += HALF_ULP[dtype] * (ref.abs() + bnd) + HALF_SUB[dtype]
    if not from_logits:
        assert not gl[bnd == HALF_SUB[dtype]].any(), "log-prob gradient is non-zero outside blank and the label"
    err = (gl - ref).abs()
    _ratio("grad_raw" if from_logits else "grad", dtype, err.cpu().numpy(), bnd.cpu().numpy())

    _end_to_end(costs.cpu().numpy(), gl, xr, row_d, lab_d, xb32, xl32, has_l, starts, lx, ly, un, wn, V, blank,
                from_logits, dtype, dl if from_logits else None, lse64 if from_logits else None, big)
    return costs, g


def _end_to_end(c, gl, xr, row_d, lab_d, xb32, xl32, has_l, starts, lx, ly, un, wn, V, blank, from_logits, dtype, dl,
                lse64, big):
    """The costs (and, for log-probs, the gradient) against `oracle.rnnt.lattice` on the exact fp64 row terms.

    Log-probs: the lattice inputs are the same numbers, so |cost - oracle| <= lattice_bound(T + U + 1) + u |cost| (the
    fp32 rounding); pb and pl differ from the oracle's by their stage bound and by exp(3 lattice_bound) - 1 relative, from
    the alpha, beta and log P in their exponent.
    Raw logits: lpb_r = fl(x_blank - lse_kernel) is off the exact log-prob by dl_r + u |lpb_r| (lpl likewise), and
    d cost / d lpb_r = -pb_r, d cost / d lpl_r = -pl_r, so to first order |d cost| <= sum_r pb_r d_b,r + pl_r d_l,r.  cost is
    minus a log-sum-exp over paths of T + U edges each, whose second derivative along any direction D is a variance of
    path sums, at most ((T + U) max |D|)^2: the remainder is at most half that."""
    N = len(lx)
    lpb = xb32.astype(np.float64) - (lse64 if from_logits else 0.0)
    lpl = xl32.astype(np.float64) - (lse64 if from_logits else 0.0)
    pb_o, pl_o = np.empty(len(lpb)), np.zeros(len(lpb))
    for n in range(N):
        T, U = int(lx[n]), int(ly[n])
        s = slice(starts[n], starts[n + 1])
        lp, _, pb, pl = R.lattice(lpb[s].reshape(T, U + 1), lpl[s].reshape(T, U + 1)[:, :U])
        pb_o[s] = pb.reshape(-1)
        pl_o[s] = np.pad(pl, ((0, 0), (0, 1))).reshape(-1)
        latt = lattice_bound(T + U + 1, big[n])
        bound = latt + U32 * abs(float(c[n]))
        if from_logits:
            db, dlb = dl[s] + U32 * np.abs(lpb[s]), dl[s] + U32 * np.abs(lpl[s])
            first = float((pb_o[s] * db).sum() + (pl_o[s] * dlb)[has_l[s]].sum())
            bound += first + 0.5 * ((T + U) * float(max(db.max(), dlb.max()))) ** 2
        _ratio("cost_e2e_raw" if from_logits else "cost_e2e", dtype, [abs(float(c[n]) + lp)], [bound])
    if from_logits:
        return
    latt = lattice_bound(lx.numpy()[un] + ly.numpy()[un] + 1, big[un])
    rel = (1 + U32) ** 2 * np.exp(3 * latt) * (1 + 2.0 ** -51 * (big[un] * 2 + 1)) - 1
    ref = torch.zeros_like(gl)
    bnd = torch.full_like(gl, HALF_SUB[dtype])
    ar = torch.arange(len(un), device="cuda")
    pbw, plw = pb_o * wn, pl_o * wn
    ref[ar, blank] -= torch.tensor(pbw, device="cuda")
    bnd[ar, blank] += torch.tensor(rel * np.abs(pbw) * (1 + HALF_ULP[dtype]) + HALF_ULP[dtype] * np.abs(pbw) + 2.0 ** -149,
                                   device="cuda")
    hl = torch.tensor(has_l, device="cuda")
    ref[ar[hl], lab_d[hl]] -= torch.tensor(plw, device="cuda")[hl]
    bnd[ar[hl], lab_d[hl]] += torch.tensor(rel * np.abs(plw) * (1 + HALF_ULP[dtype]) + HALF_ULP[dtype] * np.abs(plw)
                                           + 2.0 ** -149, device="cuda")[hl]
    _ratio("grad_e2e", dtype, (gl - ref).abs().cpu().numpy(), bnd.cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------------
# the matrix
# ---------------------------------------------------------------------------------------------------------------------
def _blanks(V):
    return sorted({0, V - 1, V // 2})


MATRIX = [(V, b) for V in (1, 2, 4, 8, 31, 33, 37, 64, 1000, 4232) for b in _blanks(V)]


@pytest.mark.parametrize("compact", [False, True], ids=["padded", "compact"])
@pytest.mark.parametrize("V,blank", MATRIX)
def test_vocab_and_blank(V, blank, compact):
    """Every vocabulary at the chunk edges (1: blank only; 4 and 8: one 16-byte chunk; 31, 33: about one element per lane;
    37: the element path) with blank first, last and in the middle, in every dtype and input mode."""
    lx, ly = [5, 1, 3, 4], ([0, 0, 0, 0] if V == 1 else [3, 2, 0, 1])
    z, y, lx, ly = _batch(lx, ly, V, blank, seed=V * 7 + blank)
    for name, dtype in DTYPES.items():
        for fl in (False, True):
            x, yt, lxt, lyt = _inputs(z, y, lx, ly, compact, fl, dtype)
            stages(x, yt, lxt, lyt, blank, compact, fl)


SHAPES = {
    "T1_U0": ([1, 1, 2], [0, 0, 0], None, None),
    "T1_Upos": ([1, 1, 1], [3, 1, 5], None, None),
    "U0_Tpos": ([7, 3, 12], [0, 0, 0], None, None),
    "padded_far": ([3, 1, 5], [2, 0, 1], 40, 30),
    "skewed": ([150] + [2] * 9, [45] + [1] * 9, None, None),
}


@pytest.mark.parametrize("shape,compact", [(s, c) for s in sorted(SHAPES) for c in (False, True)
                                           if not (c and s == "padded_far")])
def test_edge_shapes(shape, compact):
    """T = 1 with U = 0 and U > 0, U = 0 with T > 1, Tmax and Umax far beyond every length (padding filled with NaN, never
    read), and one utterance with far more rows than the batch average, which sizes the row grid."""
    lx, ly, Tmax, Umax = SHAPES[shape]
    V, blank = 33, 16
    z, y, lx, ly = _batch(lx, ly, V, blank, seed=len(shape), Tmax=Tmax, Umax=Umax)
    for n in range(len(lx)):
        z[n, lx[n]:] = np.nan
        z[n, :, ly[n] + 1:] = np.nan
    for dtype in DTYPES.values():
        for fl in (False, True):
            x, yt, lxt, lyt = _inputs(z, y, lx, ly, compact, fl, dtype)
            stages(x, yt, lxt, lyt, blank, compact, fl)


@pytest.mark.parametrize("compact", [False, True], ids=["padded", "compact"])
def test_300_ragged(compact):
    """N = 300: the prep scan carries across two 256-utterance chunks and the grids have 301 rows of CTAs."""
    rng = np.random.default_rng(300)
    lx, ly = rng.integers(1, 13, 300), rng.integers(0, 7, 300)
    lx[255:258], ly[255:258] = [1, 12, 4], [6, 0, 3]
    z, y, lx, ly = _batch(lx, ly, 31, 30, seed=3)
    for dtype, fl in ((torch.float32, False), (torch.float32, True), (torch.bfloat16, True)):
        x, yt, lxt, lyt = _inputs(z, y, lx, ly, compact, fl, dtype)
        stages(x, yt, lxt, lyt, 30, compact, fl)


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
def test_peaky_and_shifted_rows(dtype):
    """Peaky rows (scale 15: every posterior near 0 or 1) in both modes, and raw logits shifted by +-1000 per row, where
    the logsumexp rests on the max and exp(x - lse) must not lose the shift."""
    dt = DTYPES[dtype]
    z, y, lx, ly = _batch([9, 6, 11], [4, 7, 2], 64, 3, seed=15, scale=15.0)
    for fl in (False, True):
        x, yt, lxt, lyt = _inputs(z, y, lx, ly, True, fl, dt)
        stages(x, yt, lxt, lyt, 3, True, fl)
    for V in (37, 1000):
        z, y, lx, ly = _batch([6, 4, 8], [3, 5, 2], V, 1, seed=V, shift=1000.0)
        x, yt, lxt, lyt = _inputs(z, y, lx, ly, False, True, dt)
        stages(x, yt, lxt, lyt, 1, False, True)


@pytest.mark.parametrize("fl", [False, True], ids=["logprobs", "logits"])
def test_weights(fl):
    """reduction='none' backed by weights that are zero, negative and not one: the gradient rows are w_n times the
    posteriors, and a zero weight gives zero rows."""
    w = np.array([0.0, -1.5, 0.37, 2.0, 1.0, -0.0], np.float32)
    z, y, lx, ly = _batch([4, 6, 3, 7, 2, 5], [2, 3, 1, 0, 4, 2], 40, 0, seed=77)
    for dtype in DTYPES.values():
        for compact in (False, True):
            x, yt, lxt, lyt = _inputs(z, y, lx, ly, compact, fl, dtype)
            _, g = stages(x, yt, lxt, lyt, 0, compact, fl, w=w)
            if compact:
                assert not g[:4 * 3].any()


@pytest.mark.parametrize("compact", [False, True], ids=["padded", "compact"])
def test_meta_bad_from_device_lengths(compact):
    """N = 300 with device lengths and labels that make utterances bad in every way the prep and row passes check, at
    n = 255, 256 and 257 around the scan's chunk edge: meta holds the host's offsets (negative lengths counting as 0),
    `bad` is set for exactly those utterances, their costs are NaN and their gradient rows 0; the rest are finite."""
    from cat_b200.rnnt import _forward, check_rnnt_args, rnnt_loss
    N, V, blank, Tmax, Umax = 300, 12, 3, 6, 3
    rng = np.random.default_rng(255)
    lx, ly = rng.integers(1, Tmax + 1, N).astype(np.int32), rng.integers(0, Umax + 1, N).astype(np.int32)
    ly[[10, 256]] = [2, 2]
    if compact:
        lx[255] = 0                     # no frames
        ly[257] = -1                    # negative label count: its T rows still count in the offsets
    else:
        lx[255] = Tmax + 1              # more frames than the tensor
        ly[257] = Umax + 1              # more labels than the tensor
    lx[0] = 0 if not compact else lx[0]
    own = np.maximum(lx, 0).astype(np.int64) * (np.maximum(ly, 0) + 1)
    nlab = np.maximum(ly, 0).astype(np.int64)
    loff = np.cumsum(nlab) - nlab if compact else np.arange(N) * Umax
    labels = rng.choice([k for k in range(V) if k != blank], int(nlab.sum()) if compact else (N, Umax)).astype(np.int32)
    flat = labels.reshape(-1)
    flat[loff[256]] = blank             # a label equal to blank
    flat[loff[10] + 1] = V              # a label outside [0, V)
    bad = {10, 255, 256, 257} | ({0} if not compact else set())
    if compact:
        rows = int(own.sum())
        lx[-1] += 1                     # the last utterance overruns the tensor
        own[-1] = int(lx[-1]) * (max(int(ly[-1]), 0) + 1)
        bad.add(N - 1)
        roff = np.cumsum(own) - own
        span = np.minimum(own, np.maximum(rows - roff, 0))
        ts = np.maximum(ly, 0) + 1
        tail = min(int(own.sum()), rows)
        x = torch.randn(rows, V, dtype=torch.float64).log_softmax(-1).float().cuda()
    else:
        rows = N * Tmax * (Umax + 1)
        roff = np.arange(N) * Tmax * (Umax + 1)
        span, ts, tail = np.full(N, Tmax * (Umax + 1)), np.full(N, Umax + 1), rows
        x = torch.randn(N, Tmax, Umax + 1, V, dtype=torch.float64).log_softmax(-1).float().cuda()
    dev = [torch.tensor(a).cuda() for a in (labels, lx, ly)]
    shape = check_rnnt_args(x, *dev, "none", blank, compact)
    costs, _, ws, _ = _forward(x, *dev, blank, compact, False, True, shape)
    W = read_workspace(ws.cpu().numpy(), N, rows)
    m = W["meta"]
    assert m["roff"].tolist() == roff.tolist() and m["loff"].tolist() == loff.tolist()
    assert m["span"].tolist() == span.tolist() and m["ts"].tolist() == ts.tolist()
    assert m["T"].tolist() == lx.tolist() and m["U"].tolist() == ly.tolist()
    assert set(np.flatnonzero(m["bad"]).tolist()) == bad and set(np.unique(m["bad"]).tolist()) <= {0, 1}
    assert int(W["tail"][0]) == tail
    c = costs.cpu().numpy()
    assert np.isnan(c[sorted(bad)]).all() and np.isfinite(np.delete(c, sorted(bad))).all()
    xg = x.detach().requires_grad_(True)
    (g,) = torch.autograd.grad(rnnt_loss(xg, *dev, reduction="none", blank=blank, compact=compact).nan_to_num(0.0).sum(), xg)
    g = g.reshape(rows, V)
    for n in sorted(bad):
        r0 = int(roff[n])
        assert not g[r0:r0 + int(span[n])].view(torch.int32).any(), n


# ---------------------------------------------------------------------------------------------------------------------
# pointer alignment
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("V", [8, 64, 1000])
def test_misaligned_base_pointer(V, dtype):
    """x = buf[1:].view(rows, V) with V a multiple of 8: every row is a whole number of 16-byte chunks but the base is
    aligned to 4 or 2 bytes only, so the kernels take the element path.  Log-probs: the costs and gradient are
    bit-identical to a 16-byte-aligned copy.  Raw logits: both copies within the stage bounds."""
    dt = DTYPES[dtype]
    z, y, lx, ly = _batch([5, 3, 7], [2, 4, 1], V, 2, seed=V + 1)
    for fl in (False, True):
        x, yt, lxt, lyt = _inputs(z, y, lx, ly, True, fl, dt)
        assert x.data_ptr() % 16 == 0
        buf = torch.empty(x.numel() + 1, dtype=dt, device="cuda")
        buf[1:] = x.reshape(-1)
        xm = buf[1:].view(x.shape)
        assert xm.data_ptr() % 16 == x.element_size() and xm.is_contiguous()
        ca, ga = stages(x, yt, lxt, lyt, 2, True, fl)
        cm, gm = stages(xm, yt, lxt, lyt, 2, True, fl)
        if not fl:
            assert torch.equal(ca, cm) and torch.equal(ga, gm)


# ---------------------------------------------------------------------------------------------------------------------
# poisoned allocator
# ---------------------------------------------------------------------------------------------------------------------
PATTERNS = (0xFF, 0x7F)


def _bits(t):
    t = t.detach()
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16).cpu()


@pytest.fixture
def rnnt_scratch(monkeypatch):
    import cat_b200.rnnt as M
    proxy = ScratchProxy(0)
    monkeypatch.setattr(M, "torch", proxy)
    return proxy


@pytest.mark.parametrize("compact", [False, True], ids=["padded", "compact"])
@pytest.mark.parametrize("fl", [False, True], ids=["logprobs", "logits"])
def test_poisoned_scratch(rnnt_scratch, compact, fl):
    """Every buffer of rnnt.py filled with 0x00, then 0xFF (NaN, -1), then 0x7F: the same bits out.  Device lengths make
    utterance 1 bad (a label equal to blank) and, padded, utterance 4 bad (T > Tmax); compact, they sum to 9 rows fewer
    than the tensor holds, so those tail rows are the gradient pass's to zero.  Padding, bad and tail rows are exactly 0."""
    from cat_b200 import _lib
    from cat_b200.rnnt import rnnt_costs_both_ways, rnnt_loss
    V, blank = 24, 5
    z, y, lx, ly = _batch([6, 4, 7, 3, 5], [3, 2, 4, 1, 2], V, blank, seed=9, Tmax=8, Umax=5)
    x, yt, lxt, lyt = _inputs(z, y, lx, ly, compact, fl, torch.float32)
    yt = yt.clone()
    if compact:
        yt[int(ly[0])] = blank
        x = torch.cat([x, torch.randn(9, V, device="cuda")])
    else:
        yt[1, 0] = blank
        lxt = lxt.clone()
        lxt[4] = 9
    bad = [1] if compact else [1, 4]
    N, rows = len(lx), x.shape[0] if compact else x[..., 0].numel()
    w = torch.tensor([0.5, 1.0, -2.0, 1.5, 0.25], device="cuda")
    dev = [t.cuda() for t in (yt, lxt, lyt)]

    def run():
        xg = x.detach().clone().requires_grad_(True)
        c = rnnt_loss(xg, *dev, reduction="none", blank=blank, compact=compact, from_logits=fl)
        (g,) = torch.autograd.grad((c * w).nan_to_num(0.0).sum(), xg)
        with torch.no_grad():
            c_eval = rnnt_loss(x, *dev, reduction="none", blank=blank, compact=compact, from_logits=fl)
        a, b = rnnt_costs_both_ways(x, *dev, blank=blank, compact=compact, from_logits=fl)
        return dict(c=c, g=g, c_eval=c_eval, a=a, b=b)

    rnnt_scratch.byte = 0
    del rnnt_scratch.record[:]
    clean = {k: _bits(v) for k, v in run().items()}
    seen = {nb for nb, _, d in rnnt_scratch.record if d.type == "cuda"}
    assert int(_lib.lib().ccb_rnnt_workspace_bytes(N, rows)) in seen, sorted(seen)
    costs = clean["c"].view(torch.float32)
    assert torch.isnan(costs[bad]).all() and torch.isfinite(costs[[n for n in range(N) if n not in bad]]).all()
    g = clean["g"].reshape(rows, V)
    keep = torch.zeros(rows, dtype=torch.bool)
    if compact:
        o = 0
        for n in range(N):
            r = int(lx[n]) * (int(ly[n]) + 1)
            keep[o:o + r] = n not in bad
            o += r
        assert o == rows - 9
    else:
        for n in range(N):
            if n not in bad:
                keep.view(N, 8, 6)[n, :lx[n], :ly[n] + 1] = True
    assert not g[~keep].any() and g[keep].any()
    for byte in PATTERNS:
        rnnt_scratch.byte = byte
        got = {k: _bits(v) for k, v in run().items()}
        for k in clean:
            assert torch.equal(got[k], clean[k]), (hex(byte), k)
    rnnt_scratch.byte = 0


@pytest.mark.parametrize("host", [True, False], ids=["host_lengths", "device_lengths"])
def test_poisoned_gather_sum(rnnt_scratch, host):
    import gather
    N, H = 7, 300
    la = torch.tensor([3, 0, 5, 2, 4, 1, 6])
    lb = torch.tensor([2, 4, 0, 3, 1, 5, 2])
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randn(int(la.sum()), H, device="cuda", generator=g)
    b = torch.randn(int(lb.sum()), H, device="cuda", generator=g)
    go = torch.randn(int((la * lb).sum()), H, device="cuda", generator=g)
    lens = (la, lb) if host else (la.cuda(), lb.cuda())

    def run():
        aa, bb = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        out = gather.sum(aa, bb, *lens)
        ga, gb = torch.autograd.grad(out, (aa, bb), go)
        return dict(out=out, ga=ga, gb=gb)

    rnnt_scratch.byte = 0
    del rnnt_scratch.record[:]
    clean = {k: _bits(v) for k, v in run().items()}
    from cat_b200 import _lib
    assert int(_lib.lib().ccb_gather_ws_bytes(N)) in {nb for nb, _, d in rnnt_scratch.record if d.type == "cuda"}
    for byte in PATTERNS:
        rnnt_scratch.byte = byte
        got = {k: _bits(v) for k, v in run().items()}
        for k in clean:
            assert torch.equal(got[k], clean[k]), (hex(byte), k)
    rnnt_scratch.byte = 0
    # utterance 1 has no a rows and utterance 2 no b rows: their other side's gradient rows are sums of nothing
    assert not clean["gb"].view(torch.float32)[2:6].any()
    assert not clean["ga"].view(torch.float32)[3:8].any()


# ---------------------------------------------------------------------------------------------------------------------
# an infeasible utterance
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("compact", [False, True], ids=["padded", "compact"])
@pytest.mark.parametrize("fl", [False, True], ids=["logprobs", "logits"])
def test_infeasible_utterance_leaves_others_alone(compact, fl):
    """The final blank of utterance 2 at -inf: its cost is +inf, and every other utterance's cost and gradient rows are
    bit-identical to the same batch without it."""
    from cat_b200.rnnt import rnnt_loss
    z, y, lx, ly = _batch([5, 4, 6, 3], [2, 3, 2, 1], 29, 0, seed=21)
    if not fl:
        z = z - np.logaddexp.reduce(z, axis=-1, keepdims=True)
    z2 = z.copy()
    z2[2, lx[2] - 1, ly[2], 0] = -np.inf
    out = []
    for zz in (z, z2):
        x, yt, lxt, lyt = _inputs(zz, y, lx, ly, compact, True, torch.float32)   # zz already in the wanted mode
        xg = x.requires_grad_(True)
        c = rnnt_loss(xg, yt, lxt, lyt, reduction="none", compact=compact, from_logits=fl)
        (g,) = torch.autograd.grad(c.sum(), xg)
        out.append((c.detach().cpu(), g.cpu()))
    (c1, g1), (c2, g2) = out
    assert c2[2] == float("inf")
    others = [0, 1, 3]
    assert torch.equal(c1[others], c2[others])
    if compact:
        blocks = np.cumsum([0] + [int(lx[n]) * (int(ly[n]) + 1) for n in range(4)])
        for n in others:
            assert torch.equal(g1[blocks[n]:blocks[n + 1]], g2[blocks[n]:blocks[n + 1]])
    else:
        assert torch.equal(g1[others], g2[others])


# ---------------------------------------------------------------------------------------------------------------------
# no host synchronisation
# ---------------------------------------------------------------------------------------------------------------------
def test_no_host_synchronisation():
    """rnnt_loss forward and backward with host and with device lengths and labels, and gather.sum with CPU lengths, run
    under torch.cuda.set_sync_debug_mode('error') after a warm-up: none of them waits for the device."""
    import gather
    from cat_b200.rnnt import rnnt_loss
    z, y, lx, ly = _batch([6, 4, 7], [3, 2, 4], 32, 0, seed=5)
    calls = []
    for fl in (False, True):
        x, yt, lxt, lyt = _inputs(z, y, lx, ly, True, fl, torch.float16)
        for lens in ((yt, lxt, lyt), tuple(t.cuda() for t in (yt, lxt, lyt))):
            calls.append((x, lens, fl))
    la, lb = torch.tensor([3, 0, 5, 2]), torch.tensor([2, 4, 1, 3])
    a = torch.randn(10, 64, device="cuda", requires_grad=True)
    b = torch.randn(10, 64, device="cuda", requires_grad=True)

    def work():
        for x, lens, fl in calls:
            xg = x.detach().requires_grad_(True)
            loss = rnnt_loss(xg, *lens, compact=True, from_logits=fl)
            loss.backward()
            with torch.no_grad():
                rnnt_loss(x, *lens, reduction="none", compact=True, from_logits=fl)
        gather.sum(a, b, la, lb).sum().backward()

    for _ in range(6):                 # more calls than the staging ring has slots
        work()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(6):
            work()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# gather.sum against fp64
# ---------------------------------------------------------------------------------------------------------------------
GATHER = [(300, H) for H in (1, 31, 33, 256, 257, 640, 1024)] + [(1, 257), (1, 1024), (257, 33), (257, 640)]


@pytest.mark.parametrize("N,H", GATHER)
def test_gather_sum_fp64(N, H):
    """The forward is bit-equal to torch's broadcast sum; each backward element is a fixed-order fp32 sum of k terms
    (k = lb_n for a row of a, la_n for a row of b), so within gamma_k sum |g| of the fp64 sum, plus half an ulp of the
    dtype.  Lengths include la = 0, lb = 0 and one la of 2000; N = 257 and 300 carry the offset scans across 256-utterance
    chunks, H = 257 and up loop h past one CTA."""
    import gather
    rng = np.random.default_rng(N * 1000 + H)
    la, lb = rng.integers(0, 12, N), rng.integers(0, 8, N)
    la[0], lb[0] = 2000, max(int(lb[0]), 3)
    if N > 2:
        la[1], lb[2] = 0, 0
    la_t, lb_t = torch.tensor(la), torch.tensor(lb)
    ia = np.concatenate([np.repeat(np.arange(a0, a0 + a), b) for a0, a, b in zip(np.cumsum(la) - la, la, lb)])
    ib = np.concatenate([np.tile(np.arange(b0, b0 + b), a) for b0, a, b in zip(np.cumsum(lb) - lb, la, lb)])
    ia_d, ib_d = torch.tensor(ia, device="cuda"), torch.tensor(ib, device="cuda")
    for dtype in DTYPES.values():
        g = torch.Generator(device="cuda").manual_seed(H)
        a = torch.randn(int(la.sum()), H, device="cuda", generator=g).to(dtype).requires_grad_(True)
        b = torch.randn(int(lb.sum()), H, device="cuda", generator=g).to(dtype).requires_grad_(True)
        for lens in ((la_t, lb_t), (la_t.cuda(), lb_t.cuda())):
            out = gather.sum(a, b, *lens)
            assert out.dtype == dtype and torch.equal(out, a.detach()[ia_d] + b.detach()[ib_d])
        go = torch.randn(out.shape, device="cuda", generator=g).to(dtype)
        ga, gb = torch.autograd.grad(out, (a, b), go)
        gd = go.double()
        for grad, idx, k_of, n in ((ga, ia_d, lb, a.shape[0]), (gb, ib_d, la, b.shape[0])):
            ref = torch.zeros(n, H, dtype=torch.float64, device="cuda").index_add_(0, idx, gd)
            mag = torch.zeros(n, H, dtype=torch.float64, device="cuda").index_add_(0, idx, gd.abs())
            k = torch.tensor(np.repeat(k_of, la if grad is ga else lb), dtype=torch.float64, device="cuda")[:, None]
            gam = k * U32 / (1 - k * U32)
            bound = gam * mag + HALF_ULP[dtype] * (ref.abs() + gam * mag) + HALF_SUB[dtype]
            _ratio("gather_bwd", dtype, (grad.double() - ref).abs().cpu().numpy(), bound.cpu().numpy())
