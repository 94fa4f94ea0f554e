"""Test infrastructure, not product code: an fp64 numpy restatement of the RNN-T loss of ``cat_b200.rnnt.rnnt_loss``
(DESIGN.md §7 "RNN-T loss"), the yardstick the CPU and GPU tests compare against.  It is checked against
``torchaudio.functional.rnnt_loss`` in tests/test_rnnt_dispatch.py.

Utterance n has T frames, U labels y_1..y_U, and per row (t, u) the log-probs lpb(t,u) of blank and lpl(t,u) of y_{u+1}:
    alpha(0,0) = 0,  alpha(t,u) = logaddexp(alpha(t-1,u) + lpb(t-1,u), alpha(t,u-1) + lpl(t,u-1)),
    log P = alpha(T-1,U) + lpb(T-1,U),  cost = -log P.
The posteriors of the blank and label transitions out of (t,u) are pb and pl; the gradient of the cost with respect to
log-prob input is -pb at blank and -pl at y_{u+1}; with respect to raw logits it is softmax (pb + pl) minus the same terms.
"""
from __future__ import annotations

import numpy as np


def cells(lpb: np.ndarray, lpl: np.ndarray):
    """lpb (T, U+1), lpl (T, U) in fp64.  Returns the lattice cells (alpha, beta), each (T, U+1)."""
    lpb = np.asarray(lpb, np.float64)
    lpl = np.asarray(lpl, np.float64).reshape(lpb.shape[0], lpb.shape[1] - 1)
    T, U1 = lpb.shape
    U = U1 - 1
    alpha = np.full((T, U1), -np.inf)
    beta = np.full((T, U1), -np.inf)
    alpha[0, 0] = 0.0
    lplp = np.concatenate([lpl, np.full((T, 1), -np.inf)], 1)     # lpl with a column of -inf at u = U
    with np.errstate(invalid="ignore"):
        for d in range(1, T + U):       # anti-diagonals t + u = d
            u = np.arange(max(0, d - T + 1), min(U, d) + 1)
            t = d - u
            a1 = np.where(t > 0, alpha[np.maximum(t - 1, 0), u] + lpb[np.maximum(t - 1, 0), u], -np.inf)
            a2 = np.where(u > 0, alpha[t, np.maximum(u - 1, 0)] + lplp[t, np.maximum(u - 1, 0)], -np.inf)
            alpha[t, u] = np.logaddexp(a1, a2)
        beta[T - 1, U] = lpb[T - 1, U]
        for d in range(1, T + U):       # (T-1-t) + (U-u) = d
            k = np.arange(max(0, d - T + 1), min(U, d) + 1)
            u = U - k
            t = T - 1 - (d - k)
            b1 = np.where(t < T - 1, beta[np.minimum(t + 1, T - 1), u] + lpb[t, u], -np.inf)
            b2 = np.where(u < U, beta[t, np.minimum(u + 1, U)] + lplp[t, u], -np.inf)
            beta[t, u] = np.logaddexp(b1, b2)
    return alpha, beta


def lattice(lpb: np.ndarray, lpl: np.ndarray):
    """lpb (T, U+1), lpl (T, U) in fp64.  Returns (log P, log P from beta, pb (T, U+1), pl (T, U))."""
    lpb = np.asarray(lpb, np.float64)
    lpl = np.asarray(lpl, np.float64).reshape(lpb.shape[0], lpb.shape[1] - 1)
    T, U1 = lpb.shape
    U = U1 - 1
    alpha, beta = cells(lpb, lpl)
    with np.errstate(invalid="ignore"):
        logp = alpha[T - 1, U] + lpb[T - 1, U]
        nxt = np.full((T, U1), -np.inf)
        nxt[:-1] = beta[1:]
        nxt[T - 1, U] = 0.0
        pb = np.exp(alpha + lpb + nxt - logp)
        pl = np.exp(alpha[:, :U] + lpl + beta[:, 1:] - logp) if U else np.zeros((T, 0))
    return logp, beta[0, 0], pb, pl


def _blocks(x, labels, lx, ly, compact):
    """(row index array (T, U+1), labels (U,)) per utterance, in either layout."""
    off = loff = 0
    for n, (T, U) in enumerate(zip(np.asarray(lx).tolist(), np.asarray(ly).tolist())):
        if compact:
            rows = off + np.arange(T * (U + 1)).reshape(T, U + 1)
            y = np.asarray(labels[loff:loff + U])
            off += T * (U + 1)
            loff += U
        else:
            Tmax, U1 = x.shape[1], x.shape[2]
            rows = n * Tmax * U1 + (np.arange(T)[:, None] * U1 + np.arange(U + 1)[None, :])
            y = np.asarray(labels[n, :U])
        yield rows, y.astype(np.int64)


def rnnt_loss(x, labels, lx, ly, blank=0, compact=False, from_logits=False):
    """The costs (N,) and the gradient of sum_n cost_n with respect to x (x's shape, fp64; zero outside the utterances)."""
    xf = np.asarray(x, np.float64)
    V = xf.shape[-1]
    flat = xf.reshape(-1, V)
    grad = np.zeros_like(flat)
    costs = []
    for rows, y in _blocks(xf, np.asarray(labels), lx, ly, compact):
        z = flat[rows]                                  # (T, U+1, V)
        if from_logits:
            m = z.max(-1, keepdims=True)
            lse = m + np.log(np.exp(z - m).sum(-1, keepdims=True))
            lp = z - lse
        else:
            lp = z
        T, U1 = rows.shape
        lpb = lp[:, :, blank]
        lpl = np.take_along_axis(lp[:, :U1 - 1], np.broadcast_to(y[None, :, None], (T, U1 - 1, 1)), -1)[..., 0]
        logp, _, pb, pl = lattice(lpb, lpl)
        costs.append(-logp)
        g = np.exp(lp) * (pb + np.pad(pl, ((0, 0), (0, 1))))[..., None] if from_logits else np.zeros_like(lp)
        g[:, :, blank] -= pb
        tt, uu = np.meshgrid(np.arange(T), np.arange(U1 - 1), indexing="ij")
        g[tt, uu, np.broadcast_to(y[None, :], (T, U1 - 1))] -= pl
        grad[rows] = g
    return np.array(costs), grad.reshape(xf.shape)
