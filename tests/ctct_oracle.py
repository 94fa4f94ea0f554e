"""Test infrastructure: an fp64 numpy restatement of the CTC-T loss (``cat_b200.ctct``, DESIGN.md §7 "CTC-T loss"), written
from its definition, in both layouts and both input modes, and of the LogAdd joiner's CTC-T loss.

Utterance n has T frames, labels y_1..y_U and per row (t, u) the log-probs lp(t,u,k).  States: (u, b) (u labels emitted, the
last emission blank or none yet) and (u, l) (the last emission y_u).  With (+) logaddexp, alpha_0(0,b) = 0 and every other
alpha_0 = -inf:
    alpha_{t+1}(u,b) = [alpha_t(u,b) (+) alpha_t(u,l)] + lp(t,u,blank)
    alpha_{t+1}(u,l) = [alpha_t(u,l) + lp(t,u,y_u)] (+) [alpha_t(u-1,b) + lp(t,u-1,y_u)]
                       (+) [alpha_t(u-1,l) + lp(t,u-1,y_u)]   (only if u = 1 or y_u != y_{u-1})
    log P = alpha_T(U,b) (+) alpha_T(U,l).
The transitions that read row (t,u) are blank (pb), the repeat of y_u (pr, u >= 1) and the new label y_{u+1} (pl, u < U);
the gradient of the cost with respect to log-prob input is -pb at blank, -pr at y_u and -pl at y_{u+1} (added where
y_u = y_{u+1}); with respect to raw logits, softmax (pb + pr + pl) minus the same terms.  log P = -inf (no path): cost +inf
and zero posteriors.
"""
from __future__ import annotations

import numpy as np

from oracle.rnnt import _blocks

NEG = -np.inf


def lattice(lpb, lpl, lpr, y):
    """lpb (T, U+1), lpl (T, U) = lp(t, u, y_{u+1}), lpr (T, U) = lp(t, u+1, y_{u+1}) (the repeat read at row u+1), y (U,).
    Returns (log P, log P from beta, pb, pr, pl), the posteriors each (T, U+1): pr is 0 at u = 0, pl at u = U."""
    lpb = np.asarray(lpb, np.float64)
    T, U1 = lpb.shape
    U = U1 - 1
    y = np.asarray(y, np.int64)
    lpl = np.concatenate([np.asarray(lpl, np.float64).reshape(T, U), np.full((T, 1), NEG)], 1)    # column u: y_{u+1}
    lpr = np.concatenate([np.full((T, 1), NEG), np.asarray(lpr, np.float64).reshape(T, U)], 1)    # column u: y_u
    # skip[u] (u >= 1): the new label y_u may come from (u-1, l)
    skip = np.array([u == 1 or (u >= 2 and y[u - 1] != y[u - 2]) for u in range(U1)])
    Ab, Al = np.full((T + 1, U1), NEG), np.full((T + 1, U1), NEG)
    Bb, Bl = np.full((T + 1, U1), NEG), np.full((T + 1, U1), NEG)
    Ab[0, 0] = 0.0
    Bb[T, U] = 0.0
    if U:
        Bl[T, U] = 0.0
    with np.errstate(invalid="ignore"):
        for t in range(T):
            Ab[t + 1] = np.logaddexp(Ab[t], Al[t]) + lpb[t]
            src = np.where(skip[1:], np.logaddexp(Ab[t, :-1], Al[t, :-1]), Ab[t, :-1])
            Al[t + 1, 1:] = np.logaddexp(Al[t, 1:] + lpr[t, 1:], src + lpl[t, :-1])
        for t in range(T - 1, -1, -1):
            xb = Bb[t + 1] + lpb[t]
            xn = np.append(Bl[t + 1, 1:] + lpl[t, :-1], NEG)                 # new label y_{u+1}, into (u+1, l)
            Bb[t] = np.logaddexp(xb, xn)
            xn_l = np.where(np.append(skip[1:], False), xn, NEG)              # from (u, l) only if y_{u+1} != y_u
            Bl[t] = np.logaddexp(np.logaddexp(xb, Bl[t + 1] + lpr[t]), xn_l)
            Bl[t, 0] = NEG
        logp = np.logaddexp(Ab[T, U], Al[T, U])
        if logp == NEG:
            z = np.zeros((T, U1))
            return logp, Bb[0, 0], z, z.copy(), z.copy()
        a = np.logaddexp(Ab[:T], Al[:T])
        pb = np.exp(a + lpb + Bb[1:] - logp)
        pr = np.exp(Al[:T] + lpr + Bl[1:] - logp)
        src = np.where(np.append(skip[1:], False)[None, :], a, Ab[:T])
        nxt = np.concatenate([Bl[1:, 1:], np.full((T, 1), NEG)], 1)
        pl = np.exp(src + lpl + nxt - logp)
    return logp, Bb[0, 0], pb, pr, pl


def utterance(lp, y, blank=0):
    """lp (T, U+1, V) log-probs, y (U,).  Returns (log P, log P from beta, d cost / d lp (T, U+1, V), pb + pr + pl
    (T, U+1))."""
    lp = np.asarray(lp, np.float64)
    T, U1, V = lp.shape
    U = U1 - 1
    y = np.asarray(y, np.int64)
    tt = np.arange(T)[:, None]
    lpb = lp[:, :, blank]
    lpl = lp[tt, np.arange(U)[None, :], y[None, :]]                 # row u, label y_{u+1}
    lpr = lp[tt, np.arange(1, U1)[None, :], y[None, :]]             # row u+1, label y_{u+1}
    logp, logp_b, pb, pr, pl = lattice(lpb, lpl, lpr, y)
    g = np.zeros_like(lp)
    g[:, :, blank] -= pb
    if U:
        g[tt, np.arange(1, U1)[None, :], y[None, :]] -= pr[:, 1:]
        g[tt, np.arange(U)[None, :], y[None, :]] -= pl[:, :U]
    return logp, logp_b, g, pb + pr + pl


def ctct_loss(x, labels, lx, ly, blank=0, compact=False, from_logits=False):
    """The costs (N,) and the gradient of sum_n cost_n with respect to x (x's shape, fp64; zero outside the utterances)."""
    xf = np.asarray(x, np.float64)
    V = xf.shape[-1]
    flat = xf.reshape(-1, V)
    grad = np.zeros_like(flat)
    costs = []
    for rows, y in _blocks(xf, np.asarray(labels), lx, ly, compact):
        z = flat[rows]
        if from_logits:
            m = z.max(-1, keepdims=True)
            lp = z - (m + np.log(np.exp(z - m).sum(-1, keepdims=True)))
        else:
            lp = z
        logp, _, g, occ = utterance(lp, y, blank)
        costs.append(-logp)
        if from_logits:
            g = g + np.exp(lp) * occ[..., None]
        grad[rows] = g
    return np.array(costs), grad.reshape(xf.shape)


def simple(f, g, y, blank=0):
    """The LogAdd joiner: f (T, V), g (U+1, V), y (U,).  Returns (log P, d cost / d f (T, V), d cost / d g (U+1, V))."""
    f = np.asarray(f, np.float64)
    g = np.asarray(g, np.float64)
    z = f[:, None, :] + g[None, :, :]
    with np.errstate(invalid="ignore", divide="ignore"):
        m = z.max(-1, keepdims=True)
        m = np.where(np.isfinite(m), m, 0.0)
        lp = z - (m + np.log(np.exp(z - m).sum(-1, keepdims=True)))
    logp, _, G, occ = utterance(lp, y, blank)
    G = G + np.exp(lp) * occ[..., None]
    return logp, G.sum(1), G.sum(0)


def simple_batch(f, g, labels, lx, ly, blank=0):
    """The padded batch: f (N, Tmax, V), g (N, Umax+1, V), labels (N, Umax).  Returns costs (N,) and the gradients of
    sum_n cost_n with respect to f and g, zero outside the utterances."""
    f = np.asarray(f, np.float64)
    g = np.asarray(g, np.float64)
    costs, gf, gg = [], np.zeros_like(f), np.zeros_like(g)
    for n, (T, U) in enumerate(zip(np.asarray(lx).tolist(), np.asarray(ly).tolist())):
        lp, df, dg = simple(f[n, :T], g[n, :U + 1], np.asarray(labels)[n, :U], blank)
        costs.append(-lp)
        gf[n, :T], gg[n, :U + 1] = df, dg
    return np.array(costs), gf, gg
