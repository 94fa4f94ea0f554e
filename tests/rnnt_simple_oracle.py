"""Test infrastructure: an fp64 numpy restatement of the RNN-T loss of CAT's LogAdd joiner
(``cat_b200.rnnt_simple.rnnt_loss_simple``, DESIGN.md §7 "RNN-T loss, LogAdd joiner") on top of ``oracle.rnnt.lattice``.

For one utterance with encoder rows f (T, V), predictor rows g (U+1, V) and labels y (U,):
    lp(t,u,k) = log_softmax_k(f[t] + g[u]),  lpb = lp(., ., blank),  lpl(t,u) = lp(t, u, y_{u+1}),
the cost is the RNN-T cost over these cells, and with occ = pb + pl and soft = exp(lp),
    d cost / d f[t,k] = sum_u occ soft - [k = blank] sum_u pb - sum_u pl [k = y_{u+1}],
    d cost / d g[u,k] = sum_t occ soft - [k = blank] sum_t pb - [k = y_{u+1}] sum_t pl.
"""
from __future__ import annotations

import numpy as np

from oracle import rnnt as R


def simple(f, g, y, blank=0):
    """f (T, V), g (U+1, V), y (U,).  Returns (log P, d cost / d f (T, V), d cost / d g (U+1, V)), all fp64."""
    f = np.asarray(f, np.float64)
    g = np.asarray(g, np.float64)
    y = np.asarray(y, np.int64)
    T, U1 = f.shape[0], g.shape[0]
    U = U1 - 1
    z = f[:, None, :] + g[None, :, :]
    with np.errstate(invalid="ignore", divide="ignore"):
        m = z.max(-1, keepdims=True)
        m = np.where(np.isfinite(m), m, 0.0)
        lp = z - (m + np.log(np.exp(z - m).sum(-1, keepdims=True)))
    lpb = lp[:, :, blank]
    lpl = np.take_along_axis(lp[:, :U], np.broadcast_to(y[None, :, None], (T, U, 1)), -1)[..., 0]
    logp, _, pb, pl = R.lattice(lpb, lpl)
    occ = pb + np.pad(pl, ((0, 0), (0, 1)))
    G = np.exp(lp) * occ[..., None]
    G[:, :, blank] -= pb
    tt, uu = np.meshgrid(np.arange(T), np.arange(U), indexing="ij")
    G[tt, uu, np.broadcast_to(y[None, :], (T, U))] -= pl
    return logp, G.sum(1), G.sum(0)


def batch(f, g, labels, lx, ly, blank=0):
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
