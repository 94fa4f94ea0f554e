"""TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

ctypes front-end of ``liboracle.so`` (fp64 CPU restatement, ``ctc_crf_oracle.c``) and of
``_ref/libctc_crf_ref.so`` (the unmodified reference CUDA sources built for sm_90a).
Importers allowed: tests/, __graft_entry__.smoke(), bench.py's cpu_baseline / --impl reference.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force: bool = False) -> None:
    """Compile the checkers (``make -C oracle``).  Building the checker is not using it."""
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "ctc_crf_oracle.c")
    stale = (not os.path.exists(so)) or os.path.getmtime(so) < os.path.getmtime(src)
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "liboracle.so"], stdout=subprocess.DEVNULL)
    # the reference CUDA builds under _ref/ (oracle/Makefile finds the reference sources, or keeps what _ref/ holds)
    subprocess.check_call(["make", "-C", _HERE, "ref"], stdout=subprocess.DEVNULL)
    # the reference's own binding.cpp linked against this repository's library (tests/test_ref_binding.py)
    if os.path.exists(os.path.join(_HERE, "..", "cat_b200", "libctc_crf_b200.so")):
        subprocess.check_call(["make", "-C", _HERE, "ref_binding"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


def lib():
    global _LIB
    if _LIB is None:
        build()
        _LIB = C.CDLL(os.path.join(_HERE, "liboracle.so"))
        _LIB.oracle_assemble.restype = C.c_double
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def den(graph, y: np.ndarray, lens, nthreads: int = 0, fast: bool = False):
    """Denominator forward-backward.  y: (N,T,V) float32 log-probs.
    Returns (logz_alpha[N], logz_beta[N], gamma_den[N,T,V]) in float64.
    fast: the fp64 scaled-linear evaluation (oracle_den_linear, pinned against the log-domain restatement by
    tests/test_oracle.py) -- seconds instead of minutes per utterance at the benchmark sizes."""
    y = np.ascontiguousarray(y, dtype=np.float32)
    N, T, V = y.shape
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    src, dst, lab, lw = graph.log_arcs()
    assert lab.min() >= 0 and lab.max() < V, "den graph label out of range for these logits"
    sw, ew = graph.start_weight(), graph.end_weight()
    la = np.zeros(N, np.float64)
    lb = np.zeros(N, np.float64)
    g = np.zeros((N, T, V), np.float64)
    nt = nthreads or os.cpu_count()
    fn = lib().oracle_den_linear if fast else lib().oracle_den
    rc = fn(C.c_int(graph.num_states), C.c_long(graph.num_arcs),
            _p(src, C.c_int), _p(dst, C.c_int), _p(lab, C.c_int), _p(lw, C.c_float),
            _p(sw, C.c_float), _p(ew, C.c_float), _p(y, C.c_float),
            C.c_long(T * V), C.c_long(V), C.c_int(N), C.c_int(T), C.c_int(V),
            _p(lens, C.c_int), _p(la, C.c_double), _p(lb, C.c_double),
            _p(g, C.c_double), C.c_int(nt))
    assert rc == 0, f"oracle_den failed ({rc})"
    return la, lb, g


def ctc(y: np.ndarray, labels, label_lens, lens, blank: int = 0, nthreads: int = 0, want_grad=True):
    """Numerator CTC forward-backward on log-probs y (N,T,V).
    Returns (logp[N], gamma_ctc[N,T,V]) float64 (gamma None if not want_grad)."""
    y = np.ascontiguousarray(y, dtype=np.float32)
    N, T, V = y.shape
    labels = np.ascontiguousarray(labels, dtype=np.int32)
    label_lens = np.ascontiguousarray(label_lens, dtype=np.int32)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    assert labels.shape[0] == int(label_lens.sum())
    lp = np.zeros(N, np.float64)
    g = np.zeros((N, T, V), np.float64) if want_grad else None
    nt = nthreads or os.cpu_count()
    rc = lib().oracle_ctc(_p(y, C.c_float), C.c_long(T * V), C.c_long(V), C.c_int(N), C.c_int(V),
                          _p(labels, C.c_int), _p(label_lens, C.c_int), _p(lens, C.c_int),
                          C.c_int(blank), _p(lp, C.c_double),
                          _p(g, C.c_double) if want_grad else None, C.c_int(nt))
    assert rc == 0, f"oracle_ctc failed ({rc})"
    return lp, g


def ctc_crf(graph, y, labels, lx, ly, lamb: float = 0.1, size_average: bool = True, nthreads: int = 0,
            fast: bool = False):
    """Full loss: returns (loss, grad[N,T,V], parts) following ctc_crf/__init__.py:58-90."""
    y = np.ascontiguousarray(y, dtype=np.float32)
    N = y.shape[0]
    la, lb, gden = den(graph, y, lx, nthreads, fast=fast)
    lp, gctc = ctc(y, labels, ly, lx, 0, nthreads)
    grad = gden.copy()
    loss = lib().oracle_assemble(C.c_int(N), C.c_long(grad.size), _p(la, C.c_double), _p(lp, C.c_double),
                                 _p(grad, C.c_double), _p(gctc, C.c_double), C.c_double(lamb),
                                 C.c_int(1 if size_average else 0))
    return float(loss), grad, dict(logz_alpha=la, logz_beta=lb, logp_ctc=lp, gamma_den=gden, gamma_ctc=gctc)


def ctc_crf_from_logits(graph, z, labels, lx, ly, lamb: float = 0.1, size_average: bool = True, nthreads: int = 0):
    """The loss on RAW encoder outputs z (N,T,V), as cat/ctc/train.py:173-174,184-190 composes it:
    y = log_softmax(z) (fp64 here), loss = ctc_crf(y), d loss / d z = g - softmax(z) * sum_k g_k  (g = d loss / d y)."""
    z64 = np.asarray(z, np.float64)
    lse = z64.max(-1, keepdims=True) + np.log(np.exp(z64 - z64.max(-1, keepdims=True)).sum(-1, keepdims=True))
    y64 = z64 - lse
    loss, g, parts = ctc_crf(graph, y64.astype(np.float32), labels, lx, ly, lamb, size_average, nthreads)
    dz = g - np.exp(y64) * g.sum(-1, keepdims=True)
    return loss, dz, parts


# ---------------------------------------------------------------------------------------------
# synthetic inputs (SURVEY.md 8d) shared by tests and bench
# ---------------------------------------------------------------------------------------------
def synth_batch(N, T, V, seed=1234, lens=None, max_label=400, scale=3.0):
    rng = np.random.default_rng(seed)
    x = (scale * rng.standard_normal((N, T, V))).astype(np.float32)
    x = x - x.max(-1, keepdims=True)
    y = (x - np.log(np.exp(x.astype(np.float64)).sum(-1, keepdims=True))).astype(np.float32)
    lens = np.full(N, T, np.int32) if lens is None else np.asarray(lens, np.int32)
    ly = np.minimum(lens // 6, max_label).astype(np.int32)
    labels = rng.integers(1, V, size=int(ly.sum())).astype(np.int32)
    return y, labels, lens, ly
