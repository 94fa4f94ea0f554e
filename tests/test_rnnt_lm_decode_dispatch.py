"""CPU: the restatements of the RNN-T beam search with LM fusion and ILM estimation (tests/rnnt_fusion_oracle.py) against
each other, the search without fusion and exhaustive enumeration; the dense-chain n-gram rows against the textbook
scorer; the constructor and argument checks of ``cat_b200.rnnt_decode`` (raised before any native call) and of the new
C ABI entries."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from cat_b200 import _lib, rnnt_decode
from cat_b200.ngram import NGramLM, make_random_arpa
from cat_b200.rnnt_decode import RNNTDecoder, rnnt_beam_search
from rnnt_decode_oracle import LogAdd, LSTMPredictor, beam_ref, exhaustive, module_lp
from rnnt_fusion_oracle import (CatNGram, JointNet, LSTMLM, beam_ref_fused, cat_decode_fused, fuse_term,
                                ngram_rows_dense, prefix_ilm, prefix_lm)
from test_ngram_dispatch import CASES, LN10, Textbook, Walk, cat_labels


def _labels(V):
    return ["<blk>", "<unk>"] + [str(i) for i in range(2, V)]


def _setup(V=7, H=6, seed=0, mode="add"):
    torch.manual_seed(seed)
    pred = LSTMPredictor(V, H).double()
    joiner = JointNet(H, H, V, 8, mode).double()
    for m in (pred, joiner):
        for p in m.parameters():
            p.data.mul_(3.0)
    return pred, joiner


def _agree(got, ref, tol=1e-9):
    assert len(got) == len(ref)
    for (gh, gs), (rh, rs) in zip(got, ref):
        assert gh == rh
        for a, b in zip(gs, rs):
            assert abs(a - b) <= tol * (1 + abs(b)), (a, b)


def _lm(kind, tmp_path, V):
    if kind == "lstm":
        torch.manual_seed(3)
        lm = LSTMLM(V, 5).double()
        for p in lm.parameters():
            p.data.mul_(3.0)
        return lm
    order = int(kind[-1])
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, order, [3 * V] * (order - 1), seed=order)
    return CatNGram(path, _labels(V))


@pytest.mark.parametrize("lm_kind, alpha, beta, w", [
    ("ngram2", 0.7, 0.5, 0.0), ("ngram3", 0.4, -0.2, 0.0), ("ngram5", 1.3, 0.8, 0.0), ("lstm", 0.6, 0.3, 0.0),
    (None, 0.0, 0.0, 0.35), ("ngram3", 0.28125, 0.5, -0.3125), ("lstm", 0.5, 0.0, -0.4),
])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_cat_restatement_matches_beam_ref_fused(lm_kind, alpha, beta, w, B, tmp_path):
    V, T = 7, 5
    pred, joiner = _setup(V)
    lm = _lm(lm_kind, tmp_path, V) if lm_kind else None
    torch.manual_seed(1)
    enc = torch.randn(2, T, 6, dtype=torch.float64) * 2
    lens = torch.tensor([T, 3])
    got = cat_decode_fused(enc, lens, pred, joiner, B, lm=lm, alpha=alpha, beta=beta, ilm_weight=w)
    lmrow = prefix_lm(lm) if lm is not None else None
    ilm = prefix_ilm(pred, joiner, 6) if w else None

    def term(t, p):
        return fuse_term(lmrow(p) if lmrow else None, ilm(p) if ilm else None, alpha, beta, w)

    for n in range(2):
        lp = module_lp(lambda t: enc[n, t].reshape(1, 1, -1), pred, joiner)
        ref = beam_ref_fused(int(lens[n]), V, B, lp, term)
        _agree([got[n]], [([list(p) for p, _ in ref], [s for _, s in ref])])


@pytest.mark.parametrize("B", [1, 3, 8])
def test_fused_beam_ref_without_terms_is_beam_ref(B):
    V, T = 6, 5
    pred, joiner = _setup(V)
    enc = torch.randn(1, T, 6, dtype=torch.float64) * 2
    lp = module_lp(lambda t: enc[0, t].reshape(1, 1, -1), pred, joiner)
    zero = lambda t, p: fuse_term(np.zeros(V), None, 0.0, 0.0, 0.0)   # alpha = 0, beta = 0: a zero term
    a, b, c = beam_ref(T, V, B, lp), beam_ref_fused(T, V, B, lp), beam_ref_fused(T, V, B, lp, zero)
    assert a == b == c


@pytest.mark.parametrize("T", [1, 2, 3, 4])
def test_unpruned_scores_are_exhaustive_plus_lm_part(T, tmp_path):
    # without pruning every prefix survives with its full acoustic log-sum; the LM part is a function of the prefix
    V = 3
    lm = _lm("ngram3", tmp_path, V)
    lmrow = prefix_lm(lm)
    rng = np.random.default_rng(T)
    rows = {}

    def lp(t, p):
        if (t, p) not in rows:
            z = rng.standard_normal(V) * 2
            rows[(t, p)] = z - np.logaddexp.reduce(z)
        return rows[(t, p)]

    term = lambda t, p: fuse_term(lmrow(p), None, 0.6, 0.4, 0.0)
    got = beam_ref_fused(T, V, 10 ** 6, lp, term)
    ex = exhaustive(T, V, lp)
    assert len(got) == len(ex)
    for p, s in got:
        m = sum(0.4 + 0.6 * lmrow(p[:i])[p[i]] for i in range(len(p)))
        assert abs(s - (ex[p] + m)) <= 1e-12 * (1 + abs(s)), (p, s, ex[p], m)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_dense_chain_rows_equal_textbook(tmp_path, case):
    V, order, counts, opt = CASES[case]
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, order, counts, seed=case, **opt)
    labels = cat_labels(V)
    lm = NGramLM(path, labels)
    t = lm.tables()
    tb, walk = Textbook(path, labels), Walk(lm)
    rng = np.random.default_rng(case)
    S = len(t["bow"])
    # every state (a sample of them and of the labels at V = 8192): the row is the walk's value, rounded once
    states = range(S) if S <= 2000 else rng.choice(S, 300, replace=False)
    ks = range(1, V) if V <= 100 else rng.choice(np.arange(1, V), 64, replace=False)
    for s in states:
        row = ngram_rows_dense(t, int(s))
        for k in ks:
            acc, _ = walk(int(s), int(t["tok2word"][k]))
            assert row[k] == np.float32(acc * LN10), (s, k)
    # along token sequences from the start state (after </s>): the row is the textbook's ln P(. | </s> + prefix)
    grams = [g for g in tb.g if len(g) == order and all(w.isdigit() for w in g)]
    tok = {w: i for i, w in enumerate(labels) if i > 0 and w}
    for j in range(200):
        seq = [tok[w] for w in grams[rng.integers(len(grams))] if w in tok] if grams and j % 2 else \
            list(rng.integers(1, V, rng.integers(0, 2 * order + 2)))
        s = int(t["root_dst"][t["eos"]])
        for c in seq:
            s = walk(s, int(t["tok2word"][c]))[1]
        hist = ["</s>"] + [tb.word(labels[c]) for c in seq]
        h = tuple(hist[max(0, len(hist) - (order - 1)):]) if order > 1 else ()
        row = ngram_rows_dense(t, s)
        for k in ks:
            ref = tb.log10(h, tb.word(labels[k])) * LN10
            assert abs(float(row[k]) - ref) <= 1e-6 * (1 + abs(ref)), (seq, k, row[k], ref)


# ---- constructor and argument checks -------------------------------------------------------------------------------------
class _NoNative:
    """Stands in for the native library: any call fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"native call {name} reached")


@pytest.fixture
def no_native(monkeypatch):
    monkeypatch.setattr(rnnt_decode._lib, "lib", lambda: _NoNative())


def test_decoder_refusals_name_the_type(no_native):
    class NGram(torch.nn.Module):
        def get_log_prob(self, *a):
            pass

    class MultiDecoder(NGram):
        pass

    with pytest.raises(NotImplementedError, match="NGramLM"):
        RNNTDecoder(None, None, lm_module=NGram(), alpha=0.5)
    with pytest.raises(NotImplementedError, match="MultiDecoder"):
        RNNTDecoder(None, None, lm_module=MultiDecoder(), alpha=0.5)
    with pytest.raises(NotImplementedError, match="LogAdd"):
        RNNTDecoder(None, LogAdd(), est_ilm=True, ilm_weight=0.3)
    with pytest.raises(NotImplementedError, match="impl_forward"):
        RNNTDecoder(None, torch.nn.Linear(2, 2), est_ilm=True, ilm_weight=0.3)
    for bad in (float("nan"), float("inf"), "0.5", True):
        with pytest.raises(ValueError):
            RNNTDecoder(None, JointNet(2, 2, 3, 2), est_ilm=True, ilm_weight=bad)


def test_decoder_accepts_fusion(no_native, tmp_path):
    pred, joiner = _setup()
    d = RNNTDecoder(pred, joiner, lm_module=LSTMLM(7, 4), alpha=0.3, beta=-0.5, est_ilm=True, ilm_weight=-0.3125)
    assert d.alpha == 0.3 and d.beta == -0.5 and d.ilm_weight == -0.3125
    # est_ilm off: the ILM weight is dropped, and a LogAdd joiner is fine
    assert RNNTDecoder(None, LogAdd(), est_ilm=False, ilm_weight=0.4).ilm_weight == 0.0


@pytest.mark.skipif(not torch.cuda.is_available(), reason="the search's argument checks need a CUDA enc_out")
def test_search_fusion_errors_before_native(no_native, tmp_path):
    V = 7
    pred, joiner = (m.float().cuda() for m in _setup(V))
    enc = torch.randn(2, 3, 6, device="cuda")
    lens = torch.tensor([3, 2])
    with pytest.raises(ValueError, match="V = 5"):   # an LSTM LM over 5 labels, a joiner over 7
        rnnt_beam_search(enc, lens, pred, joiner, lm=LSTMLM(5, 4).cuda(), alpha=0.5)
    with pytest.raises(NotImplementedError, match="LM"):
        rnnt_beam_search(enc, lens, pred, joiner, lm=object(), alpha=0.5)
    with pytest.raises(NotImplementedError, match="ILM"):
        rnnt_beam_search(enc, lens, pred, LogAdd(), ilm_weight=0.5)
    with pytest.raises(ValueError, match="alpha"):
        rnnt_beam_search(enc, lens, pred, joiner, lm=LSTMLM(V, 4).cuda(), alpha=float("nan"))


def test_ngram_lm_v_mismatch_and_blank_are_value_errors(monkeypatch, tmp_path):
    path = make_random_arpa(str(tmp_path / "lm.arpa"), 9, 3, 30)
    lm = NGramLM(path, _labels(9))
    monkeypatch.setattr(rnnt_decode._lib, "lib", lambda: _NoNative())
    with pytest.raises(ValueError, match="blank"):
        rnnt_decode._Fusion(lm, 0.5, 0.0, 0.0, None, 2, "x")
    if torch.cuda.is_available():
        pred, joiner = (m.float().cuda() for m in _setup(7))
        with pytest.raises(ValueError, match="V = 9"):
            rnnt_beam_search(torch.randn(1, 2, 6, device="cuda"), torch.tensor([2]), pred, joiner, lm=lm, alpha=0.5)


def test_native_entries_reject_bad_arguments(tmp_path):
    L = _lib.lib()
    N, T, B, V = 2, 3, 4, 9
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    args = [p, None, 0, 0, N, T, B, V, 0, p, 0, p, p, p, p, p]
    ok = dict(lm_rows=p, lm_dtype=0, alpha=0.5, beta=0.1, ilm_rows=None, ilm_dtype=0, w=0.0, lm_part=p)

    def call(**kw):
        a = dict(ok, **kw)
        return L.ccb_rnnt_beam_step_fused(*args, a["lm_rows"], a["lm_dtype"], a["alpha"], a["beta"], a["ilm_rows"],
                                          a["ilm_dtype"], a["w"], a["lm_part"], None)

    assert call(lm_rows=None) != 0 and "rnnt_beam_step" in _lib.last_error()
    assert call(lm_part=None) != 0 and "missing buffer" in _lib.last_error()
    for bad in (dict(alpha=math.inf), dict(beta=math.nan), dict(ilm_rows=p, w=-math.inf)):
        assert call(**bad) != 0 and "finite" in _lib.last_error()
    assert call(lm_dtype=7) != 0
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, 3, 30)
    lm = NGramLM(path, _labels(V))
    assert L.ccb_ngram_slot_rows(lm.handle, N, B, V + 1, None, None, None, p, p, None) != 0
    assert "labels" in _lib.last_error()
    assert L.ccb_ngram_slot_rows(lm.handle, N, B, V, None, None, None, None, p, None) != 0
    assert "missing buffer" in _lib.last_error()
    assert L.ccb_ngram_slot_rows(lm.handle, N, B, V, p, None, p, p, p, None) != 0   # a parent without tokens
    assert L.ccb_ngram_slot_rows(None, N, B, V, None, None, None, p, p, None) != 0
    assert L.ccb_ngram_slot_rows(lm.handle, N, 129, V, None, None, None, p, p, None) != 0
