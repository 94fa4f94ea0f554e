"""CPU: the RNN-T beam search with an LM mix (``cat_b200.rnnt_decode.MultiLM``): the constructor rules, CAT's
``MultiDecoder`` accepted or refused, the mix restatement (tests/multilm_oracle.py) against the textbook ARPA scorer,
``beam_ref_fused`` with the mix term against CAT's decoder with ``CatMultiDecoder``, and the argument checks, all raised
before any native call, and those of ``ccb_lm_mix_slot_rows``."""
import ctypes as C

import numpy as np
import pytest
import torch

from cat_b200 import _lib, rnnt_decode
from cat_b200.ngram import NGramLM, make_random_arpa
from cat_b200.rnnt_decode import MAX_MIX, MultiLM, RNNTDecoder, rnnt_beam_search
from multilm_oracle import CatMultiDecoder, mix_rows
from rnnt_decode_oracle import LSTMPredictor, module_lp
from rnnt_fusion_oracle import (CatNGram, JointNet, LSTMLM, beam_ref_fused, cat_decode_fused, fuse_term,
                                ngram_rows_dense, prefix_ilm, prefix_lm)
from test_ngram_dispatch import LN10, Textbook, Walk


def _labels(V):
    return ["<blk>", "<unk>"] + [str(i) for i in range(2, V)]


class _NoNative:
    """Stands in for the native library: any call fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"native call {name} reached")


@pytest.fixture
def no_native(monkeypatch):
    monkeypatch.setattr(rnnt_decode._lib, "lib", lambda: _NoNative())


def _arpa(tmp_path, V, order, seed=None, counts=None):
    return make_random_arpa(str(tmp_path / f"lm{order}_{V}.arpa"), V, order, counts or [3 * V] * (order - 1),
                            seed=order if seed is None else seed)


# ---- constructor rules ---------------------------------------------------------------------------------------------------
def test_constructor_rules(tmp_path, monkeypatch):
    V = 9
    ng = NGramLM(_arpa(tmp_path, V, 3), _labels(V))
    ng2 = NGramLM(_arpa(tmp_path, V + 2, 2), _labels(V + 2))
    monkeypatch.setattr(rnnt_decode._lib, "lib", lambda: _NoNative())
    lstm = LSTMLM(V, 4)
    m = MultiLM([0.28125, 0.0, -0.3125], [ng, object(), lstm])   # zero-weight members are dropped, whatever they are
    assert m.weights == [0.28125, -0.3125] and m.lms == [ng, lstm] and m.has_ngram
    assert MultiLM((1, 2.5), (lstm, lstm)).weights == [1.0, 2.5]
    with pytest.raises(ValueError, match="2 weights for 1"):
        MultiLM([0.5, 0.5], [ng])
    for bad in (float("nan"), float("inf"), -float("inf"), "0.5", True, None):
        with pytest.raises(ValueError, match="finite"):
            MultiLM([0.5, bad], [ng, lstm])
    with pytest.raises(ValueError, match="zero"):
        MultiLM([0.0, 0.0], [ng, lstm])
    with pytest.raises(ValueError, match="zero"):
        MultiLM([], [])
    with pytest.raises(ValueError, match=f"at most {MAX_MIX}"):
        MultiLM([0.1] * (MAX_MIX + 1), [lstm] * (MAX_MIX + 1))
    MultiLM([0.1] * MAX_MIX + [0.0], [lstm] * (MAX_MIX + 1))   # the zero weight does not count
    with pytest.raises(ValueError, match="different numbers of labels"):
        MultiLM([0.5, -0.2], [ng, ng2])


def test_refusals_by_type(no_native):
    class NGram(torch.nn.Module):
        def get_log_prob(self, *a):
            pass

    class PretrainedTransformer(NGram):
        pass

    lstm = LSTMLM(7, 4)
    with pytest.raises(NotImplementedError, match="NGramLM"):
        MultiLM([0.5, -0.3], [lstm, NGram()])
    with pytest.raises(NotImplementedError, match="Transformer"):
        MultiLM([0.5, -0.3], [lstm, PretrainedTransformer()])
    with pytest.raises(NotImplementedError, match="get_log_prob"):
        MultiLM([0.5, -0.3], [lstm, object()])
    with pytest.raises(NotImplementedError, match="nest"):
        MultiLM([0.5, -0.3], [lstm, MultiLM([1.0], [lstm])])
    with pytest.raises(NotImplementedError, match="nest"):
        MultiLM([0.5, -0.3], [lstm, CatMultiDecoder([1.0], [lstm])])


def test_shared_memory_limit(tmp_path, monkeypatch):
    # 8 (W + V) bytes of shared memory: a 13 000-label LM (W > V) fits ccb_ngram_slot_rows (8 W bytes) but not a mix
    V = 13000
    big = NGramLM(make_random_arpa(str(tmp_path / "big.arpa"), V, 2, 100), _labels(V))
    assert 8 * (big.num_words + V) > 200 * 1024 >= 8 * big.num_words
    monkeypatch.setattr(rnnt_decode._lib, "lib", lambda: _NoNative())
    with pytest.raises(ValueError, match="shared memory"):
        MultiLM([0.5, -0.2], [big, LSTMLM(V, 4)])
    # a neural-only mix: checked against the joiner's V when the search starts (below, before any native call)
    MultiLM([0.5, -0.2], [LSTMLM(30000, 2), LSTMLM(30000, 2)])


def test_cat_multidecoder_accepted_or_refused(monkeypatch, tmp_path):
    V = 7
    ng = NGramLM(_arpa(tmp_path, V, 2), _labels(V))
    monkeypatch.setattr(rnnt_decode._lib, "lib", lambda: _NoNative())
    a, b = LSTMLM(V, 4), LSTMLM(V, 5)
    d = RNNTDecoder(None, None, lm_module=CatMultiDecoder([0.5, 0.0, -0.25], [a, LSTMLM(V, 3), b]), alpha=0.3)
    assert isinstance(d.lm, MultiLM) and d.lm.weights == [0.5, -0.25] and d.lm.lms == [a, b]
    # NGramLM objects the user put into _decs
    md = CatMultiDecoder([0.5, -0.25], [ng, b])
    assert RNNTDecoder(None, None, lm_module=md, alpha=0.3).lm.lms == [ng, b]

    # without readable members: NotImplementedError naming MultiDecoder and MultiLM
    class MultiDecoder(torch.nn.Module):
        def get_log_prob(self, *a):
            pass

    with pytest.raises(NotImplementedError, match="MultiDecoder.*MultiLM"):
        RNNTDecoder(None, None, lm_module=MultiDecoder(), alpha=0.5)
    # readable members the search cannot carry: the member's refusal
    bad = CatMultiDecoder([0.5, -0.25], [a, b])

    class NGram(torch.nn.Module):
        def get_log_prob(self, *a):
            pass

    bad._decs = torch.nn.ModuleList([a, NGram()])
    with pytest.raises(NotImplementedError, match="NGramLM"):
        RNNTDecoder(None, None, lm_module=bad, alpha=0.5)
    # all-zero weights: nothing to fuse (CAT fails at its first frame)
    with pytest.raises(ValueError, match="zero"):
        RNNTDecoder(None, None, lm_module=CatMultiDecoder([0.0, 0.0], [a, b]), alpha=0.5)
    # alpha = 0 drops the LM whatever it is, as for one LM
    assert RNNTDecoder(None, None, lm_module=MultiDecoder(), alpha=0.0).lm is None


def test_blank_must_be_zero_with_an_ngram_member(monkeypatch, tmp_path):
    V = 9
    ng = NGramLM(_arpa(tmp_path, V, 3), _labels(V))
    monkeypatch.setattr(rnnt_decode._lib, "lib", lambda: _NoNative())
    with pytest.raises(ValueError, match="blank"):
        rnnt_decode._Fusion(MultiLM([0.5, -0.1], [LSTMLM(V, 4), ng]), 0.5, 0.0, 0.0, None, 2, "x")
    rnnt_decode._Fusion(MultiLM([0.5, -0.1], [LSTMLM(V, 4), LSTMLM(V, 3)]), 0.5, 0.0, 0.0, None, 2, "x")


@pytest.mark.skipif(not torch.cuda.is_available(), reason="the search's argument checks need a CUDA enc_out")
def test_search_errors_before_native(monkeypatch, tmp_path):
    V = 7
    ng = NGramLM(_arpa(tmp_path, 9, 2), _labels(9))
    monkeypatch.setattr(rnnt_decode._lib, "lib", lambda: _NoNative())
    torch.manual_seed(0)
    pred, joiner = LSTMPredictor(V, 6).cuda(), JointNet(6, 6, V, 8).cuda()
    enc = torch.randn(2, 3, 6, device="cuda")
    lens = torch.tensor([3, 2])
    with pytest.raises(ValueError, match="member 1 of the LM mix has V = 5"):
        rnnt_beam_search(enc, lens, pred, joiner, lm=MultiLM([0.5, 0.2], [LSTMLM(V, 4).cuda(), LSTMLM(5, 4).cuda()]),
                         alpha=0.5)
    with pytest.raises(ValueError, match="member 0 of the LM mix has V = 9"):
        rnnt_beam_search(enc, lens, pred, joiner, lm=MultiLM([0.5], [ng]), alpha=0.5)
    big = MultiLM([0.5, 0.2], [LSTMLM(26000, 2).cuda(), LSTMLM(26000, 2).cuda()])
    pred2, joiner2 = LSTMPredictor(26000, 6).cuda(), JointNet(6, 6, 26000, 8).cuda()
    with pytest.raises(ValueError, match="shared memory"):
        rnnt_beam_search(enc, lens, pred2, joiner2, lm=big, alpha=0.5)


# ---- the mix restatement -------------------------------------------------------------------------------------------------
def test_mix_rows_order_rounding_and_inf():
    r = [np.array([1.0, -np.inf, 0.1, 3.0], np.float32), np.array([2.0, 5.0, -np.inf, 1e-8], np.float32),
         np.array([0.5, 1.0, 2.0, -3.0], np.float32)]
    w = [0.3, -0.7, 1.1]
    got = mix_rows(r, w)
    assert got.dtype == np.float32
    assert got[1] == -np.inf and got[2] == -np.inf   # whatever the weights' signs
    x = [np.float64(wi) * np.float64(ri[0]) for wi, ri in zip(w, r)]
    assert got[0] == np.float32((x[0] + x[1]) + x[2])
    assert mix_rows(r[:1], [1.0])[3] == r[0][3]   # one member of weight 1: its row
    assert mix_rows(r, w, np.float64)[3] == (0.3 * np.float64(r[0][3]) + -0.7 * np.float64(r[1][3])) + 1.1 * -3.0


@pytest.mark.parametrize("orders", [(5, 2), (3, 2), (2, 2, 3)])
def test_mix_of_dense_rows_is_the_textbook_sum(tmp_path, orders):
    V = 40
    labels = _labels(V)
    paths = [_arpa(tmp_path, V, o, seed=10 + i, counts=[4 * V] * (o - 1)) for i, o in enumerate(orders)]
    lms = [NGramLM(p, labels) for p in paths]
    tbs = [Textbook(p, labels) for p in paths]
    walks = [Walk(lm) for lm in lms]
    tabs = [lm.tables() for lm in lms]
    w = [0.28125, -0.3125, 0.125][:len(orders)]
    rng = np.random.default_rng(len(orders))
    for _ in range(60):
        seq = list(rng.integers(1, V, rng.integers(0, 8)))
        rows = []
        for t, walk in zip(tabs, walks):
            s = int(t["root_dst"][t["eos"]])
            for c in seq:
                s = walk(s, int(t["tok2word"][c]))[1]
            rows.append(ngram_rows_dense(t, s))
        got = mix_rows(rows, w)
        ref = np.zeros(V)
        for wi, tb in zip(w, tbs):
            hist = ["</s>"] + [tb.word(labels[c]) for c in seq]
            h = tuple(hist[max(0, len(hist) - (tb.order - 1)):])
            ref += wi * np.array([0.0] + [tb.log10(h, tb.word(labels[k])) * LN10 for k in range(1, V)])
        assert np.allclose(got, ref, rtol=1e-6, atol=1e-6), seq
        assert got[0] == 0.0


# ---- the search with the mix term against CAT's decoder ------------------------------------------------------------------
def _setup(V=7, H=6, seed=0):
    torch.manual_seed(seed)
    pred = LSTMPredictor(V, H).double()
    joiner = JointNet(H, H, V, 8).double()
    for m in (pred, joiner):
        for p in m.parameters():
            p.data.mul_(3.0)
    return pred, joiner


def _members(kind, tmp_path, V):
    if kind == "lstm":
        torch.manual_seed(3)
        lm = LSTMLM(V, 5).double()
        for p in lm.parameters():
            p.data.mul_(3.0)
        return lm
    order = int(kind[-1])
    return CatNGram(_arpa(tmp_path, V, order, seed=20 + order, counts=[3 * V] * (order - 1)), _labels(V))


@pytest.mark.parametrize("mix, alpha, beta, w", [
    (("ngram5", "ngram2"), 0.9, 0.5, 0.0), (("ngram3", "ngram2"), 1.0, 0.3, 0.0), (("lstm", "ngram2"), 0.8, -0.2, 0.0),
    (("ngram5", "ngram2"), 1.0, 0.5, -0.3125),
])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_cat_multidecoder_matches_beam_ref_fused(mix, alpha, beta, w, B, tmp_path):
    V, T = 7, 5
    pred, joiner = _setup(V)
    members = [_members(k, tmp_path, V) for k in mix]
    weights = [0.28125 * 3, -0.3125 * 2] if mix[0] != "lstm" else [1.0, -0.3125]
    lm = CatMultiDecoder(weights, members)
    torch.manual_seed(1)
    enc = torch.randn(2, T, 6, dtype=torch.float64) * 2
    lens = torch.tensor([T, 3])
    got = cat_decode_fused(enc, lens, pred, joiner, B, lm=lm, alpha=alpha, beta=beta, ilm_weight=w)
    rows = [prefix_lm(m) for m in members]
    ilm = prefix_ilm(pred, joiner, 6) if w else None

    def term(t, p):
        return fuse_term(mix_rows([r(p) for r in rows], weights, np.float64), ilm(p) if ilm else None, alpha, beta, w)

    for n in range(2):
        lp = module_lp(lambda t: enc[n, t].reshape(1, 1, -1), pred, joiner)
        ref = beam_ref_fused(int(lens[n]), V, B, lp, term)
        assert got[n][0] == [list(p) for p, _ in ref]
        for a, (_, b) in zip(got[n][1], ref):
            assert abs(a - b) <= 1e-9 * (1 + abs(b)), (a, b)


# ---- the native entry's argument checks ----------------------------------------------------------------------------------
def test_native_entry_rejects_bad_arguments(tmp_path):
    L = _lib.lib()
    N, B, V = 2, 4, 9
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    lm = NGramLM(_arpa(tmp_path, V, 3), _labels(V))
    lm2 = NGramLM(_arpa(tmp_path, V + 1, 2), _labels(V + 1))

    def arr(t, xs):
        return (t * len(xs))(*xs)

    def call(ngrams=(lm,), ng_w=(0.5,), n_neural=1, nn_w=(-0.2,), dtypes=(0,), order=(0, 1), beam=B, K=None, V=V,
             rows=p, parent=None, token=None, st_out=p, nrow=p):
        n_ng = len(ngrams)
        hs = arr(C.c_void_p, [None if g is None else g.handle for g in ngrams] or [None])
        return L.ccb_lm_mix_slot_rows(n_ng if K is None else K, hs, arr(C.c_double, list(ng_w) or [0.0]),
                                      arr(C.c_void_p, [p] * max(n_ng, 1)), arr(C.c_void_p, [st_out] * max(n_ng, 1)),
                                      n_neural, arr(C.c_void_p, [nrow] * max(n_neural, 1)),
                                      arr(C.c_int, list(dtypes) or [0]), arr(C.c_double, list(nn_w) or [0.0]),
                                      None if order is None else arr(C.c_int, list(order)), N, beam, V, parent, token,
                                      rows, None)

    assert call(ngrams=(lm2,)) != 0 and "labels" in _lib.last_error()
    assert call(ngrams=(None,)) != 0 and "missing LM" in _lib.last_error()
    assert call(ng_w=(0.0,)) != 0 and "non-zero" in _lib.last_error()
    assert call(nn_w=(float("nan"),)) != 0 and "finite" in _lib.last_error()
    assert call(order=(0, 0)) != 0 and "permutation" in _lib.last_error()
    assert call(order=(2, 0)) != 0 and "permutation" in _lib.last_error()
    assert call(order=None) != 0 and "missing buffer" in _lib.last_error()
    assert call(rows=None) != 0 and "missing buffer" in _lib.last_error()
    assert call(st_out=None) != 0 and "missing buffer" in _lib.last_error()
    assert call(nrow=None) != 0 and "missing buffer" in _lib.last_error()
    assert call(parent=p) != 0 and "missing buffer" in _lib.last_error()   # a parent without tokens
    assert call(dtypes=(7,)) != 0
    assert call(beam=129) != 0 and "beam" in _lib.last_error()
    assert call(ngrams=(), ng_w=(), n_neural=0, order=()) != 0 and "members" in _lib.last_error()
    n = MAX_MIX + 1
    assert call(ngrams=(), ng_w=(), n_neural=n, nn_w=[0.1] * n, dtypes=[0] * n, order=range(n)) != 0
    assert "members" in _lib.last_error()
    V2 = 26000
    assert call(ngrams=(), ng_w=(), order=(0,), V=V2) != 0 and "shared memory" in _lib.last_error()
