"""CPU side of n-gram sentence scoring (``NGramLM.score``, ``MultiLM.score``, ``cat_b200.rescore.rescore_nbest``): a numpy
restatement of the kernel's window replay (``Replay``) against the textbook scorer over CAT's word string, the replayed
states against the sequential walk's, CAT's conventions, the argument checks (all raised before any native call), the
native entry's refusal of LMs without <s> or </s>, and ``rescore_nbest``'s arithmetic against CAT's ``rescore.py``;
tests/test_gpu_ngram_score.py compares the kernel against ``Replay``."""
import ctypes as C
import math
import re

import numpy as np
import pytest
import torch

from cat_b200 import _lib
from cat_b200.ngram import NGramLM, make_random_arpa
from cat_b200.rescore import rescore_nbest
from cat_b200.rnnt_decode import MultiLM
from test_ngram_dispatch import CASES, LN10, Textbook, Walk, cat_labels

SLOTS = 1024        # the kernel's summation tree (ngram_score.cu kSlots)


def word_ids(path, labels):
    """The loader's word ids: the unigrams some label names, and <s>, </s>, <unk>, in file order, <unk> appended if the
    file has none."""
    named = {(w or "<unk>") for w in labels[1:]} | {"<s>", "</s>", "<unk>"}
    ids, k = {}, 0
    for line in open(path):
        t = line.split()
        if t and t[0].startswith("\\"):
            k = int(t[0][1:].split("-")[0]) if t[0].endswith("-grams:") else 0
        elif k == 1 and t and t[1] in named and t[1] not in ids:
            ids[t[1]] = len(ids)
    ids.setdefault("<unk>", len(ids))
    return ids


def cat_string(ids, last, L, labels):
    """CAT's NGram.score word string of one row: labels of ids[:L] (token 0 </s>, 1 <unk>), a leading </s> made <s>, and
    the word of the last target appended."""
    word = lambda k: "</s>" if k == 0 else (labels[k] or "<unk>")
    seq = [word(int(k)) for k in ids[:L]]
    if seq[0] == "</s>":
        seq[0] = "<s>"
    return seq + [word(int(last))]


def textbook_score(tb, seq):
    """ln 10 * sum_i log10 P(w_i | the n-1 words before it), from the empty history (KenLM's bos = eos = False)."""
    ws = [tb.word(w) for w in seq]
    return sum(tb.log10(tuple(ws[max(0, i - tb.order + 1):i]), w) for i, w in enumerate(ws)) * LN10


class Replay:
    """The kernel (ngram_score.cu) restated: every term from the state the destination rule reaches from the root over
    the n-1 words before it, each LmLog10's walk (``Walk``), summed over the fixed tree in fp64 and rounded once."""

    def __init__(self, lm, path, labels):
        self.walk = Walk(lm)
        self.t = self.walk.t
        self.order, self.V = lm.order, lm.V
        self.bos_word = word_ids(path, labels)["<s>"]

    def next(self, s, w):
        t = self.t
        while s != 0:
            lo, hi = int(t["arc_off"][s]), int(t["arc_off"][s + 1])
            i = lo + int(np.searchsorted(t["arc_word"][lo:hi], w))
            if i < hi and t["arc_word"][i] == w:
                return int(t["arc_dst"][i])
            s = int(t["back"][s])
        return int(t["root_dst"][w])

    def words(self, ids, last, L):
        toks = [int(k) for k in ids[:L]] + [int(last)]
        return [-1 if not 0 <= k < self.V else
                (self.bos_word if i == 0 else int(self.t["eos"])) if k == 0 else int(self.t["tok2word"][k])
                for i, k in enumerate(toks)]

    def state(self, ws, i):
        s = 0
        for v in ws[max(0, i - self.order + 1):i]:
            s = self.next(s, v)
        return s

    def terms(self, ws):
        out = []
        for i, w in enumerate(ws):
            window = ws[max(0, i - self.order + 1):i + 1]
            out.append(math.nan if min(window) < 0 else self.walk(self.state(ws, i), w)[0])
        return out

    def score(self, ids, last, L=None):
        U = len(ids)
        L = U if L is None else int(L)
        if not 1 <= L <= U:
            return np.float32(np.nan)
        return np.float32(tree_sum(self.terms(self.words(ids, last, L))) * LN10)


def tree_sum(terms):
    slots = [-0.0] * SLOTS
    for i, x in enumerate(terms):
        slots[i % SLOTS] += x
    h = SLOTS // 2
    while h:
        for j in range(h):
            slots[j] += slots[j + h]
        h //= 2
    return slots[0]


def _case_lm(tmp_path, case):
    V, order, counts, opt = CASES[case]
    opt = dict(opt, bos=True)     # a sentence score starts with <s>: the entry refuses files without it
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, order, counts, seed=case, **opt)
    labels = cat_labels(V)
    rng = np.random.default_rng(case)
    for i in rng.choice(np.arange(2, V), size=min(3, V - 2), replace=False):
        labels[i] = f"oov{i}"
    labels[-1] = ""
    return path, labels, NGramLM(path, labels)


def _sentences(tb, labels, V, order, rng, n):
    """Rows drawn from the LM's own n-grams (long histories reached) and at random, with token 0 at position 0 or inside."""
    grams = [g for g in tb.g if len(g) == order and all(w.isdigit() for w in g)]
    tok = {w: i for i, w in enumerate(labels) if i > 0 and w}
    for k in range(n):
        if grams and k % 2:
            seq = [tok[w] for w in grams[rng.integers(len(grams))] if w in tok]
            seq += list(rng.integers(0, V, rng.integers(0, 3)))
        else:
            seq = list(rng.integers(1, V, rng.integers(0, 2 * order + 3)))
        if k % 3 == 0 or not seq:
            seq = [0] + seq
        yield np.array(seq, np.int64)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_replay_equals_textbook_and_sequential_walk(tmp_path, case):
    path, labels, lm = _case_lm(tmp_path, case)
    V, order = CASES[case][0], CASES[case][1]
    tb, rp = Textbook(path, labels), Replay(lm, path, labels)
    ids = word_ids(path, labels)
    assert all(int(rp.t["tok2word"][k]) == ids.get(labels[k] or "<unk>", ids["<unk>"]) for k in range(1, V))
    rng = np.random.default_rng(100 + case)
    for seq in _sentences(tb, labels, V, order, rng, 1200):
        last = 0 if rng.random() < 0.8 else int(rng.integers(1, V))
        want = textbook_score(tb, cat_string(seq, last, len(seq), labels))
        ws = rp.words(seq, last, len(seq))
        got = tree_sum(rp.terms(ws)) * LN10
        assert abs(got - want) <= 1e-12 * max(1.0, abs(want)), (seq, got, want)
        assert float(rp.score(seq, last)) == float(np.float32(got))
        # the replayed state before each word is the one the sequential walk over the whole row reaches
        s = 0
        for i, w in enumerate(ws):
            assert rp.state(ws, i) == s, (seq, i)
            s = rp.walk(s, w)[1]


def test_cat_conventions(tmp_path):
    V = 20
    labels = cat_labels(V)
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, 3, [80, 120], seed=7)
    lm = NGramLM(path, labels)
    tb, rp = Textbook(path, labels), Replay(lm, path, labels)
    row = np.array([0, 5, 0, 7, 3, 9, 11])
    # a leading 0 is <s>, an interior 0 is </s>; the last column of targets, not targets[b, L - 1], ends the string
    assert cat_string(row, 0, 4, labels) == ["<s>", "5", "</s>", "7", "</s>"]
    assert cat_string(row, 6, 3, labels) == ["<s>", "5", "</s>", "6"]
    for L in (1, 3, 4, 7):
        for last in (0, 6):
            want = textbook_score(tb, cat_string(row, last, L, labels))
            assert abs(float(rp.score(row, last, L)) - want) <= 2e-6 * max(1.0, abs(want))
    # only position 0 is rewritten: <s> scored as a unigram (-99 as make_random_arpa writes it)
    ws = rp.words(row, 0, 3)
    assert ws[0] == rp.bos_word and ws[2] == rp.t["eos"] and ws[3] == rp.t["eos"]
    assert abs(rp.terms(ws)[0] - float(np.float32(-99.0))) < 1e-9
    # input_lengths None is the full width
    assert rp.score(row, 0) == rp.score(row, 0, len(row))
    # a bad token or length is NaN for that row
    assert np.isnan(rp.score(np.array([3, V, 4]), 0)) and np.isnan(rp.score(row, -1)) and np.isnan(rp.score(row, 0, 0))


# ---------------------------------------------------------------------------------------------------------------------
# argument checks, before any native call
# ---------------------------------------------------------------------------------------------------------------------
class _NoNative:
    def __getattr__(self, name):
        raise AssertionError(f"native call {name} reached")


@pytest.fixture
def small_lm(tmp_path):
    return NGramLM(make_random_arpa(str(tmp_path / "lm.arpa"), 6, 2, 10, seed=0), cat_labels(6))


def test_score_argument_checks(monkeypatch, small_lm):
    monkeypatch.setattr(_lib, "lib", lambda: _NoNative())
    ids = torch.tensor([[0, 2, 3], [0, 4, 5]])
    tg = torch.zeros((2, 3), dtype=torch.int64)
    lens = torch.tensor([3, 2])
    bad = [
        (dict(input_ids=ids[0]), "input_ids must be an int32 or int64 \\(N, U\\)"),
        (dict(input_ids=ids.float()), "input_ids must be an int32 or int64"),
        (dict(input_ids=ids[:, :0]), "U >= 1"),
        (dict(targets=tg[0]), "targets must be an int32 or int64"),
        (dict(targets=tg[:1]), "targets must be an int32 or int64"),
        (dict(targets=tg[:, :0]), "targets must be"),
        (dict(targets=tg.short()), "targets must be"),
        (dict(input_lengths=lens[:1]), "input_lengths must be None or"),
        (dict(input_lengths=lens.float()), "input_lengths must be None or"),
        (dict(input_lengths=torch.tensor([3, 0])), "input_lengths must lie in \\[1, U = 3\\]"),
        (dict(input_lengths=torch.tensor([4, 1])), "input_lengths must lie in \\[1, U = 3\\]"),
        (dict(input_ids=torch.tensor([[0, 2, 6], [0, 4, 5]])), "tokens must lie in \\[0, V = 6\\)"),
        (dict(input_ids=torch.tensor([[0, 2, -1], [0, 4, 5]])), "tokens must lie in"),
        (dict(targets=torch.tensor([[0, 0, 0], [0, 0, 9]])), "tokens must lie in"),
    ]
    for kw, msg in bad:
        args = dict(input_ids=ids, targets=tg, input_lengths=lens)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            small_lm.score(**args)
    # positions at or past a row's length are not looked at
    with pytest.raises(AssertionError, match="native call"):
        small_lm.score(torch.tensor([[0, 2, 99]]), torch.zeros((1, 1), dtype=torch.int64), torch.tensor([2]))
    # MultiLM.score and rescore_nbest go through the same checks
    mix = MultiLM([0.5, 1.0], [small_lm, small_lm])
    with pytest.raises(ValueError, match="tokens must lie in"):
        mix.score(torch.tensor([[0, 7]]), torch.zeros((1, 1), dtype=torch.int64))
    tok = torch.full((1, 2, 3), -1, dtype=torch.int32)
    for a, b, msg in [(math.nan, 0.0, "alpha must be a finite"), (1.0, math.inf, "beta must be a finite"),
                      (None, 0.0, "alpha must be a finite"), (True, 0.0, "alpha must be a finite")]:
        with pytest.raises(ValueError, match=msg):
            rescore_nbest(tok, torch.zeros((1, 2), dtype=torch.int32), torch.zeros((1, 2)), small_lm, a, b)
    with pytest.raises(ValueError, match="lengths and scores \\(N, K\\)"):
        rescore_nbest(tok, torch.zeros((1, 3), dtype=torch.int32), torch.zeros((1, 2)), small_lm)


def _no_boundary(tmp_path, which):
    """make_random_arpa's LM without <s> (bos=False), or without </s> and every n-gram that contains it."""
    p = make_random_arpa(str(tmp_path / f"{which}.arpa"), 6, 2, 10, seed=1, bos=which != "bos")
    if which == "eos":
        keep, n, k = [], {}, 0
        for ln in open(p).read().split("\n"):
            if ln.startswith("\\"):
                k = int(ln[1]) if ln.endswith("-grams:") else 0
            elif k and ln.strip() and "</s>" in ln.split():
                continue
            elif k and ln.strip():
                n[k] = n.get(k, 0) + 1
            keep.append(ln)
        text = "\n".join(keep)
        for k, c in n.items():
            text = re.sub(rf"ngram {k}=\d+", f"ngram {k}={c}", text)
        open(p, "w").write(text)
    return NGramLM(p, cat_labels(6))


@pytest.mark.parametrize("which,word", [("bos", "<s>"), ("eos", "</s>")])
def test_entry_refuses_lm_without_sentence_boundaries(tmp_path, which, word):
    lm = _no_boundary(tmp_path, which)
    L = _lib.lib()
    buf = (C.c_longlong * 8)()
    p = C.cast(buf, C.c_void_p)
    n0 = L.ccb_launch_count()
    assert L.ccb_ngram_score(lm.handle, 1, 2, p, 2, 1, p, 1, 1, None, 0, p, None) != 0
    assert f"ngram_score: the LM lists no {word}" in _lib.last_error()
    assert L.ccb_launch_count() == n0


def test_entry_argument_checks(small_lm):
    L = _lib.lib()
    buf = (C.c_longlong * 8)()
    p = C.cast(buf, C.c_void_p)
    args = lambda lm=small_lm.handle, R=1, U=2, ids=p, st=2, i64=1, last=p, out=p: \
        (lm, R, U, ids, st, i64, last, 1, 1, None, 0, out, None)
    for kw, what in [(dict(lm=None), "missing LM"), (dict(R=0), "R and U must be positive"),
                     (dict(U=0), "R and U must be positive"), (dict(st=1), "ids_stride must be >= U"),
                     (dict(i64=2), "flags are 0 (int32) or 1 (int64)"), (dict(ids=None), "missing buffer"),
                     (dict(last=None), "missing buffer"), (dict(out=None), "missing buffer")]:
        assert L.ccb_ngram_score(*args(**kw)) != 0
        assert what in _lib.last_error(), (kw, _lib.last_error())


# ---------------------------------------------------------------------------------------------------------------------
# rescore_nbest against CAT's rescore.py
# ---------------------------------------------------------------------------------------------------------------------
class FakeLM:
    """CAT's score interface over the textbook scorer, recording what it was given."""

    def __init__(self, tb, labels):
        self.tb, self.labels, self.calls = tb, labels, []

    def score(self, input_ids, targets, input_lengths=None):
        self.calls.append((input_ids.clone(), targets.clone(), input_lengths.clone()))
        return torch.tensor([textbook_score(self.tb, cat_string(r.numpy(), int(t[-1]), int(L), self.labels))
                             for r, t, L in zip(input_ids, targets, input_lengths)], dtype=torch.float32)


def cat_rescore(texts, scores, lm_scores, alpha, beta):
    """rescore.py main_worker on one batch: keys "nid-okey", in_lens counting <s>, the first of the highest total kept."""
    in_lens = torch.tensor([len(t) + 1 for t in texts])
    final = scores + alpha * lm_scores + beta * in_lens
    indiv = {}
    for k, s in zip(range(len(texts)), final):
        if 0 not in indiv:
            indiv[0] = (s, k)
        elif indiv[0][0] < s:
            indiv[0] = (s, k)
    return final, indiv[0][1]


@pytest.mark.parametrize("alpha,beta", [(0.0, 0.0), (0.37, -0.8), (1.0, 2.5), (0.5, 0.0)])
def test_rescore_nbest_matches_cat(tmp_path, alpha, beta):
    V, T, K = 15, 9, 6
    labels = cat_labels(V)
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, 3, [60, 80], seed=3)
    tb = Textbook(path, labels)
    lm = FakeLM(tb, labels)
    rng = np.random.default_rng(int(alpha * 100 + beta * 10 + 50))
    N = 5
    tokens = torch.full((N, K, T), -1, dtype=torch.int32)
    lengths = torch.full((N, K), -1, dtype=torch.int32)
    scores = torch.full((N, K), float("-inf"))
    hyps = []
    for n in range(N):
        rows = []
        for k in range(K - (n % 3)):        # absent rows at the end, as the searches leave them
            L = int(rng.integers(0, T + 1))
            seq = rng.integers(1, V, L)
            tokens[n, k, :L] = torch.from_numpy(seq)
            lengths[n, k] = L
            scores[n, k] = float(np.float32(-rng.uniform(1, 30)))
            rows.append(list(seq))
        if n == 1 and len(rows) >= 3:       # a tie: two copies of one hypothesis with the same score
            tokens[n, 2], lengths[n, 2], scores[n, 2] = tokens[n, 0], lengths[n, 0], scores[n, 0]
            rows[2] = rows[0]
        hyps.append(rows)
    lm_scores, total, best = rescore_nbest(tokens, lengths, scores, lm, alpha, beta)
    # CAT's input: token 0 first, length + 1, 0 in the last target column
    ids, tg, ln = lm.calls[0]
    assert ids.shape == (N * K, T + 1) and bool((ids[:, 0] == 0).all()) and bool((tg[:, -1] == 0).all())
    assert torch.equal(ln, lengths.reshape(-1).clamp(min=0).long() + 1)
    for n in range(N):
        texts = hyps[n]
        lm_cat = torch.tensor([textbook_score(tb, ["<s>"] + [labels[t] for t in h] + ["</s>"]) for h in texts],
                              dtype=torch.float32)
        final, keep = cat_rescore(texts, scores[n, :len(texts)], lm_cat, alpha, beta)
        assert torch.equal(lm_scores[n, :len(texts)], lm_cat)
        assert torch.equal(total[n, :len(texts)], final)
        assert bool((total[n, len(texts):] == float("-inf")).all()) and bool((lm_scores[n, len(texts):] == float("-inf")).all())
        assert int(best[n]) == keep
    if len(hyps[1]) >= 3:
        assert total[1, 0] == total[1, 2] and int(best[1]) != 2
