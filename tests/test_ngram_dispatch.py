"""CPU side of the token n-gram LM fused into the prefix beam search (``ctc_crf.ctc_beam_search(..., lm=NGramLM(...))``):
the ARPA loader against a textbook back-off scorer, its error messages, the argument checks, the ``CTCBeamDecoder`` options,
and ``beam_lm_ref``, a numpy restatement of the search with the LM, checked against the search without one and against
exhaustive enumeration; tests/test_gpu_beam_lm.py compares the kernel against it."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from cat_b200 import _C, _lib
from cat_b200.ngram import NGramLM, make_random_arpa
from test_beam_dispatch import NEG, _FakeCuda, _Steps, _ext_in, _near, beam_ref, enum_plain, hyps, lse

LN10 = 2.302585092994045684      # the kernel's constant


def cat_labels(V):
    """CAT's token labels: blank, <unk>, then the token ids as words."""
    return ["<s>", "<unk>"] + [str(i) for i in range(2, V)]


# ---------------------------------------------------------------------------------------------------------------------
# the textbook scorer (from the text) and the walk over the loader's tables
# ---------------------------------------------------------------------------------------------------------------------
class Textbook:
    """ARPA back-off straight from the text: values rounded to fp32, the history truncated to n-1 words, a word the file
    does not list as a unigram scored as <unk> (log10 p = -100 when the file has no <unk>)."""

    def __init__(self, path, labels):
        self.g, k, self.order = {}, 0, 0
        for line in open(path):
            t = line.split()
            if not t or t[0] == "ngram":
                continue
            if t[0].startswith("\\"):
                k = int(t[0][1:].split("-")[0]) if t[0].endswith("-grams:") else 0
                self.order = max(self.order, k)
                continue
            if k:
                b = float(np.float32(float(t[k + 1]))) if len(t) == k + 2 else 0.0
                self.g.setdefault(tuple(t[1:k + 1]), (float(np.float32(float(t[0]))), b))
        self.g.setdefault(("<unk>",), (-100.0, 0.0))
        self.labels = labels

    def word(self, w):
        w = w or "<unk>"
        return w if (w,) in self.g else "<unk>"

    def log10(self, h, w):
        if h + (w,) in self.g:
            return self.g[h + (w,)][0]
        return self.g.get(h, (0.0, 0.0))[1] + self.log10(h[1:], w)

    def ln_seq(self, seq):
        """ln P(l </s>) of the token sequence seq, and the per-word terms."""
        hist = ["<s>"] if ("<s>",) in self.g else []
        terms = []
        for w in [self.word(self.labels[t]) for t in seq] + [self.word("</s>")]:
            h = tuple(hist[max(0, len(hist) - (self.order - 1)):])
            terms.append(self.log10(h, w) * LN10)
            hist.append(w)
        return sum(terms), terms


class Walk:
    """The kernel's walk (beam_search.cu LmLog10) over the tables ``ccb_ngram_copy`` exports, memoised per (state, word)."""

    def __init__(self, lm):
        self.t = lm.tables()
        self.memo = {}

    def __call__(self, s, w):
        key = (s, w)
        if key in self.memo:
            return self.memo[key]
        t, s0, acc, d = self.t, s, 0.0, -1
        while True:
            if s == 0:
                acc += float(t["root_p"][w])
                d = int(t["root_dst"][w]) if d < 0 else d
                break
            lo, hi = int(t["arc_off"][s]), int(t["arc_off"][s + 1])
            i = lo + int(np.searchsorted(t["arc_word"][lo:hi], w))
            if i < hi and t["arc_word"][i] == w:
                d = int(t["arc_dst"][i]) if d < 0 else d
                p = t["arc_p"][i]
                if not np.isnan(p):
                    acc += float(p)
                    break
            acc += float(t["bow"][s])
            s = int(t["back"][s])
        self.memo[(s0, w)] = (acc, d)
        return acc, d

    def ln_seq(self, seq):
        s, terms = self.t["bos"], []
        for w in [int(self.t["tok2word"][c]) for c in seq] + [self.t["eos"]]:
            acc, s = self(s, w)
            terms.append(acc * LN10)
        return sum(terms), terms


# (V, order, counts, options): orders 1-5, V up to 8192, pruned prefixes, missing suffixes, OOV labels, words no label names,
# no <unk>, no <s>
CASES = [
    (6, 1, [], {}),
    (12, 2, 40, dict(unk=False)),
    (30, 3, [200, 300], dict(pruned_prefixes=0.5, extra_words=5)),
    (50, 3, [300, 400], dict(missing_suffixes=True, bos=False)),
    (40, 4, [300, 400, 400], dict(pruned_prefixes=0.3, missing_suffixes=True, unk=False, extra_words=3)),
    (25, 5, [150, 250, 300, 300], dict(pruned_prefixes=0.4)),
    (8192, 3, [3000, 3000], dict(extra_words=20, pruned_prefixes=0.2)),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_walk_equals_textbook_backoff(tmp_path, case):
    V, order, counts, opt = CASES[case]
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, order, counts, seed=case, **opt)
    labels = cat_labels(V)
    rng = np.random.default_rng(case)
    # OOV labels: some tokens name words the file does not list, and one is empty
    for i in rng.choice(np.arange(2, V), size=min(3, V - 2), replace=False):
        labels[i] = f"oov{i}"
    labels[-1] = ""
    lm = NGramLM(path, labels)
    assert lm.order == order and lm.counts[0] >= V - 2 and lm.unk_substituted == (not opt.get("unk", True))
    tb, walk = Textbook(path, labels), Walk(lm)
    # sequences drawn from the LM's own n-grams too, so that the long histories are reached and not only backed off
    grams = [g for g in tb.g if len(g) == order and all(w.isdigit() for w in g)]
    tok = {w: i for i, w in enumerate(labels) if i > 0 and w}
    for k in range(1500):
        if grams and k % 2:
            seq = [tok[w] for w in grams[rng.integers(len(grams))] if w in tok]
            seq += list(rng.integers(1, V, rng.integers(0, 3)))
        else:
            seq = list(rng.integers(1, V, rng.integers(0, 2 * order + 3)))
        a, ta = tb.ln_seq(seq)
        b, tw = walk.ln_seq(seq)
        np.testing.assert_allclose(tw, ta, rtol=1e-12, atol=1e-12)
        assert abs(a - b) <= 1e-12 * max(1.0, abs(a)), (seq, a, b)


def test_closure_inserts_missing_prefixes_and_drops_unnamed_words(tmp_path):
    p = tmp_path / "lm.arpa"
    p.write_text("\\data\\\nngram 1=5\nngram 2=1\nngram 3=1\n\n\\1-grams:\n-1.0\t<s>\t-0.5\n-0.7\t2\t-0.25\n-0.9\t3\t-0.1\n"
                 "-1.1\tzz\t-0.2\n-0.3\t</s>\n\n\\2-grams:\n-0.4\tzz 2\t-0.3\n\n\\3-grams:\n-0.2\t<s> 2 3\n\n\\end\\\n")
    lm = NGramLM(str(p), ["<s>", "<unk>", "2", "3"])
    t = lm.tables()
    # words: <s>, 2, 3, </s> and the substituted <unk>; zz is unnamed, so its bigram is dropped
    assert lm.num_words == 5 and lm.unk_substituted and lm.counts == [5, 1, 1]
    # states: root, 5 unigrams and the inserted bigram "<s> 2"; its only arc is "3" (the listed trigram)
    assert lm.num_states == 7 and lm.num_arcs == 2
    nan = np.isnan(t["arc_p"])
    assert nan.sum() == 1 and t["bow"][t["arc_dst"][nan][0]] == 0.0
    tb, walk = Textbook(str(p), ["<s>", "<unk>", "2", "3"]), Walk(lm)
    for seq in ([2, 3], [2], [3, 2, 3], [1, 2, 3], []):
        assert abs(tb.ln_seq(seq)[0] - walk.ln_seq(seq)[0]) <= 1e-12 * max(1, abs(tb.ln_seq(seq)[0]))
    # "<s> 2 3": the trigram's own value
    assert abs(walk.ln_seq([2, 3])[1][1] - np.float32(-0.2) * LN10) < 1e-12


# ---------------------------------------------------------------------------------------------------------------------
# loader errors
# ---------------------------------------------------------------------------------------------------------------------
GOOD = "\\data\\\nngram 1=3\nngram 2=1\n\n\\1-grams:\n-1.0\t<s>\t-0.5\n-0.7\t2\t-0.25\n-0.3\t</s>\n\n\\2-grams:\n-0.4\t<s> 2\n\n\\end\\\n"


@pytest.mark.parametrize("text,msg", [
    ("hello\n" + GOOD, r"line 1: an ARPA file starts with \\data\\"),
    (GOOD.replace("ngram 1=3", "ngram 1=4"), r"line 5: \\1-grams: lists 3 n-grams, \\data\\ declares 4"),
    (GOOD.replace("-0.7\t2", "-0.7x\t2"), r"line 7: '-0.7x' is not a number"),
    (GOOD.replace("2\t-0.25", "2\tnan"), r"line 7: 'nan' is not a number"),
    (GOOD.replace("-0.4\t<s> 2", "-0.4\t<s>"), r"line 11: a 2-gram line has log10 p, 2 words and an optional back-off "
                                               r"weight, not 2 fields"),
    (GOOD.replace("\\2-grams:", "\\bigrams:"), r"line 10: unknown section '\\bigrams:'"),
    (GOOD.replace("\\2-grams:", "\\3-grams:"), r"line 10: unknown section '\\3-grams:'"),
    (GOOD.replace("\\end\\\n", ""), r"the file ends at line 12 without \\end\\"),
    (GOOD.replace("ngram 2=1", "ngram 3=1"), r"line 3: the counts must be listed for orders 1, 2, \.\.\. in turn"),
    ("mmap lm http://kheafield.com/code\0\0binary", r"KenLM binary; pass the ARPA text that `ngram.sh --arpa`"),
])
def test_malformed_files_name_the_line(tmp_path, text, msg):
    p = tmp_path / "bad.arpa"
    p.write_bytes(text.encode())
    with pytest.raises(RuntimeError, match=msg):
        NGramLM(str(p), ["<s>", "<unk>", "2"])
    p.write_bytes(GOOD.encode())
    assert NGramLM(str(p), ["<s>", "<unk>", "2"]).order == 2


def test_loader_refuses_sentence_boundaries_as_labels(tmp_path):
    p = tmp_path / "lm.arpa"
    p.write_text(GOOD)
    for bad in ("<s>", "</s>"):
        with pytest.raises(ValueError, match="sentence boundaries"):
            NGramLM(str(p), ["_", bad, "2"])
        arr = (C.c_char_p * 3)(b"_", bad.encode(), b"2")
        assert not _lib.lib().ccb_ngram_create(str(p).encode(), arr, 3)
        assert f"label 1 is {bad}" in _lib.last_error()
    with pytest.raises(RuntimeError, match="cannot open"):
        NGramLM(str(tmp_path / "missing.arpa"), ["_", "2"])


# ---------------------------------------------------------------------------------------------------------------------
# the restatement with the LM
# ---------------------------------------------------------------------------------------------------------------------
def beam_lm_ref(y, lens, B, topn, lm=None, alpha=1.0, beta=0.0, tol=1e-9):
    """``beam_ref`` in plain mode with the LM fused in, as the kernel's LM instantiation computes it: each entry carries an
    LM state and an LM part (the sum over its extensions of alpha ln P + beta, fp64, rounded operation by operation); a
    candidate ranks by its mass plus its prefix's LM part; after the last frame each entry adds alpha ln P(</s> | state).
    lm None: the search without an LM.  Same returns as ``beam_ref``, the scores including the LM."""
    y = np.asarray(y, np.float32)
    N, T, V = y.shape
    step = _Steps(None, V)
    if lm is not None:
        walk = Walk(lm)
        tok2word = walk.t["tok2word"]

    def term(s, c):      # what extending an entry in LM state s by token c adds, and the next state
        if alpha == 0:
            return beta, s
        acc, d = walk(s, int(tok2word[c]))
        return alpha * (acc * LN10) + beta, d

    tokens = np.full((N, B, T), -1, np.int32)
    stamps = np.full((N, B, T), -1, np.int32)
    lengths = np.full((N, B), -1, np.int32)
    scores = np.full((N, B), NEG)
    near = np.zeros(N, bool)
    for n in range(N):
        parent, tok, frame = [-1], [-1], [-1]
        trie = {}
        node = np.array([0]); last = np.array([-1]); par = np.array([-1])
        mb = np.array([0.0]); mt = np.array([NEG])
        sb = np.array([-1]); st = np.array([-1])
        lmp = np.array([0.0]); ls = np.array([walk.t["bos"] if lm is not None else 0])
        rank = {0: 0}
        for t in range(int(lens[n])):
            yr = y[n, t].astype(np.float64)
            nb = len(node)
            toks = np.lexsort((np.arange(V), -yr))[:topn] if topn < V else np.arange(V)
            flag = np.zeros(V, bool)
            flag[toks] = True
            par = np.full(nb, -1)
            merged = set()
            for r in range(nb):
                p = parent[node[r]]
                pr = rank.get(p, -1) if p >= 0 else -1
                c = int(last[r])
                if pr >= 0 and (flag[c] or c == last[pr]):
                    par[r] = pr
                    merged.add(pr * (V + 1) + c)
            rr = np.arange(nb)
            lw1, d1 = step(sb, 0)
            lw2, d2 = step(st, 0)
            a, b = mb + lw1, mt + lw2
            bin_ = lse(a, b)
            mbn = np.where(bin_ > NEG, bin_ + yr[0], NEG)
            lw3, d3 = step(st, last)
            rep = np.where(last >= 1, mt + lw3, NEG)
            pe = np.maximum(par, 0)
            ein, d4 = _ext_in(step, mb, mt, sb, st, last, pe, last)
            ext = np.where(par >= 0, ein, NEG)
            tin = lse(rep, ext)
            ok = (last >= 1) & (tin > NEG)
            mtn = np.where(ok, tin + yr[np.maximum(last, 0)], NEG)
            m_stay = lse(mbn, mtn)
            if lm is not None:
                m_stay = m_stay + lmp
            k_stay = rr * (V + 1)
            R = np.repeat(rr, len(toks))
            Cc = np.tile(toks, nb)
            extra = (last >= 1) & ~flag[np.maximum(last, 0)]
            R = np.concatenate([R, rr[extra]])
            Cc = np.concatenate([Cc, last[extra]])
            keep = (Cc >= 1) & ~np.isin(R * (V + 1) + Cc, list(merged))
            R, Cc = R[keep], Cc[keep]
            ein, dst = _ext_in(step, mb, mt, sb, st, last, R, Cc)
            m_ext = np.where(ein > NEG, ein + yr[Cc], NEG)
            if lm is not None:
                add = np.array([lmp[r] + term(int(ls[r]), int(c))[0] if m > NEG else 0.0 for r, c, m in zip(R, Cc, m_ext)])
                m_ext = m_ext + add
            M = np.concatenate([m_stay, m_ext])
            K = np.concatenate([k_stay, R * (V + 1) + Cc + 1])
            fin = M > NEG
            M, K = M[fin], K[fin]
            order = np.lexsort((K, -M))
            if len(order) > B and _near(M[order[B - 1]], M[order[B]], tol):
                near[n] = True
            n_node, n_last, n_mb, n_mt, n_lmp, n_ls = [], [], [], [], [], []
            for i in order[:B]:
                key = int(K[i])
                r, c = key // (V + 1), key % (V + 1) - 1
                if c < 0:
                    n_node.append(int(node[r])); n_last.append(int(last[r]))
                    n_mb.append(mbn[r]); n_mt.append(mtn[r])
                    n_lmp.append(lmp[r]); n_ls.append(int(ls[r]))
                else:
                    e, _ = _ext_in(step, mb, mt, sb, st, last, np.array([r]), np.array([c]))
                    x = trie.get((int(node[r]), c))
                    if x is None:
                        x = len(parent)
                        parent.append(int(node[r])); tok.append(c); frame.append(t)
                        trie[(int(node[r]), c)] = x
                    n_node.append(x); n_last.append(c)
                    n_mb.append(NEG); n_mt.append(float(e[0]) + yr[c])
                    if lm is not None:
                        dl, d = term(int(ls[r]), c)
                        n_lmp.append(lmp[r] + dl); n_ls.append(d)
                    else:
                        n_lmp.append(0.0); n_ls.append(0)
            node, last = np.array(n_node, np.int64), np.array(n_last, np.int64)
            mb, mt = np.array(n_mb, np.float64), np.array(n_mt, np.float64)
            sb, st = np.full(len(node), -1), np.full(len(node), -1)
            lmp, ls = np.array(n_lmp, np.float64), np.array(n_ls, np.int64)
            rank = {int(x): k for k, x in enumerate(node)}
        fs = lse(mb, mt)
        if lm is not None:
            eos = np.array([alpha * (walk(int(s), walk.t["eos"])[0] * LN10) if alpha != 0 else 0.0 for s in ls])
            fs = np.where(fs > NEG, fs + (lmp + eos), fs)
        good = np.nonzero(fs > NEG)[0]
        order = good[np.lexsort((good, -fs[good]))]
        if any(_near(fs[order[i]], fs[order[i + 1]], tol) for i in range(len(order) - 1)):
            near[n] = True
        for row, k in enumerate(order):
            seq, ts = [], []
            x = int(node[k])
            while x > 0:
                seq.append(tok[x]); ts.append(frame[x])
                x = parent[x]
            tokens[n, row, :len(seq)] = seq[::-1]
            stamps[n, row, :len(ts)] = ts[::-1]
            lengths[n, row] = len(seq)
            scores[n, row] = fs[k]
    return tokens, lengths, stamps, scores, near


def _logsoftmax(x):
    return (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)


def _same(a, b):
    return all(np.array_equal(x, z) for x, z in zip(a, b))


@pytest.mark.parametrize("B,cut,seed", [(1, 5, 0), (4, 3, 1), (8, 9, 2), (16, 9, 3)])
def test_restatement_without_lm_and_at_zero_weights_is_beam_ref(tmp_path, B, cut, seed):
    rng = np.random.default_rng(seed)
    V = 9
    y = _logsoftmax(rng.standard_normal((4, 12, V)) * 2)
    lens = np.array([12, 7, 1, 0])
    want = beam_ref(y, lens, B, cut)
    assert _same(beam_lm_ref(y, lens, B, cut), want)
    lm = NGramLM(make_random_arpa(str(tmp_path / "lm.arpa"), V, 3, [30, 40], seed=seed), cat_labels(V))
    assert _same(beam_lm_ref(y, lens, B, cut, lm, alpha=0.0, beta=0.0), want)
    # and a real weight changes the lists
    assert not _same(beam_lm_ref(y, lens, B, cut, lm, alpha=1.7, beta=0.5)[:4], want[:4])


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("T,V,seed", [(1, 3, 0), (4, 3, 1), (5, 4, 2), (6, 4, 3)])
def test_restatement_is_exact_at_full_beam(tmp_path, order, T, V, seed):
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, order, [6, 10][:order - 1], seed=seed + 10 * order,
                            pruned_prefixes=0.3, missing_suffixes=bool(seed % 2))
    labels = cat_labels(V)
    lm = NGramLM(path, labels)
    tb = Textbook(path, labels)
    y = _logsoftmax(np.random.default_rng(seed).standard_normal((1, T, V)) * 1.5)
    plain = enum_plain(y[0], T)
    for alpha in (0.5, 1.7):
        for beta in (-0.5, 0.0, 1.0):
            tokens, lengths, _, scores, _ = beam_lm_ref(y, [T], 4000, V, lm, alpha, beta)
            got = hyps(tokens, lengths, scores, 0)
            assert set(got) == set(plain)
            for k, v in plain.items():
                want = v + alpha * tb.ln_seq(k)[0] + beta * len(k)
                assert abs(got[k] - want) <= 1e-12 * max(1, abs(want)), (alpha, beta, k, got[k], want)
            assert np.all(np.diff(scores[0][lengths[0] >= 0]) <= 0)


# ---------------------------------------------------------------------------------------------------------------------
# arguments (checked before anything touches a device) and the decoder
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def small_lm(tmp_path):
    return NGramLM(make_random_arpa(str(tmp_path / "lm.arpa"), 4, 2, 6, seed=0), cat_labels(4))


def test_argument_checks(monkeypatch, small_lm):
    monkeypatch.setattr(_FakeCuda, "is_cuda", property(lambda self: True))
    y = torch.zeros((2, 5, 4)).as_subclass(_FakeCuda)
    lx = torch.tensor([5, 3], dtype=torch.int32)
    for kw, msg in [(dict(alpha=-0.1), "alpha must be >= 0"), (dict(alpha=math.inf), "alpha must be a finite"),
                    (dict(alpha=math.nan), "alpha must be a finite"), (dict(beta=math.nan), "beta must be a finite"),
                    (dict(beta=-math.inf), "beta must be a finite"), (dict(alpha=None), "alpha must be a finite"),
                    (dict(crf=True), "cannot be combined with crf=True")]:
        args = dict(crf=False, alpha=1.0, beta=0.0)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            _C.ctc_beam_search(y, lx, 4, 4, args["crf"], small_lm, args["alpha"], args["beta"])
    with pytest.raises(ValueError, match="loaded for 4 labels, the logits have V = 5"):
        _C.ctc_beam_search(torch.zeros((2, 5, 5)).as_subclass(_FakeCuda), lx, 4, 4, False, small_lm)
    # without an LM, alpha and beta are not looked at
    _C._check_lm_args(None, math.nan, math.nan, True, 4)
    _C._check_lm_args(small_lm, 0.0, -3.0, False, 4)


def test_native_lm_entry_rejects_bad_arguments(small_lm):
    L = _lib.lib()
    buf = (C.c_int * 4)()
    p = C.cast(buf, C.c_void_p)
    args = lambda crf=0, V=4, a=1.0, b=0.0: (p, 0, 1, 2, V, p, 4, 2, crf, p, p, p, p, p, small_lm.handle, a, b, None)
    for kw, what in [(dict(crf=1), "cannot be combined with crf=1"), (dict(a=-1.0), "alpha must be finite and >= 0"),
                     (dict(a=math.nan), "alpha must be finite"), (dict(b=math.inf), "beta must be finite"),
                     (dict(V=5), "loaded for 4 labels, V is 5")]:
        assert L.ccb_ctc_beam_search_lm(*args(**kw)) != 0
        assert what in _lib.last_error(), (kw, _lib.last_error())
    info = (C.c_long * 18)()
    assert L.ccb_ngram_info(small_lm.handle, info) == 0 and info[0] == 2 and info[5] == 4
    assert L.ccb_ngram_copy(small_lm.handle, 9, p, 16) != 0
    assert L.ccb_ngram_copy(small_lm.handle, 0, p, 4) == 2         # too small for tok2word[4]


def test_decoder_lm_options(tmp_path):
    import ctc_crf
    V = 30
    labels = cat_labels(V)
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, 3, [100, 100], seed=4)
    d = ctc_crf.CTCBeamDecoder(labels, model_path=path, alpha=0.25, beta=-0.5, beam_width=32, cutoff_top_n=40,
                               num_processes=6, log_probs_input=True, is_token_based=True)
    assert d._lm.order == 3 and d._lm.V == V and (d._alpha, d._beta) == (0.25, -0.5) and d._cutoff_top_n == V
    with pytest.raises(NotImplementedError, match="word-level"):
        ctc_crf.CTCBeamDecoder(labels, model_path=path, alpha=0.25, beta=-0.5)
    binary = tmp_path / "lm.bin"
    binary.write_bytes(b"mmap lm http://kheafield.com/code\0\0\0\1" + bytes(100))
    for bad in (str(tmp_path / "missing.arpa"), str(binary)):
        with pytest.raises(NotImplementedError, match="only ARPA text") as e:
            ctc_crf.CTCBeamDecoder(labels, model_path=bad, is_token_based=True)
        assert bad in str(e.value)
    broken = tmp_path / "broken.arpa"
    broken.write_text(open(path).read().replace("\\end\\", ""))
    with pytest.raises(RuntimeError, match="without"):
        ctc_crf.CTCBeamDecoder(labels, model_path=str(broken), is_token_based=True)
    with pytest.raises(ValueError, match="sentence boundaries"):
        ctc_crf.CTCBeamDecoder(["<s>", "</s>", "2"], model_path=path, is_token_based=True)
    assert ctc_crf.NGramLM is NGramLM
