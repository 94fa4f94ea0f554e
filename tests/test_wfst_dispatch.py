"""CPU: the decoding-graph reader and its load checks, ``fst.make_tlg`` against textbook back-off costs, the numpy float32
restatement ``wfst_decode_ref`` of the TLG Viterbi beam search (csrc/wfst_decode.cu) against an fp64 exhaustive Viterbi, and
the argument checks of ``ctc_crf.fst_decode``.  ``wfst_decode_ref`` is what tests/test_gpu_wfst_decode.py holds the kernel to."""
import math
import struct

import numpy as np
import pytest
import torch

from cat_b200 import fst
from cat_b200.ngram import make_random_arpa
from cat_b200.wfst import DecodingGraph, check_decode_args

NOARC = (1 << 32) - 1
F32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------------
def random_wfst(S, V, W, seed, n_emit=None, n_eps=None, chain=0, neg_eps=True, dead_ends=0, no_final=False):
    """A random decoding graph: emitting arcs anywhere, epsilon arcs only from lower to higher positions of a random
    permutation (an acyclic epsilon subgraph), an epsilon chain through `chain` states, words on emitting and epsilon arcs,
    parallel arcs, negative epsilon weights, `dead_ends` states without out-arcs, and optionally no final state."""
    rng = np.random.default_rng(seed)
    n_emit = n_emit or 4 * S
    n_eps = n_eps if n_eps is not None else S
    perm = rng.permutation(S)
    pos = np.empty(S, np.int64)
    pos[perm] = np.arange(S)
    dead = set(rng.choice(np.arange(1, S), size=dead_ends, replace=False).tolist()) if dead_ends else set()
    src, dst, il, ol, w = [], [], [], [], []
    live = [s for s in range(S) if s not in dead]
    for _ in range(n_emit):
        s = int(rng.choice(live)); d = int(rng.integers(S))
        src.append(s); dst.append(d); il.append(int(rng.integers(1, V + 1)))
        ol.append(int(rng.integers(1, W + 1)) if rng.random() < 0.3 else 0); w.append(float(rng.uniform(0.0, 3.0)))
    for _ in range(n_eps):
        a, b = sorted(rng.choice(S, size=2, replace=False).tolist(), key=lambda q: pos[q])
        if a in dead:
            continue
        src.append(a); dst.append(b); il.append(0)
        ol.append(int(rng.integers(1, W + 1)) if rng.random() < 0.3 else 0)
        w.append(float(rng.uniform(-1.0 if neg_eps else 0.0, 2.0)))
    order = sorted((q for q in range(S) if q not in dead), key=lambda q: pos[q])[:chain]
    for a, b in zip(order, order[1:]):
        src.append(a); dst.append(b); il.append(0); ol.append(int(rng.integers(0, W + 1))); w.append(float(rng.uniform(-0.5, 1)))
    for j in range(min(len(src), S // 2)):          # parallel arcs: same ends and label, another weight or word
        k = int(rng.integers(len(src)))
        src.append(src[k]); dst.append(dst[k]); il.append(il[k]); ol.append(int(rng.integers(0, W + 1)))
        w.append(float(w[k] + rng.uniform(-0.3, 0.3)))
    final = np.full(S, np.inf, np.float32)
    if not no_final:
        final[rng.choice(S, size=max(1, S // 4), replace=False)] = rng.uniform(0, 2, size=max(1, S // 4))
    return fst.DenGraph(num_states=S, start=0, src=np.array(src, np.int32), dst=np.array(dst, np.int32),
                        ilabel=np.array(il, np.int32), olabel=np.array(ol, np.int32), weight=np.array(w, np.float32),
                        final=final)


def tiny_lexicon(V, n_words, seed, homophones=True):
    rng = np.random.default_rng(seed)
    lex = [(str(i), rng.integers(1, V, size=int(rng.integers(1, 4))).tolist()) for i in range(2, 2 + n_words)]
    if homophones:
        lex.append((str(3), list(lex[0][1])))       # a second pronunciation that is another word's
        lex.append((str(4), list(lex[2][1]) + [1]))  # one that extends another word's
    return lex


# ---------------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------------
class Tables:
    """The loader's tables plus the per-arc source, in the layout the search walks."""

    def __init__(self, graph: DecodingGraph):
        t = graph.tables()
        self.__dict__.update(t)
        self.S, self.A, self.start, self.L = graph.num_states, graph.num_arcs, graph.start, graph.L
        self.src = np.repeat(np.arange(self.S), np.diff(self.arc_off))
        self.lay = np.empty(self.A, np.int64)
        self.lay[self.fid] = np.arange(self.A)


def _ranges(lo, hi):
    """The concatenated index ranges [lo_i, hi_i), and for each index the position i of its range."""
    n = hi - lo
    idx = np.repeat(lo - np.cumsum(n) + n, n) + np.arange(int(n.sum()))
    return idx, np.repeat(np.arange(len(lo)), n)


def _recombine(st, co, aid):
    """The smallest (cost, arc id) per state, as (states, costs, ids) sorted by state."""
    o = np.lexsort((aid, co, st))
    st, co, aid = st[o], co[o], aid[o]
    first = np.ones(len(st), bool)
    first[1:] = st[1:] != st[:-1]
    return st[first], co[first], aid[first]


def _search(tb, y, ln, nacs, wps, beam, K):
    """Layers of one utterance: per layer (states, costs, arc ids) of every token and the kept states; None when dead."""
    layers = []
    st, co, aid = np.array([tb.start]), np.array([0], F32), np.array([NOARC])
    cutoff = F32(beam)
    for t in range(ln + 1):
        if t > 0:
            ks, kc = layers[-1][3], layers[-1][4]
            idx, which = _ranges(tb.arc_off[ks], tb.eps_off[ks])
            x = (kc[which] + tb.weight[idx]) + nacs * y[t - 1][tb.token[idx]]
            x = np.where(tb.olabel[idx] != 0, x + wps, x).astype(F32)
            best = x.min() if len(x) else F32(np.inf)
            if not best < np.inf:
                return None
            cutoff = F32(best + F32(beam))
            m = (x <= cutoff) & (x < np.inf)
            st, co, aid = _recombine(tb.dst[idx[m]], x[m], tb.fid[idx[m]].astype(np.int64))
        for lv in range(tb.L + 1):
            sel = tb.level[st] == lv
            idx, which = _ranges(tb.eps_off[st[sel]], tb.arc_off[st[sel] + 1])
            if len(idx) == 0:
                continue
            x = co[sel][which] + tb.weight[idx]
            x = np.where(tb.olabel[idx] != 0, x + wps, x).astype(F32)
            m = (x <= cutoff) & (x < np.inf)
            st, co, aid = _recombine(np.concatenate([st, tb.dst[idx[m]]]), np.concatenate([co, x[m]]),
                                     np.concatenate([aid, tb.fid[idx[m]].astype(np.int64)]))
        o = np.lexsort((st, co))[:K]
        layers.append((st, co, aid, st[o], co[o]))
    return layers


def wfst_decode_ref(tb: Tables, y, lens, acwt=1.0, lmwt=1.0, wip=0.0, beam=17.0, max_active=7000):
    """numpy float32 restatement of ccb_wfst_decode; returns the outputs of ``fst_decode`` as numpy arrays."""
    y = np.asarray(y, np.float32)
    N, T, V = y.shape
    acs, wps = F32(acwt) / F32(lmwt), F32(wip) / F32(lmwt)
    nacs = -acs
    Wcap = (T + 1) * (1 + tb.L)
    out = dict(words=np.full((N, Wcap), -1, np.int32), num_words=np.full(N, -1, np.int32), align=np.full((N, T), -1, np.int32),
               ac_logp=np.full(N, -np.inf, np.float32), graph_cost=np.full(N, np.inf, np.float32),
               cost=np.full(N, np.inf, np.float32), reached_final=np.zeros(N, np.int32))
    for n in range(N):
        ln = int(lens[n])
        layers = _search(tb, y[n], ln, nacs, wps, beam, max_active)
        if layers is None:
            continue
        ks, kc = layers[-1][3], layers[-1][4]
        fin = tb.final[ks]
        fc = (kc + fin).astype(F32)
        ok = (fin < np.inf) & (fc < np.inf)
        if ok.any():
            i = np.nonzero(ok)[0][np.lexsort((ks[ok], fc[ok]))[0]]
        else:
            i = np.lexsort((ks, kc))[0]
        s = int(ks[i])
        g = float(tb.final[s]) if ok.any() else 0.0
        arcs = []
        f = ln
        while True:
            st, _, aid = layers[f][:3]
            a_id = int(aid[np.searchsorted(st, s)])
            if a_id == NOARC:
                break
            a = int(tb.lay[a_id])
            arcs.append(a)
            s = int(tb.src[a])
            if tb.token[a] >= 0:
                f -= 1
        arcs = arcs[::-1]
        words = [int(tb.olabel[a]) for a in arcs if tb.olabel[a] != 0]
        em = [a for a in arcs if tb.token[a] >= 0]
        assert len(em) == ln
        g += sum(float(tb.weight[a]) for a in arcs)
        ac = sum(float(y[n, t, tb.token[a]]) for t, a in enumerate(em))
        out["words"][n, :len(words)] = words
        out["num_words"][n] = len(words)
        out["align"][n, :ln] = [tb.token[a] for a in em]
        out["ac_logp"][n], out["graph_cost"][n] = ac, g
        out["cost"][n] = lmwt * g - acwt * ac + wip * len(words)
        out["reached_final"][n] = int(ok.any())
    return out


def viterbi_fp64(tb: Tables, y, ln, acwt=1.0, lmwt=1.0, wip=0.0):
    """Exhaustive Viterbi over all states in fp64 (no beam, no max_active): (words, align, search cost, reached_final)."""
    acs, wps = acwt / lmwt, wip / lmwt
    S = tb.S
    order = np.argsort(tb.level, kind="stable")

    def close(d, bp):
        for s in order:
            if not np.isfinite(d[s]):
                continue
            for j in range(tb.eps_off[s], tb.arc_off[s + 1]):
                x = d[s] + tb.weight[j] + (wps if tb.olabel[j] else 0.0)
                if x < d[tb.dst[j]]:
                    d[tb.dst[j]], bp[tb.dst[j]] = x, j

    d = np.full(S, np.inf); bp = np.full(S, -1); d[tb.start] = 0.0
    close(d, bp)
    bps = [bp]
    for t in range(ln):
        nd = np.full(S, np.inf); nbp = np.full(S, -1)
        for s in np.nonzero(np.isfinite(d))[0]:
            for j in range(tb.arc_off[s], tb.eps_off[s]):
                x = d[s] + tb.weight[j] - acs * float(y[t, tb.token[j]]) + (wps if tb.olabel[j] else 0.0)
                if x < nd[tb.dst[j]]:
                    nd[tb.dst[j]], nbp[tb.dst[j]] = x, j
        close(nd, nbp)
        d = nd
        bps.append(nbp)
    fc = d + tb.final.astype(np.float64)
    reached = bool(np.isfinite(fc).any())
    s = int(np.argmin(fc if reached else d))
    cost = float(fc[s] if reached else d[s])
    arcs, f = [], ln
    while bps[f][s] >= 0:
        j = int(bps[f][s])
        arcs.append(j)
        s = int(tb.src[j])
        if tb.token[j] >= 0:
            f -= 1
    arcs = arcs[::-1]
    return ([int(tb.olabel[a]) for a in arcs if tb.olabel[a]], [int(tb.token[a]) for a in arcs if tb.token[a] >= 0],
            cost, reached)


def write_graph(tmp_path, name, g):
    p = str(tmp_path / name)
    fst.write_fst(p, g)
    return p


def peaky(N, T, V, seed, lens=None):
    rng = np.random.default_rng(seed)
    y = rng.standard_normal((N, T, V)).astype(np.float32) * 2.0
    y = torch.log_softmax(torch.tensor(y), -1).numpy()
    return y, np.asarray(lens if lens is not None else [T] * N, np.int32)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the reader and its load checks
# ---------------------------------------------------------------------------------------------------------------------
def _py_derived(g: fst.DenGraph):
    """Levels, L, E, the largest emitting out-degree and the largest ilabel, recomputed from the file's arcs."""
    S = g.num_states
    eps = g.ilabel == 0
    succ, pred = [[] for _ in range(S)], [[] for _ in range(S)]
    for a, b in zip(g.src[eps].tolist(), g.dst[eps].tolist()):
        succ[a].append(b)
        pred[b].append(a)
    memo = {}

    def level(s):
        if s not in memo:
            memo[s] = max([0] + [level(p) + 1 for p in pred[s]])
        return memo[s]

    def reach(s):
        seen, st = set(), [s]
        while st:
            for b in succ[st.pop()]:
                if b not in seen:
                    seen.add(b)
                    st.append(b)
        return len(seen)
    lv = np.array([level(s) for s in range(S)])
    outdeg = np.bincount(g.src[~eps], minlength=S)
    return lv, int(lv.max()), max(reach(s) for s in range(S)), int(outdeg.max()), int(g.ilabel.max())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_reader_keeps_olabels_and_epsilons_and_derives_the_sizes(tmp_path, seed):
    g = random_wfst(60, 7, 20, seed, chain=6, dead_ends=3)
    p = write_graph(tmp_path, "g.fst", g)
    dg = DecodingGraph(p)
    t = dg.tables()
    fg = fst.read_fst(p)                          # file order: the Python reader's arc order
    A = fg.num_arcs
    assert (dg.num_states, dg.num_arcs, dg.start) == (fg.num_states, A, fg.start)
    assert dg.eps_arcs == int((fg.ilabel == 0).sum()) > 0
    inv = np.empty(A, np.int64)
    inv[t["fid"]] = np.arange(A)
    src = np.repeat(np.arange(fg.num_states), np.diff(t["arc_off"]))
    np.testing.assert_array_equal(src[inv], fg.src)
    np.testing.assert_array_equal(t["dst"][inv], fg.dst)
    np.testing.assert_array_equal(t["token"][inv], fg.ilabel - 1)
    np.testing.assert_array_equal(t["olabel"][inv], fg.olabel)
    np.testing.assert_array_equal(t["weight"][inv], fg.weight)
    np.testing.assert_array_equal(t["final"], fg.final)
    for s in range(fg.num_states):                # emitting arcs first, each class in file order
        a, e, b = t["arc_off"][s], t["eps_off"][s], t["arc_off"][s + 1]
        assert (t["token"][a:e] >= 0).all() and (t["token"][e:b] < 0).all()
        assert (np.diff(t["fid"][a:e]) > 0).all() and (np.diff(t["fid"][e:b]) > 0).all()
    level, L, E, D, il = _py_derived(fg)
    np.testing.assert_array_equal(t["level"], level)
    assert (dg.L, dg.E, dg.max_out, dg.max_ilabel) == (L, E, D, il)


def test_epsilon_cycle_is_refused_naming_a_state_on_it(tmp_path):
    g = random_wfst(30, 5, 4, 3, n_eps=0)
    cyc = [7, 12, 20]
    g.src = np.concatenate([g.src, cyc, [3]]).astype(np.int32)
    g.dst = np.concatenate([g.dst, cyc[1:] + cyc[:1], [7]]).astype(np.int32)
    g.ilabel = np.concatenate([g.ilabel, [0, 0, 0, 0]]).astype(np.int32)
    g.olabel = np.concatenate([g.olabel, [0, 2, 0, 0]]).astype(np.int32)
    g.weight = np.concatenate([g.weight, [0.1, 0.2, 0.3, 0.4]]).astype(np.float32)
    p = write_graph(tmp_path, "cyc.fst", g)
    with pytest.raises(RuntimeError, match=r"epsilon arcs of the decoding graph form a cycle through state (\d+)") as e:
        DecodingGraph(p)
    assert int(str(e.value).split("through state ")[1].split(";")[0]) in cyc
    g.src[-4:] = [5, 5, 5, 5]; g.dst[-4:] = [5, 6, 8, 9]          # a self loop is a cycle too
    with pytest.raises(RuntimeError, match="cycle through state 5"):
        DecodingGraph(write_graph(tmp_path, "self.fst", g))


def test_const_fst_symbol_tables_and_aligned_files_are_refused(tmp_path):
    p = write_graph(tmp_path, "g.fst", random_wfst(10, 3, 3, 0))
    raw = open(p, "rb").read()
    const = raw[:4] + struct.pack("<i", 5) + b"const" + raw[4 + 4 + 6:]
    (tmp_path / "c.fst").write_bytes(const)
    with pytest.raises(RuntimeError, match=r"is a const FST; convert it with `fstconvert --fst_type=vector`"):
        DecodingGraph(str(tmp_path / "c.fst"))
    off = 4 + 4 + 6 + 4 + 8 + 4          # magic, "vector", "standard", version: the flags
    for flags, msg in ((1, r"embedded symbol tables; strip them with `fstsymbols --clear_isymbols --clear_osymbols`"),
                       (2, r"embedded symbol tables"), (4, r"aligned fields; rewrite it with `fstconvert --fst_align=false`")):
        b = raw[:off] + struct.pack("<i", flags) + raw[off + 4:]
        (tmp_path / "f.fst").write_bytes(b)
        with pytest.raises(RuntimeError, match=msg):
            DecodingGraph(str(tmp_path / "f.fst"))
    with pytest.raises(RuntimeError, match="cannot open decoding graph"):
        DecodingGraph(str(tmp_path / "missing.fst"))


def test_den_reader_still_refuses_epsilons(tmp_path):
    """The den path keeps its behaviour: the same graph that loads as a decoding graph is refused as a den graph."""
    from cat_b200 import _lib
    import ctypes as C
    p = write_graph(tmp_path, "g.fst", random_wfst(10, 3, 3, 0))
    assert DecodingGraph(p).eps_arcs > 0
    L = _lib.lib()
    assert not L.ccb_plan_create(p.encode(), 4, 4)
    assert "epsilon input labels are not allowed" in _lib.last_error()


# ---------------------------------------------------------------------------------------------------------------------
# 2. make_tlg against textbook back-off
# ---------------------------------------------------------------------------------------------------------------------
def textbook_cost(grams, order, words, pron_cost):
    """The cheapest G cost of a word sequence from the ARPA n-grams: from history h, either the listed n-gram h.w (into the
    longest listed suffix of h.w) or the back-off weight of h and the same from h[1:]; </s> at the end.  Natural log."""
    ln10 = math.log(10)
    hists = {g for g in grams if len(g) < order and g[-1] != "</s>"} | {()}

    def state(ws):
        for j in range(len(ws) + 1):
            if ws[j:] in hists:
                return ws[j:]

    def step(h, w):                # {next history: cost} of word w from history h
        out = {}
        if h + (w,) in grams:
            out[state(h + (w,)) if w != "</s>" else None] = -grams[h + (w,)][0] * ln10
        if h:
            bow = -grams.get(h, (0, 0))[1] * ln10
            for k, v in step(state(h[1:]), w).items():
                out[k] = min(out.get(k, np.inf), bow + v)
        return out

    cur = {state(("<s>",)) if ("<s>",) in grams else (): 0.0}
    for w in list(words) + ["</s>"]:
        nxt = {}
        for h, c in cur.items():
            for nh, v in step(h, w).items():
                nxt[nh] = min(nxt.get(nh, np.inf), c + v)
        cur = nxt
    return min(cur.values()) + sum(pron_cost)


def constrained_cost(tb, align, word_ids):
    """The cheapest path of the graph whose emitting arcs read `align` and whose words are `word_ids`, in fp64."""
    order = np.argsort(tb.level, kind="stable")
    nW = len(word_ids)

    def close(d):
        for s in order:
            for k in range(nW + 1):
                if (s, k) not in d:
                    continue
                for j in range(tb.eps_off[s], tb.arc_off[s + 1]):
                    o = tb.olabel[j]
                    if o and (k == nW or o != word_ids[k]):
                        continue
                    key = (int(tb.dst[j]), k + (1 if o else 0))
                    d[key] = min(d.get(key, np.inf), d[(s, k)] + float(tb.weight[j]))
        return d

    d = close({(tb.start, 0): 0.0})
    for c in align:
        nd = {}
        for (s, k), v in d.items():
            for j in range(tb.arc_off[s], tb.eps_off[s]):
                o = tb.olabel[j]
                if tb.token[j] != c or (o and (k == nW or o != word_ids[k])):
                    continue
                key = (int(tb.dst[j]), k + (1 if o else 0))
                nd[key] = min(nd.get(key, np.inf), v + float(tb.weight[j]))
        d = close(nd)
    return min((v + float(tb.final[s]) for (s, k), v in d.items() if k == nW), default=np.inf)


def _ctc_align(prons, rng):
    """A CTC alignment of the concatenated pronunciations: blanks between repeats, random blank and repeat frames."""
    out, last = [], -1
    for x in [t for p in prons for t in p]:
        if x == last or rng.random() < 0.3:
            out += [0] * int(rng.integers(1, 3))
        out += [x] * int(rng.integers(1, 3))
        last = x
    return out + [0] * int(rng.integers(0, 2))


@pytest.mark.parametrize("order", [1, 2, 3])
def test_make_tlg_costs_textbook_backoff_plus_pronunciation(tmp_path, order):
    V = 6
    arpa = make_random_arpa(str(tmp_path / "w.arpa"), 9, order, [12, 10][:order - 1], seed=order)
    lex = tiny_lexicon(V, 7, seed=order)
    lex = [(w, p, 0.25 * i) for i, (w, p) in enumerate(lex)]
    g, words = fst.make_tlg(V, lex, arpa)
    p = write_graph(tmp_path, "tlg.fst", g)
    dg = DecodingGraph(p)
    tb = Tables(dg)
    assert dg.max_ilabel <= V and dg.eps_arcs > 0
    grams, _ = fst.read_arpa(arpa)
    rng = np.random.default_rng(order)
    wid = {w: i for i, w in enumerate(words)}
    n_prons = {w: sum(e[0] == w for e in lex) for w in wid}
    checked = 0
    for _ in range(40):
        seq = [lex[int(i)] for i in rng.integers(0, len(lex), size=int(rng.integers(1, 4)))]
        align = _ctc_align([e[1] for e in seq], rng)
        got = constrained_cost(tb, align, [wid[e[0]] for e in seq])
        want = textbook_cost(grams, order, [e[0] for e in seq], [e[2] for e in seq])
        assert got <= want + 1e-4, (seq, align)
        if all(n_prons[e[0]] == 1 for e in seq):   # another pronunciation of a word might read the alignment more cheaply
            assert got == pytest.approx(want, rel=1e-5, abs=1e-4), (seq, align)
            checked += 1
    assert checked >= 4


# ---------------------------------------------------------------------------------------------------------------------
# 3. the restatement against exhaustive Viterbi
# ---------------------------------------------------------------------------------------------------------------------
GRAPHS = [
    dict(S=40, V=5, W=9, seed=1, chain=5),
    dict(S=60, V=7, W=12, seed=2, chain=8, dead_ends=4),
    dict(S=25, V=4, W=5, seed=3, n_eps=40, chain=6),
    dict(S=50, V=6, W=8, seed=4, no_final=True, chain=3),
]


@pytest.mark.parametrize("spec", range(len(GRAPHS)))
@pytest.mark.parametrize("weights", [(1.0, 1.0, 0.0), (0.7, 1.3, -0.4), (1.5, 0.5, 0.8)])
def test_restatement_at_full_beam_equals_exhaustive_viterbi(tmp_path, spec, weights):
    g = random_wfst(**GRAPHS[spec])
    dg = DecodingGraph(write_graph(tmp_path, "g.fst", g))
    tb = Tables(dg)
    acwt, lmwt, wip = weights
    T = 9
    y, lens = peaky(5, T, GRAPHS[spec]["V"] + 1, seed=spec, lens=[T, T, 5, 1, 0])
    r = wfst_decode_ref(tb, y, lens, acwt, lmwt, wip, beam=np.inf, max_active=dg.num_states)
    for n in range(5):
        words, align, c, reached = viterbi_fp64(tb, y[n], lens[n], acwt, lmwt, wip)
        if not np.isfinite(c):
            assert r["num_words"][n] == -1 and r["cost"][n] == np.inf
            continue
        assert r["reached_final"][n] == int(reached)
        assert list(r["words"][n, :r["num_words"][n]]) == words and (r["words"][n, r["num_words"][n]:] == -1).all()
        assert list(r["align"][n, :lens[n]]) == align and (r["align"][n, lens[n]:] == -1).all()
        assert r["cost"][n] / lmwt == pytest.approx(c, rel=1e-5, abs=1e-4)


def test_restatement_prunes_and_still_finds_a_path(tmp_path):
    g = random_wfst(80, 6, 10, 7, chain=6)
    tb = Tables(DecodingGraph(write_graph(tmp_path, "g.fst", g)))
    y, lens = peaky(4, 12, 7, seed=5)
    full = wfst_decode_ref(tb, y, lens, beam=np.inf, max_active=80)
    for beam, K in ((4.0, 3), (8.0, 1), (2.0, 80)):
        r = wfst_decode_ref(tb, y, lens, beam=beam, max_active=K)
        live = r["num_words"] >= 0
        assert (r["cost"][live] >= full["cost"][live] - 1e-4).all()


# ---------------------------------------------------------------------------------------------------------------------
# 4. argument checks
# ---------------------------------------------------------------------------------------------------------------------
def test_argument_checks(tmp_path):
    dg = DecodingGraph(write_graph(tmp_path, "g.fst", random_wfst(10, 5, 3, 0)))
    ok = dict(acwt=1.0, lmwt=1.0, wip=0.0, beam=17.0, max_active=7000)
    check_decode_args(dg, 6, **ok)
    check_decode_args(dg, 6, **{**ok, "beam": math.inf, "max_active": 1 << 20, "acwt": 0.0})
    for k, v in (("max_active", 0), ("max_active", (1 << 20) + 1), ("max_active", 3.0), ("max_active", True),
                 ("beam", 0.0), ("beam", -1.0), ("beam", math.nan), ("acwt", -0.1), ("acwt", math.inf),
                 ("lmwt", 0.0), ("lmwt", math.inf), ("wip", math.inf), ("wip", math.nan)):
        with pytest.raises(ValueError, match=k):
            check_decode_args(dg, 6, **{**ok, k: v})
    assert dg.max_ilabel == 5
    with pytest.raises(ValueError, match="ilabels up to 5"):
        check_decode_args(dg, 4, **ok)
    with pytest.raises(ValueError, match="DecodingGraph"):
        check_decode_args("g.fst", 6, **ok)
    from cat_b200 import _lib
    L = _lib.lib()
    assert L.ccb_wfst_decode_ws_bytes(dg.handle, 1, 10, 0) == 0
    assert L.ccb_wfst_decode_ws_bytes(dg.handle, 1, 10, 7000) > 0
    # the native entry refuses the same values before it touches a device
    for args, msg in (((1.0, 1.0, 0.0, 17.0, 0), "max_active"), ((1.0, 1.0, 0.0, 0.0, 10), "beam"),
                      ((-1.0, 1.0, 0.0, 17.0, 10), "acwt"), ((1.0, 0.0, 0.0, 17.0, 10), "lmwt"),
                      ((1.0, 1.0, math.inf, 17.0, 10), "wip")):
        assert L.ccb_wfst_decode(1, 0, 1, 10, 6, 1, dg.handle, *args, 1, 1, 1, 1, 1, 1, 1, 1, None) != 0
        assert msg in _lib.last_error()
    assert L.ccb_wfst_decode(1, 0, 1, 10, 4, 1, dg.handle, 1.0, 1.0, 0.0, 17.0, 10, 1, 1, 1, 1, 1, 1, 1, 1, None) != 0
    assert "ilabels up to 5" in _lib.last_error()


def test_to_text_reads_the_word_table(tmp_path):
    dg = DecodingGraph(write_graph(tmp_path, "g.fst", random_wfst(10, 5, 3, 0)), words=None)
    (tmp_path / "words.txt").write_text("<eps> 0\nhello 1\nworld 2\n#0 3\n")
    dg2 = DecodingGraph(dg.path, words=str(tmp_path / "words.txt"))
    w = torch.tensor([[1, 2, 7, -1], [-1, -1, -1, -1], [2, -1, -1, -1]], dtype=torch.int32)
    nw = torch.tensor([3, -1, 1], dtype=torch.int32)
    assert dg2.to_text(w, nw) == [["hello", "world", "7"], None, ["world"]]
