"""Denominator-graph files: OpenFst binary ``vector``/``standard`` reader/writer (numpy)
and the synthetic T-compose-LM shaped generator used by tests and bench.py.

The product's loader is the C++ one in ``csrc/den_graph.cc`` (used by ``CRFContext``);
this module is the host-side tool for *producing* den graphs (tests, benchmarks) and an
independent second parser the tests cross-check the C++ reader against.

Reference semantics being mirrored (nothing is copied, OpenFst is not available here):
  * ``src/ctc_crf/gpu_den/fst_read.cc:40-60`` -- weight = -tropical, label = ilabel-1,
    start weight 0 on ``Start()``, end weight = -Final for non-Zero finals.
  * ``cat/utils/tool/build_ctc_topo.py:47-60`` -- CTC topology T: every arc *into* token
    state i carries ilabel i+1, arcs into the blank state carry ilabel 1.
File layout (little endian), decoded from ``src/ctc_crf/test/den_lm.fst`` (SURVEY.md 8c):
  int32 magic 0x7EB2FDD6 | str "vector" | str "standard" | int32 version(2) | int32 flags |
  uint64 properties | int64 start | int64 num_states | int64 num_arcs |
  per state: float32 final (inf = non-final), int64 narcs,
             narcs x {int32 ilabel, int32 olabel, float32 weight, int32 nextstate}
"""
from __future__ import annotations

import struct
from dataclasses import dataclass

import numpy as np

FST_MAGIC = 0x7EB2FDD6
# kExpanded | kMutable, and "not known" for everything else is acceptable to OpenFst readers
_DEFAULT_PROPERTIES = 0x0000000000000003


@dataclass
class DenGraph:
    """Arc list of a den graph in *file* convention (tropical weights, ilabel as stored)."""
    num_states: int
    start: int
    src: np.ndarray       # int32 [A]
    dst: np.ndarray       # int32 [A]
    ilabel: np.ndarray    # int32 [A]  (token id + 1)
    olabel: np.ndarray    # int32 [A]
    weight: np.ndarray    # float32 [A] tropical (-log p)
    final: np.ndarray     # float32 [S] tropical, +inf = non-final

    @property
    def num_arcs(self) -> int:
        return int(self.src.shape[0])

    # --- the view the loss uses (fst_read.cc:43-59) ---------------------------------
    def log_arcs(self):
        """(src, dst, label, logw) with label = ilabel-1 and logw = -weight."""
        return (self.src.astype(np.int32), self.dst.astype(np.int32),
                (self.ilabel - 1).astype(np.int32), (-self.weight).astype(np.float32))

    def start_weight(self) -> np.ndarray:
        w = np.full(self.num_states, -np.inf, dtype=np.float32)
        w[self.start] = 0.0
        return w

    def end_weight(self) -> np.ndarray:
        w = np.where(np.isinf(self.final), -np.inf, -self.final).astype(np.float32)
        return w


def _read_str(buf: bytes, off: int):
    (n,) = struct.unpack_from("<i", buf, off)
    off += 4
    return buf[off:off + n].decode("ascii"), off + n


def read_fst(path: str) -> DenGraph:
    buf = open(path, "rb").read()
    off = 0
    (magic,) = struct.unpack_from("<i", buf, off)
    off += 4
    if (magic & 0xFFFFFFFF) != FST_MAGIC:
        raise ValueError(f"{path}: not an OpenFst binary file (magic {magic & 0xFFFFFFFF:#x})")
    fst_type, off = _read_str(buf, off)
    arc_type, off = _read_str(buf, off)
    if fst_type != "vector" or arc_type != "standard":
        raise ValueError(f"{path}: unsupported fst/arc type {fst_type}/{arc_type}")
    version, flags = struct.unpack_from("<ii", buf, off)
    off += 8
    if flags & 0x3:
        raise ValueError(f"{path}: embedded symbol tables are not supported (flags={flags})")
    props, start, num_states, _num_arcs_hdr = struct.unpack_from("<Qqqq", buf, off)
    off += 32
    final = np.empty(num_states, dtype=np.float32)
    srcs, dsts, ils, ols, ws = [], [], [], [], []
    arc_dt = np.dtype([("il", "<i4"), ("ol", "<i4"), ("w", "<f4"), ("ns", "<i4")])
    for s in range(num_states):
        (f, narcs) = struct.unpack_from("<fq", buf, off)
        off += 12
        final[s] = f
        if narcs:
            a = np.frombuffer(buf, dtype=arc_dt, count=narcs, offset=off)
            off += 16 * narcs
            srcs.append(np.full(narcs, s, dtype=np.int32))
            dsts.append(a["ns"].astype(np.int32))
            ils.append(a["il"].astype(np.int32))
            ols.append(a["ol"].astype(np.int32))
            ws.append(a["w"].astype(np.float32))
    if off != len(buf):
        raise ValueError(f"{path}: trailing bytes ({len(buf) - off})")
    cat = (lambda xs, dt: np.concatenate(xs) if xs else np.zeros(0, dtype=dt))
    return DenGraph(num_states=int(num_states), start=int(start),
                    src=cat(srcs, np.int32), dst=cat(dsts, np.int32),
                    ilabel=cat(ils, np.int32), olabel=cat(ols, np.int32),
                    weight=cat(ws, np.float32), final=final)


def write_fst(path: str, g: DenGraph, properties: int = _DEFAULT_PROPERTIES) -> None:
    order = np.argsort(g.src, kind="stable")
    src = g.src[order]
    counts = np.bincount(src, minlength=g.num_states).astype(np.int64)
    offs = np.concatenate([[0], np.cumsum(counts)])
    arc_dt = np.dtype([("il", "<i4"), ("ol", "<i4"), ("w", "<f4"), ("ns", "<i4")])
    arcs = np.empty(g.num_arcs, dtype=arc_dt)
    arcs["il"] = g.ilabel[order]
    arcs["ol"] = g.olabel[order]
    arcs["w"] = g.weight[order]
    arcs["ns"] = g.dst[order]
    with open(path, "wb") as f:
        f.write(struct.pack("<I", FST_MAGIC))
        for s in (b"vector", b"standard"):
            f.write(struct.pack("<i", len(s)) + s)
        f.write(struct.pack("<ii", 2, 0))
        f.write(struct.pack("<Qqqq", properties, g.start, g.num_states, g.num_arcs))
        for s in range(g.num_states):
            f.write(struct.pack("<fq", float(g.final[s]), int(counts[s])))
            f.write(arcs[offs[s]:offs[s + 1]].tobytes())


def make_synthetic_den(H: int, d: int, V: int, seed: int = 7, p_final: float = 0.05) -> DenGraph:
    """T-compose-LM shaped den graph (SURVEY.md 8d).

    LM: H history states, state 0 = start (no last label), every h>0 has a last label
    l(h) in [1,V-1]; each h has d distinct successors h'!=0 with Dirichlet(1) probabilities
    (+ p_final for h>0).  Den states: (h,B) for all h, (h,L) for h>0  => S = 2H-1.
    Arcs (weight 0 unless stated): (h,L)->(h,L) label l(h); (h,L)->(h,B) blank;
    (h,B)->(h,B) blank; per LM arc h->h' (weight w): (h,B)->(h',L) and, when
    l(h') != l(h), (h,L)->(h',L), both with label l(h').  Finals on both twins.
    """
    rng = np.random.default_rng(seed)
    assert H >= 2 and V >= 2 and 1 <= d <= H - 1
    last = np.zeros(H, dtype=np.int32)
    last[1:] = rng.integers(1, V, size=H - 1)
    # successors: d distinct h' in [1,H-1] for each h (vectorised rejection-free draw)
    succ = rng.integers(1, H, size=(H, d), dtype=np.int64)
    while True:   # re-draw the (rare) rows that contain a duplicate successor
        srt = np.sort(succ, axis=1)
        bad = np.nonzero((srt[:, 1:] == srt[:, :-1]).any(axis=1))[0]
        if bad.size == 0:
            break
        succ[bad] = rng.integers(1, H, size=(bad.size, d), dtype=np.int64)
    probs = rng.dirichlet(np.ones(d), size=H)
    pf = np.where(np.arange(H) > 0, p_final, 0.0)
    probs = probs * (1.0 - pf)[:, None]
    w_lm = (-np.log(np.maximum(probs, 1e-30))).astype(np.float32)

    B = lambda h: 2 * h - (h > 0)          # (0,B)=0, (h,B)=2h-1
    L = lambda h: 2 * h                    # (h,L)=2h  for h>0
    S = 2 * H - 1
    hs = np.arange(H)
    hpos = np.arange(1, H)
    src, dst, lab, w = [], [], [], []
    # self loops / blank arcs
    src += [L(hpos), L(hpos), B(hs)]
    dst += [L(hpos), B(hpos), B(hs)]
    lab += [last[hpos], np.zeros(H - 1, np.int32), np.zeros(H, np.int32)]
    w += [np.zeros(H - 1, np.float32), np.zeros(H - 1, np.float32), np.zeros(H, np.float32)]
    # LM arcs
    hh = np.repeat(hs, d)
    hn = succ.reshape(-1)
    ww = w_lm.reshape(-1)
    src.append(B(hh)); dst.append(L(hn)); lab.append(last[hn]); w.append(ww)
    m = (hh > 0) & (last[hn] != last[hh])
    src.append(L(hh[m])); dst.append(L(hn[m])); lab.append(last[hn[m]]); w.append(ww[m])

    final = np.full(S, np.inf, dtype=np.float32)
    fw = np.float32(-np.log(p_final))
    final[B(hpos)] = fw
    final[L(hpos)] = fw
    src = np.concatenate(src).astype(np.int32)
    dst = np.concatenate(dst).astype(np.int32)
    lab = np.concatenate(lab).astype(np.int32)
    return DenGraph(num_states=S, start=0, src=src, dst=dst, ilabel=lab + 1, olabel=lab.copy(),
                    weight=np.concatenate(w).astype(np.float32), final=final)


def make_random_den(S: int, A: int, V: int, seed: int = 0, n_final: int = 2) -> DenGraph:
    """Unstructured random graph: in-arcs of a state may carry *different* labels
    (exercises the loader's state-splitting path; not T-compose-LM shaped)."""
    rng = np.random.default_rng(seed)
    src = rng.integers(0, S, size=A).astype(np.int32)
    dst = rng.integers(0, S, size=A).astype(np.int32)
    # keep the graph connected enough: a chain 0->1->...->S-1
    src[:S - 1] = np.arange(S - 1)
    dst[:S - 1] = np.arange(1, S)
    lab = rng.integers(0, V, size=A).astype(np.int32)
    w = rng.uniform(0.1, 3.0, size=A).astype(np.float32)
    final = np.full(S, np.inf, dtype=np.float32)
    final[rng.choice(S, size=min(n_final, S), replace=False)] = 0.7
    final[S - 1] = 0.3
    return DenGraph(num_states=S, start=0, src=src, dst=dst, ilabel=lab + 1, olabel=lab.copy(),
                    weight=w, final=final)


# ---------------------------------------------------------------------------------------------------
# Den-graph construction without Kaldi/OpenFst (SURVEY.md 8f-2): T o LM for an epsilon-free phone LM
# ---------------------------------------------------------------------------------------------------
@dataclass
class PhoneLm:
    """Epsilon-free weighted acceptor over phone ids 1..V-1 (0 is the CTC blank and never appears):
    what ``chain-est-phone-lm`` produces for ``cat/utils/tool/prep_den_lm.sh:40-45`` (no back-off arcs)."""
    num_states: int
    start: int
    src: np.ndarray      # int32 [A]
    dst: np.ndarray      # int32 [A]
    phone: np.ndarray    # int32 [A] in [1, V-1]
    weight: np.ndarray   # float32 [A] tropical (-log p)
    final: np.ndarray    # float32 [S] tropical, +inf = non-final


def compose_ctc_lm(lm: PhoneLm) -> DenGraph:
    """den graph = T o LM, with T the CTC topology of ``cat/utils/tool/build_ctc_topo.py:47-66`` (state 0 = blank,
    state i = token i; every arc INTO token state i reads label i and emits phone i, arcs into the blank state and
    token self loops emit nothing), i.e. the composition ``prep_den_lm.sh:46-51`` performs with OpenFst.

    States of the result: (h,B) "LM state h, last frame was blank or nothing yet" for every reachable h, and (h,i)
    "LM state h reached by phone i, last frame was i" for every phone i entering h.  Because T emits a phone exactly
    when a token state is entered, the composition needs no epsilon handling for an epsilon-free LM, and for a
    deterministic LM the result is already deterministic (what fstdeterminizestar would return up to state order)."""
    S, A = lm.num_states, int(lm.src.shape[0])
    # token states: one per distinct (destination, phone)
    key = lm.dst.astype(np.int64) * (int(lm.phone.max(initial=0)) + 1) + lm.phone
    uniq, tok_of_arc = np.unique(key, return_inverse=True)
    n_tok = int(uniq.shape[0])
    tok_h = (uniq // (int(lm.phone.max(initial=0)) + 1)).astype(np.int32)
    tok_p = (uniq % (int(lm.phone.max(initial=0)) + 1)).astype(np.int32)
    B = lambda h: np.asarray(h, np.int64)                   # (h,B) -> h
    TK = lambda k: S + np.asarray(k, np.int64)             # token state k -> S + k
    src, dst, lab, w = [], [], [], []
    hs = np.arange(S)
    ks = np.arange(n_tok)
    # blank self loop, token self loop, token -> blank
    src += [B(hs), TK(ks), TK(ks)]
    dst += [B(hs), TK(ks), B(tok_h)]
    lab += [np.zeros(S, np.int32), tok_p, np.zeros(n_tok, np.int32)]
    w += [np.zeros(S, np.float32), np.zeros(n_tok, np.float32), np.zeros(n_tok, np.float32)]
    # per LM arc h -p-> h': from (h,B), and from every token state (h,i) with i != p
    src.append(B(lm.src)); dst.append(TK(tok_of_arc)); lab.append(lm.phone); w.append(lm.weight)
    by_h = [[] for _ in range(S)]
    for k in range(n_tok):
        by_h[int(tok_h[k])].append(k)
    s2, d2, l2, w2 = [], [], [], []
    for a in range(A):
        for k in by_h[int(lm.src[a])]:
            if tok_p[k] != lm.phone[a]:
                s2.append(S + k); d2.append(S + int(tok_of_arc[a])); l2.append(int(lm.phone[a])); w2.append(float(lm.weight[a]))
    src.append(np.asarray(s2, np.int64)); dst.append(np.asarray(d2, np.int64))
    lab.append(np.asarray(l2, np.int32)); w.append(np.asarray(w2, np.float32))
    src = np.concatenate(src); dst = np.concatenate(dst)
    lab = np.concatenate(lab).astype(np.int32); w = np.concatenate(w).astype(np.float32)
    final = np.concatenate([lm.final, lm.final[tok_h]]).astype(np.float32)
    # keep what is reachable from (start,B), renumbered in discovery order
    n_all = S + n_tok
    order = np.argsort(src, kind="stable")
    starts = np.searchsorted(src[order], np.arange(n_all + 1))
    new_id = np.full(n_all, -1, np.int64)
    new_id[lm.start] = 0
    stack, n_new = [int(lm.start)], 1
    while stack:
        q = stack.pop()
        for a in order[starts[q]:starts[q + 1]]:
            t = int(dst[a])
            if new_id[t] < 0:
                new_id[t] = n_new; n_new += 1; stack.append(t)
    keep = new_id[src] >= 0
    inv = np.argsort(np.where(new_id >= 0, new_id, n_all), kind="stable")[:n_new]
    return DenGraph(num_states=n_new, start=0, src=new_id[src[keep]].astype(np.int32), dst=new_id[dst[keep]].astype(np.int32),
                    ilabel=(lab[keep] + 1).astype(np.int32), olabel=lab[keep].copy(), weight=w[keep], final=final[inv])


def lm_logprob(lm: PhoneLm, phones) -> float:
    """log p_LM(l) of one phone sequence under a deterministic LM (the per-utterance path weight CAT adds to the
    numerator, docs/toolkitworkflow.md:124-135); -inf if the LM does not accept it."""
    h, lp = int(lm.start), 0.0
    for p in phones:
        m = np.nonzero((lm.src == h) & (lm.phone == int(p)))[0]
        if m.size == 0:
            return float("-inf")
        assert m.size == 1, "lm_logprob needs a deterministic LM"
        lp -= float(lm.weight[m[0]]); h = int(lm.dst[m[0]])
    return lp - float(lm.final[h]) if np.isfinite(lm.final[h]) else float("-inf")


def make_random_lm(H: int, V: int, d: int, seed: int = 0, p_final: float = 0.2) -> PhoneLm:
    """Small deterministic phone LM for tests: every state has d out-arcs with distinct phones, random targets."""
    rng = np.random.default_rng(seed)
    assert 1 <= d <= V - 1
    src, dst, ph, w = [], [], [], []
    final = np.full(H, np.inf, np.float32)
    for h in range(H):
        fin = h > 0 and rng.random() < 0.7
        pr = rng.dirichlet(np.ones(d)) * (1.0 - (p_final if fin else 0.0))
        for p, q in zip(rng.choice(np.arange(1, V), size=d, replace=False), pr):
            src.append(h); dst.append(int(rng.integers(0, H))); ph.append(int(p)); w.append(-np.log(q))
        if fin:
            final[h] = -np.log(p_final)
    return PhoneLm(H, 0, np.asarray(src, np.int32), np.asarray(dst, np.int32), np.asarray(ph, np.int32),
                   np.asarray(w, np.float32), final)


# ---------------------------------------------------------------------------------------------------
# Decoding graphs without Kaldi/OpenFst: a TLG-shaped graph for the word decoder (csrc/wfst_decode.cu)
# ---------------------------------------------------------------------------------------------------
_LN10 = 2.302585092994045684


def read_arpa(path: str):
    """The n-grams of an ARPA file: {tuple of words: (log10 p, log10 bow)} (bow 0 when the line has none), and the order."""
    grams, order, k = {}, 0, 0
    with open(path) as f:
        for line in f:
            p = line.split()
            if not p:
                continue
            if p[0].startswith("\\"):
                k = int(p[0][1:].split("-")[0]) if p[0].endswith("-grams:") else 0
                continue
            if p[0] == "ngram" and k == 0:
                order = max(order, int(p[1].split("=")[0]))
                continue
            if k:
                words = tuple(p[1:1 + k])
                grams.setdefault(words, (float(p[0]), float(p[1 + k]) if len(p) > k + 1 else 0.0))
    return grams, order


def make_tlg(V: int, lexicon, arpa_path: str):
    """A TLG-shaped decoding graph built without OpenFst: T o L o G in CAT's conventions (ilabel = token + 1, blank = token 0,
    ilabel 0 = epsilon, olabel = word id).  Returns (DenGraph, words) with words[i] the word of id i (words[0] = "<eps>").

    lexicon: (word, tokens) or (word, tokens, cost) entries, tokens in 1..V-1; a word may have several pronunciations.  Word
    ids follow the lexicon's order from 1.  ARPA words the lexicon does not list are left out of G.
    G follows arpa2fst: a state per history (the root, every n-gram below the top order that does not end in </s>), an arc
    per n-gram into the longest suffix of its words that is a state, a back-off arc (epsilon, the `#0` arc once T o is
    applied) into the longest proper suffix, </s> as the final cost, costs in natural log (-ln 10 log10).  The start state is
    <s>'s (the root when the file lists none).
    L is a token trie of pronunciations per G state over the words that state has arcs for, as det(L o G) shares prefixes:
    the arc completing a word carries it (into the G destination) when nothing else ends or continues at its node; else the
    node has an epsilon arc per word ending there.  This keeps the out-degree near V.
    T is CAT's CTC topology (cat/utils/tool/build_ctc_topo.py): every state of LG becomes a blank state and one state per
    token entering it (through an emitting arc, or carried along epsilon arcs); a token state repeats its token in place,
    goes to the blank state on blank, and takes LG's arcs of other tokens; the blank state takes every LG arc.
    The graph is not minimised."""
    grams, order = read_arpa(arpa_path)
    words = ["<eps>"]
    wid, prons = {}, {}
    for e in lexicon:
        w, toks, c = (e[0], e[1], e[2]) if len(e) == 3 else (e[0], e[1], 0.0)
        toks = tuple(int(x) for x in toks)
        if not toks or min(toks) < 1 or max(toks) >= V:
            raise ValueError(f"make_tlg: the pronunciation {toks} of {w!r} must be non-empty tokens in 1..{V - 1}")
        if w not in wid:
            wid[w] = len(words)
            words.append(w)
        prons.setdefault(w, []).append((toks, float(c)))
    # G
    hist = sorted({g for g in grams if len(g) < order and g[-1] != "</s>"} | {()}, key=lambda g: (len(g), g))
    gid = {h: i for i, h in enumerate(hist)}

    def state_of(ws):            # the longest suffix of ws that is a state
        for j in range(len(ws) + 1):
            if ws[j:] in gid:
                return gid[ws[j:]]

    g_arcs = [[] for _ in hist]  # per G state: (word, dst, cost)
    g_final = np.full(len(hist), np.inf)
    for ng, (p, _) in grams.items():
        h, w = ng[:-1], ng[-1]
        if h not in gid:
            if len(h) > 0 and any(x not in wid and x not in ("<s>", "</s>") for x in h):
                continue
            raise ValueError(f"make_tlg: the history {h} of an n-gram is not listed in {arpa_path}")
        if w == "</s>":
            g_final[gid[h]] = -p * _LN10
        elif w in wid:
            g_arcs[gid[h]].append((w, state_of(ng), -p * _LN10))
    start_g = gid.get(("<s>",), 0)
    # LG: G states first, then trie nodes; arcs (src, dst, token (-1: epsilon), word id, cost)
    src, dst, tok, olab, cost = [], [], [], [], []
    n_lg = len(hist)
    for g, arcs in enumerate(g_arcs):
        child = {}               # (node, token) -> node
        ends = {}                # node -> [(word id, dst, cost)]
        for w, d, c in arcs:
            for toks, pc in prons[w]:
                node = g
                for x in toks:
                    nx = child.get((node, x))
                    if nx is None:
                        nx = child[(node, x)] = n_lg
                        n_lg += 1
                    node = nx
                ends.setdefault(node, []).append((wid[w], d, c + pc))
        has_child = {node for node, _ in child}
        for (node, x), nx in child.items():
            e = ends.get(nx, [])
            if len(e) == 1 and nx not in has_child:      # the arc completes one word: it carries the word
                src.append(node); dst.append(e[0][1]); tok.append(x); olab.append(e[0][0]); cost.append(e[0][2])
            else:
                src.append(node); dst.append(nx); tok.append(x); olab.append(0); cost.append(0.0)
                for w, d, c in e:
                    src.append(nx); dst.append(d); tok.append(-1); olab.append(w); cost.append(c)
        if len(hist[g]) > 0:     # back-off
            h = hist[g]
            src.append(g); dst.append(state_of(h[1:])); tok.append(-1); olab.append(0)
            cost.append(-grams.get(h, (0.0, 0.0))[1] * _LN10)
    src, dst, tok, olab = (np.asarray(a, np.int64) for a in (src, dst, tok, olab))
    cost = np.asarray(cost, np.float64)
    lg_final = np.concatenate([g_final, np.full(n_lg - len(hist), np.inf)])
    # T o LG: the tokens of each LG state (entering through emitting arcs, carried along epsilon arcs; LG's epsilon arcs go
    # from trie nodes to G states and from G states to shorter histories, so that order is topological)
    toks_of = [set() for _ in range(n_lg)]
    em = tok >= 0
    for d, x in zip(dst[em].tolist(), tok[em].tolist()):
        toks_of[d].add(x)
    eps = np.nonzero(~em)[0]
    rank = np.array([-len(h) for h in hist] + [-order - 1] * (n_lg - len(hist)))
    for a in eps[np.argsort(rank[src[eps]], kind="stable")].tolist():
        toks_of[dst[a]] |= toks_of[src[a]]
    # CTC states grouped by LG state: blank first (key 0), then tokens ascending (key token + 1)
    cnt = np.array([1 + len(t) for t in toks_of], np.int64)
    off = np.concatenate([[0], np.cumsum(cnt)])
    ckey = np.concatenate([np.array([0] + sorted(x + 1 for x in t), np.int64) for t in toks_of])
    cstate = np.repeat(np.arange(n_lg), cnt)
    glob = cstate * (V + 1) + ckey        # sorted
    S = int(off[-1])

    def cid(x, k):
        return np.searchsorted(glob, x * (V + 1) + k)

    ar = np.arange(S)
    out_s, out_d, out_i, out_o, out_w = [], [], [], [], []
    # blank self loop on blank states, token self loop and token -> blank on token states
    isb = ckey == 0
    out_s += [ar[isb], ar[~isb], ar[~isb]]
    out_d += [ar[isb], ar[~isb], off[cstate[~isb]]]
    out_i += [np.ones(int(isb.sum()), np.int64), ckey[~isb], np.ones(int((~isb).sum()), np.int64)]
    out_o += [np.zeros(S, np.int64)]
    out_w += [np.zeros(S + int((~isb).sum()))]
    out_o += [np.zeros(int((~isb).sum()), np.int64)]
    # LG arcs from every CTC state of their source: emitting ones skip the token state of their own token
    rep = cnt[src]
    a_idx = np.repeat(np.arange(len(src)), rep)
    c_idx = off[src[a_idx]] + (np.arange(int(rep.sum())) - np.repeat(np.cumsum(rep) - rep, rep))
    keep = ~((tok[a_idx] >= 0) & (ckey[c_idx] == tok[a_idx] + 1))
    a_idx, c_idx = a_idx[keep], c_idx[keep]
    e = tok[a_idx] >= 0
    d_em = cid(dst[a_idx], tok[a_idx] + 1)
    d_ep = cid(dst[a_idx], ckey[c_idx])
    out_s.append(c_idx); out_d.append(np.where(e, d_em, d_ep)); out_i.append(np.where(e, tok[a_idx] + 1, 0))
    out_o.append(olab[a_idx]); out_w.append(cost[a_idx])
    s_ = np.concatenate(out_s); d_ = np.concatenate(out_d)
    order_ = np.argsort(s_, kind="stable")
    final = lg_final[cstate].astype(np.float32)
    g = DenGraph(num_states=S, start=int(off[start_g]), src=s_[order_].astype(np.int32), dst=d_[order_].astype(np.int32),
                 ilabel=np.concatenate(out_i)[order_].astype(np.int32), olabel=np.concatenate(out_o)[order_].astype(np.int32),
                 weight=np.concatenate(out_w)[order_].astype(np.float32), final=final)
    return g, words
