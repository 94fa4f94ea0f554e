"""CPU side of the prefix beam search (``ctc_crf.ctc_beam_search``): argument checks, the out-arc CSR and the CTC-shape
check of a den plan, the ``CTCBeamDecoder`` options, and a numpy restatement of the search (fp64, the kernel's candidate
rules and tie keys) checked against exhaustive enumeration; tests/test_gpu_beam.py compares the kernel against it."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from cat_b200 import _C, _lib, fst

NEG = -np.inf


# ---------------------------------------------------------------------------------------------------------------------
# the plan's beam-search view
# ---------------------------------------------------------------------------------------------------------------------
def plan_out(path, n_ctas=132, n_warps=16):
    """Out-arc CSR, labels, finals and start of a den plan, and the result of its CTC-shape check (None: passes, else the
    message)."""
    L = _lib.lib()
    h = L.ccb_plan_create(path.encode(), n_ctas, n_warps)
    assert h, _lib.last_error()
    try:
        info = (C.c_long * 13)()
        assert L.ccb_plan_info(h, info) == 0
        S, start = int(info[2]), int(info[5])

        def get(which, dtype, count):
            a = np.empty(count, dtype=dtype)
            assert L.ccb_plan_copy(h, which, a.ctypes.data_as(C.c_void_p), a.nbytes) == 0
            return a
        out_off = get(22, np.int32, S + 1)
        A = int(out_off[-1])
        shape = None if L.ccb_plan_ctc_shape(h) == 0 else _lib.last_error()
        return dict(S=S, start=start, out_off=out_off, out_dst=get(23, np.int32, A), out_w=get(24, np.float32, A),
                    state_label=get(0, np.int32, S), final_lin=get(1, np.float32, S), orig_state=get(2, np.int32, S),
                    shape=shape)
    finally:
        L.ccb_plan_destroy(h)


# ---------------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------------
def lse(a, b):
    """The kernel's log-add: the larger plus log1p(exp(smaller - larger)), the larger alone when the smaller is -inf."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    m, o = np.maximum(a, b), np.minimum(a, b)
    with np.errstate(invalid="ignore"):
        r = m + np.log1p(np.exp(o - m))
    return np.where(o == NEG, m, r)


class _Steps:
    """Step(s, c): log w and destination of the out-arc of state s into a state of label c (-inf, -1: none); plain mode
    (G None): 0 and -1 for every step."""

    def __init__(self, G, V):
        self.G = G
        if G is not None:
            S = G["S"]
            self.tab = np.full((S, V), -1, np.int64)
            src = np.repeat(np.arange(S), np.diff(G["out_off"]))
            self.tab[src, G["state_label"][G["out_dst"]]] = np.arange(len(src))
            self.lw = np.log(G["out_w"].astype(np.float64))

    def __call__(self, s, c):
        s, c = np.asarray(s, np.int64), np.asarray(c, np.int64)
        if self.G is None:
            return np.zeros(np.broadcast(s, c).shape), np.full(np.broadcast(s, c).shape, -1, np.int64)
        idx = np.where((s >= 0) & (c >= 0), self.tab[np.maximum(s, 0), np.maximum(c, 0)], -1)
        with np.errstate(divide="ignore"):
            lw = np.where(idx >= 0, self.lw[np.maximum(idx, 0)], NEG)
        return lw, np.where(idx >= 0, self.G["out_dst"][np.maximum(idx, 0)], -1)


def _ext_in(step, mb, mt, sb, st, last, r, c):
    lw1, d1 = step(sb[r], c)
    lw2, d2 = step(st[r], c)
    a = mb[r] + lw1
    b = np.where(c != last[r], mt[r] + lw2, NEG)
    return lse(a, b), np.where(a > NEG, d1, d2)


def _near(a, b, tol):
    return abs(a - b) <= tol * max(1.0, abs(a))


def beam_ref(y, lens, B, topn, G=None, tol=1e-9):
    """The search restated in numpy.  y (N,T,V) float32 values, G: ``plan_out`` of the den graph for crf mode.
    Returns (tokens (N,B,T), lengths (N,B), timesteps (N,B,T), scores (N,B) fp64, near (N,) bool: the utterance met a
    candidate tie within tol at a pruning boundary or in the final ranking, where the kernel's fp64 may order otherwise)."""
    y = np.asarray(y, np.float32)
    N, T, V = y.shape
    step = _Steps(G, V)
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
        sb = np.array([G["start"] if G is not None else -1]); st = np.array([-1])
        rank = {0: 0}
        for t in range(int(lens[n])):
            yr = y[n, t].astype(np.float64)
            nb = len(node)
            if topn < V:
                toks = np.lexsort((np.arange(V), -yr))[:topn]
            else:
                toks = np.arange(V)
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
            # stay candidates
            rr = np.arange(nb)
            lw1, d1 = step(sb, 0)
            lw2, d2 = step(st, 0)
            a, b = mb + lw1, mt + lw2
            bin_ = lse(a, b)
            sbn = np.where(bin_ > NEG, np.where(a > NEG, d1, d2), -1)
            mbn = np.where(bin_ > NEG, bin_ + yr[0], NEG)
            lw3, d3 = step(st, last)
            rep = np.where(last >= 1, mt + lw3, NEG)
            pe = np.maximum(par, 0)
            ein, d4 = _ext_in(step, mb, mt, sb, st, last, pe, last)
            ext = np.where(par >= 0, ein, NEG)
            d4 = np.where(par >= 0, d4, -1)
            tin = lse(rep, ext)
            ok = (last >= 1) & (tin > NEG)
            mtn = np.where(ok, tin + yr[np.maximum(last, 0)], NEG)
            stn = np.where(ok, np.where(rep > NEG, d3, d4), -1)
            m_stay = lse(mbn, mtn)
            k_stay = rr * (V + 1)
            # extension candidates: the frame's tokens but blank, and each entry's own last token
            R = np.repeat(rr, len(toks))
            Cc = np.tile(toks, nb)
            extra = (last >= 1) & ~flag[np.maximum(last, 0)]
            R = np.concatenate([R, rr[extra]])
            Cc = np.concatenate([Cc, last[extra]])
            keep = (Cc >= 1) & ~np.isin(R * (V + 1) + Cc, list(merged))
            R, Cc = R[keep], Cc[keep]
            ein, dst = _ext_in(step, mb, mt, sb, st, last, R, Cc)
            m_ext = np.where(ein > NEG, ein + yr[Cc], NEG)
            M = np.concatenate([m_stay, m_ext])
            K = np.concatenate([k_stay, R * (V + 1) + Cc + 1])
            fin = M > NEG
            M, K = M[fin], K[fin]
            order = np.lexsort((K, -M))
            if len(order) > B and _near(M[order[B - 1]], M[order[B]], tol):
                near[n] = True
            win = order[:B]
            n_node, n_last, n_mb, n_mt, n_sb, n_st = [], [], [], [], [], []
            for i in win:
                key = int(K[i])
                r, c = key // (V + 1), key % (V + 1) - 1
                if c < 0:
                    n_node.append(int(node[r])); n_last.append(int(last[r]))
                    n_mb.append(mbn[r]); n_sb.append(int(sbn[r])); n_mt.append(mtn[r]); n_st.append(int(stn[r]))
                else:
                    e, d = _ext_in(step, mb, mt, sb, st, last, np.array([r]), np.array([c]))
                    x = trie.get((int(node[r]), c))
                    if x is None:
                        x = len(parent)
                        parent.append(int(node[r])); tok.append(c); frame.append(t)
                        trie[(int(node[r]), c)] = x
                    n_node.append(x); n_last.append(c)
                    n_mb.append(NEG); n_sb.append(-1); n_mt.append(float(e[0]) + yr[c]); n_st.append(int(d[0]))
            node, last = np.array(n_node, np.int64), np.array(n_last, np.int64)
            mb, mt = np.array(n_mb, np.float64), np.array(n_mt, np.float64)
            sb, st = np.array(n_sb, np.int64), np.array(n_st, np.int64)
            rank = {int(x): k for k, x in enumerate(node)}
        if G is not None:
            fl = G["final_lin"].astype(np.float64)
            with np.errstate(divide="ignore"):
                fa = np.where(sb >= 0, mb + np.log(fl[np.maximum(sb, 0)]), NEG)
                fb = np.where(st >= 0, mt + np.log(fl[np.maximum(st, 0)]), NEG)
            fs = lse(fa, fb)
        else:
            fs = lse(mb, mt)
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


def hyps(tokens, lengths, scores, n):
    """{label sequence: score} of utterance n's finite rows."""
    return {tuple(tokens[n, k, :lengths[n, k]].tolist()): float(scores[n, k]) for k in range(lengths.shape[1]) if lengths[n, k] >= 0}


# ---------------------------------------------------------------------------------------------------------------------
# exhaustive enumeration
# ---------------------------------------------------------------------------------------------------------------------
def _collapse(path):
    return tuple(int(l) for j, l in enumerate(path) if l != 0 and (j == 0 or path[j - 1] != l))


def enum_plain(y, T):
    """{label sequence: log sum over the frame-label paths that collapse to it} of one (T,V) utterance."""
    V = y.shape[1]
    out = {}
    for path in itertools.product(range(V), repeat=T):
        s = float(sum(float(y[t, path[t]]) for t in range(T)))
        k = _collapse(path)
        out[k] = np.logaddexp(out.get(k, NEG), s)
    return out


def enum_crf(G, y, T):
    """{label sequence: log sum over the den-graph state paths (start arc, arc weights, emissions, final) that collapse to it}."""
    S, off, dst, w, lab = G["S"], G["out_off"], G["out_dst"], G["out_w"].astype(np.float64), G["state_label"]
    fin = G["final_lin"].astype(np.float64)
    out = {}
    act = [(G["start"], (), 0.0)]          # (state, frame labels, log weight)
    for t in range(T):
        nxt = []
        for q, labs, lw in act:
            for i in range(off[q], off[q + 1]):
                if w[i] > 0:
                    d = int(dst[i])
                    nxt.append((d, labs + (int(lab[d]),), lw + np.log(w[i]) + float(y[t, lab[d]])))
        act = nxt
    for q, labs, lw in act:
        if fin[q] > 0:
            k = _collapse(labs)
            out[k] = np.logaddexp(out.get(k, NEG), lw + np.log(fin[q]))
    return out


def _logsoftmax(x):
    return (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)


@pytest.mark.parametrize("T,V,seed", [(1, 3, 0), (4, 3, 1), (5, 4, 2), (6, 4, 3)])
def test_restatement_is_exact_at_full_beam_plain(T, V, seed):
    from oracle import oracle
    rng = np.random.default_rng(seed)
    y = _logsoftmax(rng.standard_normal((1, T, V)) * 1.5)
    want = enum_plain(y[0], T)
    B = 4000
    tokens, lengths, stamps, scores, near = beam_ref(y, [T], B, V)
    got = hyps(tokens, lengths, scores, 0)
    assert set(got) == set(want)
    for k, v in want.items():
        assert abs(got[k] - v) <= 1e-12 * max(1, abs(v)), (k, got[k], v)
        lp, _ = oracle.ctc(y, np.asarray(k, np.int32), [len(k)], [T], want_grad=False)
        assert abs(got[k] - lp[0]) <= 1e-5 * max(1, abs(lp[0])), (k, got[k], lp[0])
    # best first, and a smaller beam keeps a prefix of the ranking's top where nothing is near a tie
    assert np.all(np.diff(scores[0, :lengths.shape[1]][lengths[0] >= 0]) <= 0)
    for b in (1, 3):
        t2, l2, _, s2, nr = beam_ref(y, [T], b, V)
        assert np.all(s2[0][l2[0] >= 0] <= scores[0, :b][l2[0] >= 0] + 1e-12)


def _tiny_tlm(tmp_path, H, V, d, seed):
    lm = fst.make_random_lm(H=H, V=V, d=d, seed=seed)
    p = str(tmp_path / f"tlm_{H}_{V}_{seed}.fst")
    fst.write_fst(p, fst.compose_ctc_lm(lm))
    return lm, p


@pytest.mark.parametrize("T,V,seed", [(3, 3, 4), (5, 4, 5), (6, 3, 6)])
def test_restatement_is_exact_at_full_beam_crf(tmp_path, T, V, seed):
    from oracle import oracle
    lm, p = _tiny_tlm(tmp_path, 3, V, 2, seed)
    G = plan_out(p)
    assert G["shape"] is None
    rng = np.random.default_rng(seed)
    y = _logsoftmax(rng.standard_normal((1, T, V)) * 1.5)
    want = enum_crf(G, y[0], T)
    tokens, lengths, stamps, scores, near = beam_ref(y, [T], 4000, V, G)
    got = hyps(tokens, lengths, scores, 0)
    assert set(got) == set(want)
    for k, v in want.items():
        assert abs(got[k] - v) <= 1e-12 * max(1, abs(v)), (k, got[k], v)
        # T o LM: log p_LM(l) + log p_ctc(l|x)
        lp, _ = oracle.ctc(y, np.asarray(k, np.int32), [len(k)], [T], want_grad=False)
        assert abs(got[k] - (fst.lm_logprob(lm, k) + lp[0])) <= 1e-5 * max(1, abs(v)), k


def test_restatement_timesteps_and_empty_utterance(tmp_path):
    y = _logsoftmax(np.random.default_rng(0).standard_normal((2, 6, 4)))
    tokens, lengths, stamps, scores, near = beam_ref(y, [6, 0], 8, 4)
    assert lengths[1, 0] == 0 and scores[1, 0] == 0.0 and np.all(lengths[1, 1:] == -1) and np.all(np.isneginf(scores[1, 1:]))
    for k in range(8):
        L = lengths[0, k]
        if L > 0:
            ts = stamps[0, k, :L]
            assert np.all(np.diff(ts) > 0) and ts[0] >= 0 and ts[-1] < 6 and np.all(stamps[0, k, L:] == -1)
    lm, p = _tiny_tlm(tmp_path, 3, 4, 2, 1)
    G = plan_out(p)
    _, l2, _, s2, _ = beam_ref(y, [0, 0], 4, 4, G)
    with np.errstate(divide="ignore"):
        f = float(np.log(np.float64(G["final_lin"][G["start"]])))
    assert (l2[:, 0] == (0 if np.isfinite(f) else -1)).all()
    if np.isfinite(f):
        assert s2[0, 0] == f


# ---------------------------------------------------------------------------------------------------------------------
# the out-arc CSR and the CTC-shape check
# ---------------------------------------------------------------------------------------------------------------------
def _check_out_csr(path, g):
    G = plan_out(path)
    S, off, dst, w, lab, orig = G["S"], G["out_off"], G["out_dst"], G["out_w"], G["state_label"], G["orig_state"]
    assert off[0] == 0 and np.all(np.diff(off) >= 0) and dst.min() >= 0 and dst.max() < S
    src = np.repeat(np.arange(S), np.diff(off))
    # every split-graph arc once: a file arc p -> q of label l is an arc from every copy of p into the copy of q of label l
    copies = {}
    for s in range(S):
        copies.setdefault(int(orig[s]), []).append(s)
    want = []
    for p, q, l, x in zip(*g.log_arcs()):
        qs = [s for s in copies[int(q)] if lab[s] == l]
        assert len(qs) == 1
        want += [(ps, qs[0], float(np.float32(np.exp(np.float32(x))))) for ps in copies[int(p)]]
    got = sorted(zip(src.tolist(), dst.tolist(), w.tolist()))
    want = sorted(want)
    assert [(a, b) for a, b, _ in got] == [(a, b) for a, b, _ in want]
    np.testing.assert_allclose([c for _, _, c in got], [c for _, _, c in want], rtol=1e-6, atol=0)
    # sorted by destination label within each state
    for s in range(S):
        labs = lab[dst[off[s]:off[s + 1]]]
        assert np.all(np.diff(labs) >= 0)
    return G


def test_out_arc_csr_lists_every_split_arc_once_sorted_by_label(tmp_graphs, fixture_fst, tmp_path):
    for name in ("tlm_small", "random_split"):
        path, g, _ = tmp_graphs[name]
        _check_out_csr(path, g)
    _check_out_csr(fixture_fst, fst.read_fst(fixture_fst))
    lm, p = _tiny_tlm(tmp_path, 4, 5, 3, 2)
    _check_out_csr(p, fst.read_fst(p))


def test_ctc_shape_holds_on_deterministic_t_compose_lm_graphs(fixture_fst, tmp_path):
    assert plan_out(fixture_fst)["shape"] is None
    for H, V, d, seed in [(2, 3, 2, 4), (5, 6, 3, 1), (40, 30, 8, 2)]:
        _, p = _tiny_tlm(tmp_path, H, V, d, seed)
        assert plan_out(p)["shape"] is None, (H, V, d, seed)
        assert plan_out(p, 4, 2)["shape"] is None


def test_ctc_shape_fails_where_an_lm_state_has_two_successors_of_one_label(tmp_graphs):
    """make_synthetic_den draws each LM state's successors without regard to their labels, so (h,B) can have two arcs of one
    label into different states; the golden graphs are such graphs.  A two-slot prefix cannot follow both."""
    import os
    from conftest import GOLDEN
    for path in [tmp_graphs["tlm_small"][0], os.path.join(GOLDEN, "golden_tlm_a.fst"), os.path.join(GOLDEN, "golden_tlm_b.fst")]:
        msg = plan_out(path)["shape"]
        assert msg is not None and "two states of label" in msg and "file state" in msg, (path, msg)


def test_ctc_shape_fails_when_blank_twins_lead_to_different_states(tmp_path):
    """A hand-built graph: state 0 (blank twin) and state 1 (token twin of label 1) of one prefix both read token 2, but
    into different states, so the prefix '1 2' would need two states in one slot."""
    # arcs (src, dst, label): 0 -1-> 1, 1 -0-> 0 (blank back to the twin), 0 -2-> 2, 1 -2-> 3, self loops
    arcs = [(0, 0, 0), (0, 1, 1), (1, 1, 1), (1, 0, 0), (0, 2, 2), (1, 3, 2), (2, 2, 2), (3, 3, 2)]
    src, dst, lab = (np.array(c, np.int32) for c in zip(*arcs))
    final = np.full(4, np.inf, np.float32)
    final[[2, 3]] = 0.0
    g = fst.DenGraph(num_states=4, start=0, src=src, dst=dst, ilabel=lab + 1, olabel=lab.copy(),
                     weight=np.full(len(arcs), 0.7, np.float32), final=final)
    p = str(tmp_path / "twins.fst")
    fst.write_fst(p, g)
    msg = plan_out(p)["shape"]
    assert msg is not None and "step into different states" in msg, msg
    # the same graph with the token twin's arc led into state 2 passes
    dst2 = dst.copy()
    dst2[5] = 2
    g2 = fst.DenGraph(num_states=4, start=0, src=src, dst=dst2, ilabel=lab + 1, olabel=lab.copy(),
                      weight=np.full(len(arcs), 0.7, np.float32), final=final)
    p2 = str(tmp_path / "twins_ok.fst")
    fst.write_fst(p2, g2)
    assert plan_out(p2)["shape"] is None


# ---------------------------------------------------------------------------------------------------------------------
# arguments (checked before anything touches a device)
# ---------------------------------------------------------------------------------------------------------------------
class _FakeCuda(torch.Tensor):
    pass


def test_argument_checks(monkeypatch):
    def fake(shape, dtype=torch.float32):
        return torch.zeros(shape, dtype=dtype).as_subclass(_FakeCuda)
    monkeypatch.setattr(_FakeCuda, "is_cuda", property(lambda self: True))
    y = fake((2, 5, 4))
    lx = torch.tensor([5, 3], dtype=torch.int32)
    assert _C._check_beam_args(y, lx, 16, 4) == (2, 5, 4)
    assert _C._check_beam_args(y, lx, 128, 1) == (2, 5, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C._check_beam_args(torch.zeros(2, 5, 4), lx, 4, 4)
    with pytest.raises(RuntimeError, match="dtype"):
        _C._check_beam_args(fake((2, 5, 4), torch.float64), lx, 4, 4)
    with pytest.raises(RuntimeError, match="int32 CPU"):
        _C._check_beam_args(y, lx.long(), 4, 4)
    with pytest.raises(RuntimeError, match=r"\[0, T\]"):
        _C._check_beam_args(y, torch.tensor([6, 1], dtype=torch.int32), 4, 4)
    for bad in (0, 129, -1, 2.0, True, None):
        with pytest.raises(RuntimeError, match=r"beam_size must be an int in \[1, 128\]"):
            _C._check_beam_args(y, lx, bad, 4)
    for bad in (0, 5, 1.0, None):
        with pytest.raises(RuntimeError, match=r"cutoff_top_n must be an int in \[1, 4\]"):
            _C._check_beam_args(y, lx, 4, bad)


def test_native_entry_rejects_bad_arguments():
    L = _lib.lib()
    buf = (C.c_int * 4)()
    p = C.cast(buf, C.c_void_p)
    args = lambda beam, cut, V=4, dtype=0: (p, dtype, 1, 2, V, p, beam, cut, 0, p, p, p, p, p, None)
    for beam, cut, what in [(0, 2, "beam must lie in"), (129, 2, "beam must lie in"), (4, 0, "cutoff_top_n must lie in"),
                            (4, 5, "cutoff_top_n must lie in")]:
        assert L.ccb_ctc_beam_search(*args(beam, cut)) != 0
        assert what in _lib.last_error()
    assert L.ccb_ctc_beam_search(*args(4, 2, dtype=7)) != 0 and "dtype" in _lib.last_error()
    assert L.ccb_ctc_beam_search(*args(4, 2, V=9000)) != 0 and "8192" in _lib.last_error()
    assert L.ccb_ctc_beam_search_ws_bytes(2, 10, 0) == 0 and L.ccb_ctc_beam_search_ws_bytes(2, 10, 129) == 0
    assert L.ccb_ctc_beam_search_ws_bytes(2, 10, 4) >= 2 * (4 * (4 * 10 + 1) + 2 * (4 * 10 + 1)) * 4


def test_decoder_options():
    import ctc_crf
    d = ctc_crf.CTCBeamDecoder(["_", "a", "b"], beam_width=8, cutoff_top_n=40)
    assert d._cutoff_top_n == 3 and d._beam_width == 8
    for kw in (dict(model_path="lm.arpa"), dict(blank_id=1), dict(cutoff_prob=0.99)):
        with pytest.raises(NotImplementedError):
            ctc_crf.CTCBeamDecoder(["_", "a"], **kw)
    ctc_crf.CTCBeamDecoder(["_", "a"], alpha=0.5, beta=1.0, num_processes=8, log_probs_input=True)
