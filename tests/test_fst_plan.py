"""CPU: den-graph files and the host-side kernel plan (the product's C++ loader through the C ABI)."""
import numpy as np
import pytest

from cat_b200 import fst, plan, _lib
from oracle import oracle

import emulate


def test_fixture_parses(fixture_fst):
    g = fst.read_fst(fixture_fst)
    assert (g.num_states, g.num_arcs, g.start) == (9, 24, 0)
    assert sorted(np.nonzero(~np.isinf(g.final))[0].tolist()) == [4, 6]
    np.testing.assert_allclose(g.final[[4, 6]], 0.6931472, rtol=1e-6)
    P = plan.load_plan(fixture_fst, 4, 2)
    assert (P.file_states, P.file_arcs, P.num_states) == (9, 24, 9)      # T-compose-LM: no state split
    assert int((P.fwd.weights() > 0).sum()) == int(((P.bwd.weights() > 0) | (P.bwd.w1 > 0)).sum()) <= 24


def test_roundtrip_and_cxx_reader_agree(tmp_path):
    g = fst.make_synthetic_den(40, 5, 9, seed=1)
    p = str(tmp_path / "a.fst")
    fst.write_fst(p, g)
    g2 = fst.read_fst(p)
    for f in ("src", "dst", "ilabel", "weight", "final"):
        np.testing.assert_array_equal(getattr(g, f)[np.argsort(g.src, kind="stable")] if f not in ("final",) else g.final,
                                      getattr(g2, f))
    P = plan.load_plan(p, 7, 3)
    assert P.file_states == g.num_states and P.file_arcs == g.num_arcs
    # every file state appears, final weights carried over in the linear domain
    assert sorted(set(P.orig_state.tolist())) == list(range(g.num_states))
    np.testing.assert_allclose(P.final_lin, np.exp(g.end_weight()[P.orig_state]), rtol=1e-6)


@pytest.mark.parametrize("bad", ["missing", "garbage", "truncated", "wrongtype", "version1", "aligned"])
def test_bad_files_raise_not_exit(tmp_path, fixture_fst, bad):
    p = tmp_path / "x.fst"
    raw = open(fixture_fst, "rb").read()
    hdr = 4 + (4 + 6) + (4 + 8)     # magic, "vector", "standard": then int32 version, int32 flags
    if bad == "garbage":
        p.write_bytes(b"\x00" * 64)
    elif bad == "truncated":
        p.write_bytes(raw[:200])
    elif bad == "wrongtype":
        p.write_bytes(raw.replace(b"standard", b"log64xyz"))
    elif bad == "version1":
        p.write_bytes(raw[:hdr] + (1).to_bytes(4, "little") + raw[hdr + 4:])
    elif bad == "aligned":
        p.write_bytes(raw[:hdr + 4] + (4).to_bytes(4, "little") + raw[hdr + 8:])
    with pytest.raises(RuntimeError):
        plan.load_plan(str(p), 4, 2)
    assert _lib.last_error()
    if bad == "version1":
        assert "version" in _lib.last_error()
    if bad == "aligned":
        assert "aligned" in _lib.last_error()
    if bad not in ("missing", "version1", "aligned"):
        with pytest.raises(ValueError):
            fst.read_fst(str(p))


@pytest.fixture(scope="module")
def wide_label_graphs(tmp_path_factory):
    """Graphs with thousands of labels and few states per label: nearly every forward row end refreshes its emission, and a
    CTA tile spans tens to hundreds of labels.  Two T-compose-LM shaped (the G4k / G20k of tests/test_gpu_regimes.py) and
    an unstructured one with 2 500 labels, whose states the loader splits by in-label."""
    d = tmp_path_factory.mktemp("wide")
    out = {}
    for name, g, V in (("G4k", fst.make_synthetic_den(3000, 8, 4000, seed=7), 4000),
                       ("G20k", fst.make_synthetic_den(6000, 8, 20000, seed=7), 20000),
                       ("random_2500", fst.make_random_den(3000, 30000, 2500, seed=5), 2500)):
        fst.write_fst(str(d / f"{name}.fst"), g)
        out[name] = (str(d / f"{name}.fst"), g, V)
    return out


@pytest.mark.parametrize("n_ctas,n_warps", [(1, 1), (4, 2), (132, 16), (132, 32), (148, 16), (148, 32)])
def test_plan_invariants(tmp_graphs, n_ctas, n_warps):
    _check_plan_invariants(tmp_graphs, n_ctas, n_warps)


@pytest.mark.parametrize("n_ctas,n_warps", [(4, 2), (114, 16), (132, 16), (148, 16)])
def test_plan_invariants_wide_label_graphs(wide_label_graphs, n_ctas, n_warps):
    """The same invariants on graphs with thousands of labels (114 CTAs: an H100 PCIe)."""
    _check_plan_invariants(wide_label_graphs, n_ctas, n_warps)
    # most forward row ends carry the label-changed flag on these graphs: 2 990 of 3 000 on G4k at 132 x 16, 2 670 with
    # only 8 chunks (a chunk sorts its groups by label, so equal labels meet more often)
    for name in ("G4k", "G20k"):
        P = plan.load_plan(wide_label_graphs[name][0], n_ctas, n_warps)
        segs = list(P.fwd.segments())
        changed = sum(1 for _, _, _, chg in segs if chg)
        assert changed >= (0.98 if n_ctas >= 114 else 0.85) * len(segs), (name, changed, len(segs))


def _check_plan_invariants(graphs, n_ctas, n_warps):
    """graphs: name -> (path, graph, V); names starting with "random" are unstructured (split by in-label), the others
    T-compose-LM shaped."""
    for name, (path, g, V) in graphs.items():
        P = plan.load_plan(path, n_ctas, n_warps)
        S, NP = P.num_states, P.num_pairs
        assert P.num_labels <= V
        assert set(np.unique(P.state_pos)) <= {0, 1} and int((P.state_pos == 0).sum()) == NP
        # a pair is (pos0, pos1) on adjacent ids; inside a warp chunk groups are ordered by the label of their last
        # member, and CTA tiles are contiguous ranges of the global label order
        p0 = np.nonzero(P.state_pos == 0)[0]
        assert (P.state_pos[p0 + 1] == 1).all()
        np.testing.assert_array_equal(P.fwd.chunk_state, P.bwd.chunk_state)     # both passes share the cut
        cs_all = P.fwd.chunk_state
        for c in range(len(cs_all) - 1):
            st = np.arange(cs_all[c], cs_all[c + 1])
            last = P.state_label[st][P.state_pos[st] == 1]
            assert (np.diff(last) >= 0).all()
        tile_max = -1
        for c in range(n_ctas):
            st = np.arange(cs_all[c * n_warps], cs_all[(c + 1) * n_warps])
            last = P.state_label[st][P.state_pos[st] == 1]
            if len(last):
                assert last.min() >= tile_max
                tile_max = last.max()
        for pv, is_fwd in ((P.fwd, True), (P.bwd, False)):
            segs = list(pv.segments())
            merged = is_fwd and P.fwd_merged
            if merged:
                assert len(segs) == S - NP                               # one event per pair / unpaired state
                assert sum(1 for x in segs if x[2] == plan.EV_PAIR_MERGED) == NP
                assert not any(x[2] in (plan.EV_ROW_POS0, plan.EV_ROW_POS1) for x in segs)
                assert len(set(P.state_label[P.state_pos == 0].tolist())) == 1      # first members share one label
                assert (pv.arcs["peer"] < S + NP).all() and pv.w1 is None
            elif is_fwd:
                assert len(segs) == S                                    # one row-end event per state
                assert sum(1 for x in segs if x[2] == plan.EV_ROW_POS1) == NP == sum(1 for x in segs if x[2] == plan.EV_ROW_POS0)
                assert not any(x[2] == plan.EV_COMMON for x in segs)
                assert (pv.arcs["peer"] < S + NP).all() and pv.w1 is None
            else:
                assert len(segs) == S - NP                               # one group-end event per group
                assert sum(1 for x in segs if x[2] == plan.EV_ROW_POS1) == NP
                assert (pv.arcs["peer"] < S).all() and len(pv.w1) == len(pv.arcs) and (pv.w1 >= 0).all()
            assert len(pv.arcs) % plan.QUAD == 0
            assert pv.chunk_state[0] == 0 and pv.chunk_state[-1] == S
            assert (np.diff(pv.chunk_state) >= 0).all() and (np.diff(pv.chunk_pair) >= 0).all() and pv.chunk_pair[-1] == NP
            assert (pv.chunk_arc % plan.CHUNK_ARC_PAD == 0).all() and pv.chunk_arc[-1] == len(pv.arcs)
            # chunks never split a pair, and chunk_pair counts the pairs in front of each chunk
            cs = pv.chunk_state[:-1][np.diff(pv.chunk_state) > 0]
            assert (P.state_pos[cs - 1] == 1).all() if (cs > 0).any() else True
            np.testing.assert_array_equal(pv.chunk_pair, np.concatenate([[0], np.cumsum(P.state_pos == 0)])[pv.chunk_state])
            assert (pv.weights() >= 0).all()
            # sign bits appear only on a segment's last quad
            sg = np.signbit(pv.arcs["w"].reshape(-1, plan.QUAD))
            assert not sg[~sg[:, 3]].any()
            # label-changed flags == the label differs from the previous row of that position within the chunk
            q = 0
            prev = {}
            chunk_of = np.searchsorted(pv.chunk_arc, np.arange(0, len(pv.arcs), plan.QUAD), side="right") - 1
            for a0, a1, ev, chg in segs:
                c = int(chunk_of[(a1 - 1) // plan.QUAD])
                if merged and ev == plan.EV_PAIR_MERGED:
                    prev[(c, 0)] = int(P.state_label[q])           # the first member: no flag of its own
                    q += 1
                    rows = [(1, chg)]
                    # the last slot is the first member's arc (non-zero), everything between the second member's arcs and it is padding
                    assert P.own_rows or pv.arcs["w"][a1 - 1] != 0
                elif is_fwd:
                    rows = [(0 if ev == plan.EV_ROW_POS0 else 1, chg)]
                else:
                    rows = [(0, chg[0]), (1, chg[1])] if ev == plan.EV_ROW_POS1 else [(1, chg[0])]
                    if ev != plan.EV_ROW_POS1:
                        assert not chg[1]
                for k, flag in rows:
                    assert flag == (prev.get((c, k)) != int(P.state_label[q]))
                    prev[(c, k)] = int(P.state_label[q])
                    q += 1
            assert q == S
            # label accumulator ranges cover every state of the CTA
            for c in range(n_ctas):
                s0, s1 = pv.chunk_state[c * n_warps], pv.chunk_state[(c + 1) * n_warps]
                for pos, (lo, n) in ((0, pv.cta_labels[c, 0:2]), (1, pv.cta_labels[c, 2:4])):
                    labs = P.state_label[s0:s1][P.state_pos[s0:s1] == pos]
                    if len(labs):
                        assert lo <= labs.min() and labs.max() < lo + n
        nz_f = int((P.fwd.weights() > 0).sum())
        nz_b = int(((P.bwd.weights() > 0) | (P.bwd.w1 > 0)).sum())
        if name.startswith("random"):
            assert S > g.num_states
        else:
            assert S == g.num_states and NP > 0
            assert nz_f < g.num_arcs and nz_b < g.num_arcs                     # pairing removed the shared arcs
            own_f, own_b = int((P.own_fwd != 0).sum()), int((P.own_bwd != 0).sum())
            # T-compose-LM: blank arcs / self loops are own-row terms -- unless a CTA's backward stream is too large for the main
            # tier (den_graph.h kOwnRowsMaxTileBytes; here: the whole graph on 1 or 4 CTAs)
            small_tiles = int(np.diff(P.bwd.chunk_arc[::n_warps]).max()) * 12 <= 72 * 1024
            assert P.own_rows == small_tiles
            assert (own_f > 0 and own_b > 0) == P.own_rows
            assert nz_f == nz_b and own_f == own_b
        assert len(P.start_arcs) == int((np.asarray(g.src) == g.start).sum()) or name.startswith("random")


def test_pairing_halves_tlm_arcs_and_can_be_disabled(tmp_path, monkeypatch):
    g = fst.make_synthetic_den(400, 12, 40, seed=11)
    p = str(tmp_path / "g.fst")
    fst.write_fst(p, g)
    P = plan.load_plan(p, 8, 4)
    assert P.num_pairs == 399                                           # every (h,B),(h,L) twin
    assert int((P.fwd.weights() > 0).sum()) < 0.56 * g.num_arcs
    monkeypatch.setenv("CCB_NO_PAIRS", "1")
    Q = plan.load_plan(p, 8, 4)
    # (self loops are own-row terms: coefficients, not slots)
    assert Q.num_pairs == 0 and int((Q.fwd.weights() > 0).sum()) + int((Q.own_fwd != 0).sum()) == g.num_arcs


def test_merged_forward_pairs_and_switch(tmp_path, monkeypatch):
    """T-compose-LM graphs: every pair is ONE forward segment (kEvPairMerged: the label twin's in-arcs, padding, the blank
    twin's single arc in the last slot) -- fewer padded slots, half the row-end events; CCB_NO_MERGE=1 restores one segment
    per state.  Both layouts emulate to the oracle."""
    g = fst.make_synthetic_den(600, 24, 40, seed=5)
    p = str(tmp_path / "g.fst")
    fst.write_fst(p, g)
    monkeypatch.setenv("CCB_NO_OWN", "1")
    P = plan.load_plan(p, 4, 4)
    assert P.fwd_merged and not P.own_rows and P.num_pairs == 599
    n_ends = int(np.signbit(P.fwd.arcs["w"].reshape(-1, plan.QUAD)[:, 3]).sum())
    assert n_ends == P.num_states - P.num_pairs
    monkeypatch.setenv("CCB_NO_MERGE", "1")
    Q = plan.load_plan(p, 4, 4)
    assert not Q.fwd_merged and not Q.own_rows and Q.num_pairs == 599
    assert len(P.fwd.arcs) <= 0.92 * len(Q.fwd.arcs)                     # 28 instead of 28 + 4 slots per pair
    assert int((P.fwd.weights() > 0).sum()) == int((Q.fwd.weights() > 0).sum())
    # default: own-row terms on top -- the blank arcs and the token self loops are coefficients, not slots
    monkeypatch.delenv("CCB_NO_OWN"); monkeypatch.delenv("CCB_NO_MERGE")
    R = plan.load_plan(p, 4, 4)
    assert R.fwd_merged and R.own_rows
    # blank arc + token self loop per pair (+ the few LM arcs from a history to itself)
    assert int((P.fwd.weights() > 0).sum()) - 2 * 599 - 60 <= int((R.fwd.weights() > 0).sum()) <= int((P.fwd.weights() > 0).sum()) - 2 * 599
    nzb = lambda X: int(((X.bwd.weights() > 0) | (X.bwd.w1 > 0)).sum())
    assert nzb(P) - 2 * 599 - 60 <= nzb(R) <= nzb(P) - 2 * 599            # (h,B) and (h,L) rows leave the backward groups
    assert len(R.bwd.arcs) <= 0.9 * len(P.bwd.arcs)                      # 24 instead of 26 -> 28 slots per pair
    assert int(((P.bwd.weights() > 0) | (P.bwd.w1 > 0)).sum()) == int(((Q.bwd.weights() > 0) | (Q.bwd.w1 > 0)).sum())   # (the cut may differ)
    lens = [25, 14, 3]
    y, _, lens, _ = oracle.synth_batch(len(lens), max(lens), 40, seed=2, lens=lens)
    la, lb, gd = oracle.den(g, y, lens)
    for X in (P, Q, R):
        ea, eb, eg = emulate.den_emulate(X, y, lens)
        np.testing.assert_allclose(ea, la, rtol=1e-7)
        np.testing.assert_allclose(eb, lb, rtol=1e-7)
        assert np.abs(eg - gd).max() < 1e-6


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_plan_emulation_on_random_graph_families(tmp_path, monkeypatch, seed):
    """The plan builder's rewrites (in-label split, pair factoring, merged pair segments, own-row terms, hub parts) are exact:
    for several graph families and every switch setting, the kernels' arithmetic emulated on the plan arrays equals the
    arc-based oracle.  Families: synthetic T-compose-LM (with LM arcs from a history to itself), a natively composed
    CTC-topology x phone-LM graph, an unstructured random graph with self loops."""
    rng = np.random.default_rng(seed)
    V = int(rng.integers(5, 14))
    graphs = {
        "tlm": fst.make_synthetic_den(int(rng.integers(6, 40)), int(rng.integers(2, 6)), V, seed=seed),
        "composed": fst.compose_ctc_lm(fst.make_random_lm(int(rng.integers(3, 12)), V - 1, int(rng.integers(1, 4)), seed=seed)),
        "random": fst.make_random_den(int(rng.integers(8, 30)), int(rng.integers(40, 200)), V, seed=seed),
    }
    lens = [int(x) for x in rng.integers(1, 14, size=3)]
    for name, g in graphs.items():
        p = str(tmp_path / f"{name}.fst")
        fst.write_fst(p, g)
        y, _, ln, _ = oracle.synth_batch(len(lens), max(lens), V, seed=seed + 10, lens=lens)
        la, lb, gd = oracle.den(g, y, ln)
        for env in ({}, {"CCB_NO_OWN": "1"}, {"CCB_NO_MERGE": "1"}, {"CCB_NO_PAIRS": "1"}, {"CCB_HUB_IN_ARCS": "5", "CCB_PART_ARCS": "7"}):
            with monkeypatch.context() as m:
                for k, v in env.items():
                    m.setenv(k, v)
                P = plan.load_plan(p, int(rng.integers(1, 6)), int(rng.integers(1, 5)))
            ea, eb, eg = emulate.den_emulate(P, y, ln)
            fin = np.isfinite(la)
            np.testing.assert_allclose(ea[fin], la[fin], rtol=1e-7, err_msg=f"{name} {env}")
            np.testing.assert_allclose(eb[fin], lb[fin], rtol=1e-7, err_msg=f"{name} {env}")
            assert (np.isinf(ea[~fin]) & (ea[~fin] < 0)).all(), (name, env)       # no path to a final state: -inf on both sides
            if fin.any():
                assert np.abs(eg[fin] - gd[fin]).max() < 1e-6, (name, env)


def test_plan_balance(tmp_path):
    g = fst.make_synthetic_den(4000, 24, 60, seed=7)
    p = str(tmp_path / "g.fst")
    fst.write_fst(p, g)
    P = plan.load_plan(p, 132, 16)
    for pv in (P.fwd, P.bwd):
        per_cta = np.diff(pv.chunk_arc[::16])
        assert per_cta.max() <= 1.3 * per_cta.mean() + 64
        per_warp = np.diff(pv.chunk_arc).reshape(132, 16)
        assert (per_warp.max(1) - per_warp.min(1)).max() <= 48          # LPT: warps of a CTA within a few quads
    assert P.max_tile_arcs * 8 < 200 * 1024


@pytest.mark.parametrize("name,lens", [("tlm_small", [30, 22, 9, 1]), ("random_split", [20, 13, 7, 2])])
def test_kernel_arithmetic_emulation_matches_oracle(tmp_graphs, name, lens):
    """The scaled-linear / hoisted-emission / state-product algorithm the kernels implement, emulated in numpy on
    the product's own plan arrays, equals the arc-based log-domain reference semantics."""
    path, g, V = tmp_graphs[name]
    P = plan.load_plan(path, 132, 16)
    y, _, lens, _ = oracle.synth_batch(len(lens), max(lens), V, seed=6, lens=lens)
    la, lb, gd = oracle.den(g, y, lens)
    ea, eb, eg = emulate.den_emulate(P, y, lens)
    np.testing.assert_allclose(ea, la, rtol=1e-7)
    np.testing.assert_allclose(eb, lb, rtol=1e-7)
    assert np.abs(eg - gd).max() < 1e-6


def test_hub_rows_split_into_parts(tmp_graphs, monkeypatch):
    """States with a long in-arc row get their forward row computed in parts (any warp, atomically accumulated);
    thresholds lowered through the test hooks so that small graphs exercise several parts per row."""
    monkeypatch.setenv("CCB_HUB_IN_ARCS", "6")
    monkeypatch.setenv("CCB_PART_ARCS", "7")
    for name in ("tlm_small", "random_split"):
        path, g, V = tmp_graphs[name]
        P = plan.load_plan(path, 132, 16)
        assert len(P.hub_states) > 0
        parts = [x for x in P.fwd.segments() if x[2] == plan.EV_PARTIAL]
        assert len(parts) > len(P.hub_states)                      # some rows have several parts
        lens = [20, 13, 7, 2]
        y, _, lens, _ = oracle.synth_batch(len(lens), max(lens), V, seed=6, lens=lens)
        la, lb, gd = oracle.den(g, y, lens)
        ea, eb, eg = emulate.den_emulate(P, y, lens)
        np.testing.assert_allclose(ea, la, rtol=1e-7)
        np.testing.assert_allclose(eb, lb, rtol=1e-7)
        assert np.abs(eg - gd).max() < 1e-6


def test_fixture_emulation(fixture_fst, fixture_inputs):
    P = plan.load_plan(fixture_fst, 132, 16)
    ea, eb, eg = emulate.den_emulate(P, fixture_inputs["y"], fixture_inputs["lx"])
    assert abs(ea[0] + 6.25832785) < 1e-6 and abs(eb[0] + 6.25832785) < 1e-6


def test_compose_ctc_lm_is_the_lm_weighted_sum_of_ctc(tmp_path):
    """SURVEY 8f-2: den graph built natively as T o LM.  Property (what the denominator *means*,
    docs/toolkitworkflow.md:124-135): logZ_den(x) = log sum_l p_LM(l) p_CTC(l|x) over every label sequence l --
    enumerated exhaustively here with the oracle's CTC, and the composed file round-trips through both FST readers."""
    import itertools
    from oracle import oracle
    V, T = 4, 4
    lm = fst.make_random_lm(H=3, V=V, d=2, seed=5)
    g = fst.compose_ctc_lm(lm)
    rng = np.random.default_rng(2)
    x = rng.standard_normal((1, T, V))
    y = (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)
    la, lb, gamma = oracle.den(g, y, [T])
    total = -np.inf
    n_acc = 0
    for L in range(0, T + 1):
        for l in itertools.product(range(1, V), repeat=L):
            lp_lm = fst.lm_logprob(lm, l)
            if not np.isfinite(lp_lm):
                continue
            lp, _ = oracle.ctc(y, np.asarray(l, np.int32), [L], [T], want_grad=False)
            if np.isfinite(lp[0]):
                total = np.logaddexp(total, lp_lm + lp[0]); n_acc += 1
    assert n_acc > 3
    assert abs(la[0] - total) < 1e-5 and abs(lb[0] - total) < 1e-5
    # the file the product loads: same plan semantics as any other den graph
    p = str(tmp_path / "tlm.fst")
    fst.write_fst(p, g)
    g2 = fst.read_fst(p)
    assert g2.num_states == g.num_states and g2.num_arcs == g.num_arcs
    pv = plan.load_plan(p, 4, 2)
    ea, eb, eg = emulate.den_emulate(pv, y, [T])
    assert abs(ea[0] - total) < 1e-4 and abs(eb[0] - total) < 1e-4
