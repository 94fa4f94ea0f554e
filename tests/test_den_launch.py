"""The den kernels' launch decision (den_launch.h ChooseDenLaunch through ccb_plan_launch), checked without a GPU over
every batch width a call accepts."""
import ctypes as C

import pytest

from cat_b200 import _lib, fst

OPTIN = 232448   # H100: opt-in shared memory per block
TIER_SHARED, TIER_GLOBAL, TIER_STREAMED, TIER_SMALL = 0, 1, 2, 3
ARCS_IN_GLOBAL, W1_IN_GLOBAL, NO_TMA = 1, 2, 4
HOOK_SETS = [0, ARCS_IN_GLOBAL, W1_IN_GLOBAL, NO_TMA, ARCS_IN_GLOBAL | NO_TMA]   # what the GPU tests set
FIELDS = ("tier", "lanes", "U", "batch", "w1_smem", "Npad", "tile_rows", "gacc_rows", "arcs_off", "ring_off", "bar_off",
          "w1_off", "abar_off", "aring_off", "total")


class Plan:
    def __init__(self, path, n_ctas=132, n_warps=16):
        self.L = _lib.lib()
        self.h = self.L.ccb_plan_create(path.encode(), n_ctas, n_warps)
        assert self.h, _lib.last_error()

    def launch(self, N, backward, hooks=0, optin=OPTIN):
        out = (C.c_long * len(FIELDS))()
        rc = self.L.ccb_plan_launch(self.h, N, int(backward), optin, hooks, out)
        assert rc == 0, (N, backward, hooks, _lib.last_error())
        return dict(zip(FIELDS, out))

    def own_rows(self):
        """DenPlan::own_rows: the plan carries own-row coefficients (ccb_plan_copy 17 / 18) for some row."""
        info = (C.c_long * 13)()
        assert self.L.ccb_plan_info(self.h, info) == 0
        S = int(info[2])
        buf = (C.c_float * (2 * S))()
        own = False
        for which in (17, 18):
            assert self.L.ccb_plan_copy(self.h, which, buf, C.sizeof(buf)) == 0
            own = own or any(buf)
        return own

    def close(self):
        self.L.ccb_plan_destroy(self.h)


# Large-vocabulary T-compose-LM graphs: few states per label, so a CTA's tile spans many labels and the backward label
# accumulator ([labels][Npad] floats, at most 64 KB) stops fitting at some batch width
WIDE_LABEL_GRAPHS = {"G4k": (3000, 8, 4000), "G20k": (6000, 8, 20000)}
# Grids of sm_90a parts with fewer SMs than the H100 SXM's 132 (H100 PCIe 114, H20 78) and smaller ones still, where the
# tiles grow until the plan leaves the main tier.  tests/test_gpu_grids.py runs the kernels on these plans (CCB_DEN_CTAS).
OTHER_CTAS = (114, 78, 16, 4, 1)


@pytest.fixture(scope="module")
def graph_paths(tmp_graphs, fixture_fst, tmp_path_factory):
    paths = {"fixture": fixture_fst, **{k: v[0] for k, v in tmp_graphs.items()}}
    d = tmp_path_factory.mktemp("launch")
    big = str(d / "big.fst")
    fst.write_fst(big, fst.make_synthetic_den(4000, 24, 60, seed=7))
    paths["synthetic_4000"] = big
    for name, (H, deg, V) in WIDE_LABEL_GRAPHS.items():
        paths[name] = str(d / f"{name}.fst")
        fst.write_fst(paths[name], fst.make_synthetic_den(H, deg, V, seed=7))
    return paths


@pytest.fixture(scope="module")
def plans(graph_paths):
    out = {k: Plan(p) for k, p in graph_paths.items()}
    yield out
    for p in out.values():
        p.close()


@pytest.fixture(scope="module")
def grid_plans(graph_paths):
    """The same graphs' plans cut for OTHER_CTAS CTAs, by (name, n_ctas)."""
    out = {(k, n): Plan(p, n) for k, p in graph_paths.items() for n in OTHER_CTAS}
    yield out
    for p in out.values():
        p.close()


@pytest.fixture(scope="module")
def headline_plans(tmp_path_factory):
    """The benchmark's 1.02 M-arc den graph (H = 20 000 LM states, 24 successors, V = 218) at 132 and OTHER_CTAS CTAs."""
    path = str(tmp_path_factory.mktemp("headline") / "den_20000_218.fst")
    fst.write_fst(path, fst.make_synthetic_den(20000, 24, 218, seed=7))
    out = {n: Plan(path, n) for n in (132,) + OTHER_CTAS}
    yield out
    for p in out.values():
        p.close()


def test_every_batch_width_gets_a_launch_that_fits(plans, grid_plans):
    every = {**{(k, 132): p for k, p in plans.items()}, **grid_plans}
    for name, plan in every.items():
        for hooks in HOOK_SETS:
            small_ok = plan.launch(1, False, hooks)["tier"] == TIER_SMALL
            for N in range(1, 513):
                for backward in (False, True):
                    L = plan.launch(N, backward, hooks)
                    where = (name, hooks, N, backward, L)
                    assert 0 < L["total"] <= OPTIN - 1024, where
                    assert L["U"] in ((1, 2) if backward else (1, 2, 4)), where
                    small = small_ok and N <= 16
                    assert (L["tier"] == TIER_SMALL) == small, where
                    assert (L["lanes"], L["Npad"]) == (16, 16) if small else (L["lanes"] == 32 and L["Npad"] >= N), where
                    assert L["Npad"] <= 32 * L["U"] or L["Npad"] % (32 * L["U"]) == 0, where
                    if not backward:
                        assert L["tier"] != TIER_STREAMED and not L["w1_smem"], where
                    if L["tier"] in (TIER_SMALL, TIER_STREAMED):   # rings follow the arc tile, mbarriers follow the rings
                        assert L["arcs_off"] <= L["ring_off"] < L["bar_off"] < L["total"] and L["ring_off"] % 128 == 0, where


def test_tiers_the_fallback_tests_run(plans):
    """test_gpu_parity.py::test_fallback_paths runs the mid-size graph under these hooks for the tiers named here."""
    p = plans["tlm_mid"]
    for N in (12, 5):   # small-batch kernels
        for backward in (False, True):
            assert p.launch(N, backward)["tier"] == TIER_SMALL
        assert p.launch(N, True, W1_IN_GLOBAL)["tier"] == TIER_SMALL and not p.launch(N, True, W1_IN_GLOBAL)["w1_smem"]
    L = p.launch(20, True, W1_IN_GLOBAL)   # one utterance per lane, second weights from L2
    assert (L["tier"], L["U"], L["w1_smem"]) == (TIER_SHARED, 1, 0)
    for N, U in ((40, 2), (12, 1), (130, 2)):   # streamed-arc backward tier; the forward pass reads its arcs from L2
        L = p.launch(N, True, ARCS_IN_GLOBAL)
        assert (L["tier"], L["U"]) == (TIER_STREAMED, U)
        assert p.launch(N, False, ARCS_IN_GLOBAL)["tier"] == TIER_GLOBAL
    for N in (40, 12, 130):   # register gathers with the arcs from L2 in both passes
        for backward in (False, True):
            assert p.launch(N, backward, ARCS_IN_GLOBAL | NO_TMA)["tier"] == TIER_GLOBAL
    for backward in (False, True):   # the default: arcs resident, register gathers, 12-byte backward slots
        L = p.launch(64, backward)
        assert (L["tier"], L["U"], L["w1_smem"]) == (TIER_SHARED, 2, int(backward))
    assert p.launch(130, False)["U"] == 4 and p.launch(130, True)["U"] == 2


def test_label_accumulator_by_batch_width(plans):
    """Where the backward pass keeps its per-label occupancy sums in shared memory and where it adds them straight into the
    gradient with global atomics (gacc_rows = 0), at 132 CTAs.  The accumulator holds the CTA tile's label range for every
    lane, so its rows are fixed by the graph and it drops out once rows x Npad x 4 bytes pass 64 KB.
    tests/test_gpu_regimes.py runs both sides of the line on these graphs."""
    widths = {16: (1, 16), 32: (17, 32), 64: (33, 64), 128: (65, 128), 256: (129, 256), 384: (257, 384), 512: (385, 512)}
    want = {"tlm_mid": {w: 3 for w in widths},                                        # phone-shaped: 3 labels per tile
            "G4k": {**{w: 50 for w in (16, 32, 64, 128, 256)}, 384: 0, 512: 0},       # 50 x 384 x 4 B > 64 KB
            "G20k": {**{w: 213 for w in (16, 32, 64)}, 128: 0, 256: 0, 384: 0, 512: 0}}
    for name, rows in want.items():
        p = plans[name]
        for Npad, (n_lo, n_hi) in widths.items():
            for N in (n_lo, n_hi):
                L = p.launch(N, True)
                assert (L["Npad"], L["gacc_rows"]) == (Npad, rows[Npad]), (name, N, L)
                assert L["gacc_rows"] * Npad * 4 <= 64 * 1024
                assert p.launch(N, False)["gacc_rows"] == 0                           # the forward pass has none
        # the two wide graphs walk 4 and 2 utterances per lane at every width from 128 on, accumulator or not
        assert (p.launch(512, False)["U"], p.launch(512, True)["U"]) == (4, 2)


def _walk(p, N):
    """(forward tier, forward U, backward tier, backward U, second weights in shared memory, label accumulator rows)."""
    f, b = p.launch(N, False), p.launch(N, True)
    return f["tier"], f["U"], b["tier"], b["U"], b["w1_smem"], b["gacc_rows"]


def _u(N):
    """Utterances per lane of the full-width kernels: forward 1 / 2 / 4 from 17 / 33 / 65 utterances on, backward at most 2."""
    f = 1 if N <= 32 else 2 if N <= 64 else 4
    return f, min(f, 2)


def test_headline_graph_on_other_grids(headline_plans):
    """The benchmark's graph leaves the main tier as the grid shrinks (the batch widths tests/test_gpu_grids.py runs):
    132 / 114 CTAs: own-row terms, arcs resident in both passes, second weights in shared memory, 4 / 5 accumulator rows;
    78: the same tiers, but a backward tile past 72 KB drops the own-row terms (den_graph.cc BuildDenPlan);
    16: arcs from L2 forwards, streamed backwards (TMA row staging), no small-batch tier;
    4: arcs from L2 forwards; backwards streamed at one utterance per lane (N <= 32) and from L2 with register gathers at
       two (no test hook), 57 rows, none at N = 300 (57 x 384 x 4 B > 64 KB);
    1: the same with one tile of 219 labels, which fits up to N = 64."""
    SH, GL, ST, SM = TIER_SHARED, TIER_GLOBAL, TIER_STREAMED, TIER_SMALL
    want = {132: (True, SH, SH, 1, 4), 114: (True, SH, SH, 1, 5), 78: (False, SH, SH, 1, 5), 16: (False, GL, ST, 0, 16),
            4: (False, GL, GL, 0, 57), 1: (False, GL, GL, 0, 219)}
    for n, (own, ftier, btier, w1, rows) in want.items():
        p = headline_plans[n]
        assert p.own_rows() == own, n
        small = n >= 78
        for N in (5, 12, 40, 64, 130, 300):
            fu, bu = _u(N)
            gacc = 0 if (n == 4 and N > 256) or (n == 1 and N > 64) else rows
            if N <= 16 and small:
                assert _walk(p, N) == (SM, 1, SM, 1, 1, rows), (n, N)
            else:
                bt = ST if n == 4 and bu == 1 else btier     # 4 CTAs: one utterance per lane streams its backward arcs
                assert _walk(p, N) == (ftier, fu, bt, bu, w1, gacc), (n, N)


def test_small_graphs_on_other_grids(grid_plans, plans):
    """tlm_small, random_split and tlm_mid keep the 132-CTA tiers on every grid (small-batch kernels up to 16 utterances,
    arcs resident above); what moves is where the tiles are cut, and with it the label accumulator's rows.  On one CTA
    tlm_mid's backward tile passes 72 KB and its plan drops the own-row terms, which at 132 CTAs only CCB_NO_OWN does.
    tests/test_gpu_grids.py runs every one of these plans."""
    rows = {"tlm_small": {132: 2, 114: 2, 78: 3, 16: 3, 4: 6, 1: 13},
            "random_split": {132: 2, 114: 2, 78: 2, 16: 2, 4: 3, 1: 7},
            "tlm_mid": {132: 3, 114: 3, 78: 3, 16: 5, 4: 12, 1: 41}}
    for name, by_n in rows.items():
        for n, r in by_n.items():
            p = plans[name] if n == 132 else grid_plans[(name, n)]
            assert p.own_rows() == (name != "tlm_mid" or n != 1), (name, n)
            for N in (5, 12, 40, 64, 130, 300):
                fu, bu = _u(N)
                want = (TIER_SMALL, 1, TIER_SMALL, 1, 1, r) if N <= 16 else (TIER_SHARED, fu, TIER_SHARED, bu, 1, r)
                assert _walk(p, N) == want, (name, n, N)


def test_wide_label_accumulator_on_other_grids(grid_plans, plans):
    """G4k: a tile's labels grow as the grid shrinks, 50 / 57 / 74 / 285 rows at 132 / 114 / 78 / 16 CTAs, so the
    accumulator drops out at narrower batches: from N = 130 on at 78 CTAs (74 x 256 x 4 B > 64 KB; N = 64 keeps it), from
    N = 17 on at 16, at every N on 4.  On one CTA the graph runs the large-graph tiers without own-row terms and without the
    small-batch kernels."""
    want = {132: (True, 50, 256), 114: (True, 57, 256), 78: (True, 74, 64), 16: (True, 285, 16), 4: (True, 0, 0)}
    for n, (own, rows, widest) in want.items():
        p = plans["G4k"] if n == 132 else grid_plans[("G4k", n)]
        assert p.own_rows() == own, n
        for N in (8, 40, 64, 130, 300):
            fu, bu = _u(N)
            r = rows if N <= widest else 0
            want_walk = (TIER_SMALL, 1, TIER_SMALL, 1, 1, r) if N <= 16 else (TIER_SHARED, fu, TIER_SHARED, bu, 1, r)
            assert _walk(p, N) == want_walk, (n, N)
    p = grid_plans[("G4k", 1)]
    assert not p.own_rows()
    for N in (8, 40, 64, 130, 300):
        fu, bu = _u(N)
        assert _walk(p, N) == (TIER_GLOBAL, fu, TIER_STREAMED, bu, 0, 0), N
