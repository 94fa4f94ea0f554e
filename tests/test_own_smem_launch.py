"""Where the den kernels keep each warp's own rows of the last frame in shared memory (DenLaunch::own_smem, through
ccb_plan_launch_own), checked without a GPU: on for the register tiers of plans with own-row terms wherever the CTA tile's
[tile_rows][Npad] floats fit next to everything else, off otherwise, and off under CCB_OWN_IN_L2."""
import ctypes as C

import pytest

from cat_b200 import _lib, fst

OPTIN = 232448   # H100: opt-in shared memory per block
BUDGET = OPTIN - 1024
TIER_SHARED, TIER_GLOBAL, TIER_STREAMED, TIER_SMALL = 0, 1, 2, 3
ARCS_IN_GLOBAL, W1_IN_GLOBAL, NO_TMA, OWN_IN_L2 = 1, 2, 4, 8
FIELDS = ("tier", "lanes", "U", "batch", "w1_smem", "Npad", "tile_rows", "gacc_rows", "arcs_off", "ring_off", "bar_off",
          "w1_off", "abar_off", "aring_off", "total")
WIDTHS = (17, 32, 64, 128, 256, 512)
CTAS = (132, 114, 78, 16, 4, 1)


class Plan:
    def __init__(self, path, n_ctas):
        self.L = _lib.lib()
        self.h = self.L.ccb_plan_create(path.encode(), n_ctas, 16)
        assert self.h, _lib.last_error()

    def launch(self, N, backward, hooks=0):
        out, own = (C.c_long * len(FIELDS))(), (C.c_long * 2)()
        assert self.L.ccb_plan_launch(self.h, N, int(backward), OPTIN, hooks, out) == 0, _lib.last_error()
        assert self.L.ccb_plan_launch_own(self.h, N, int(backward), OPTIN, hooks, own) == 0, _lib.last_error()
        L = dict(zip(FIELDS, out))
        L["own_smem"], L["own_off"] = bool(own[0]), int(own[1])
        return L

    def own_rows(self):
        """DenPlan::own_rows: some row carries own-row coefficients (ccb_plan_copy 17 / 18)."""
        info = (C.c_long * 13)()
        assert self.L.ccb_plan_info(self.h, info) == 0
        buf = (C.c_float * (2 * int(info[2])))()
        own = False
        for which in (17, 18):
            assert self.L.ccb_plan_copy(self.h, which, buf, C.sizeof(buf)) == 0
            own = own or any(buf)
        return own

    def close(self):
        self.L.ccb_plan_destroy(self.h)


@pytest.fixture(scope="module")
def plans(tmp_graphs, fixture_fst, tmp_path_factory):
    """The suite's small graphs and the benchmark's 1.02 M-arc graph (H = 20 000, 24 successors, V = 218), cut for every
    grid in CTAS, by (name, n_ctas)."""
    paths = {"fixture": fixture_fst, **{k: v[0] for k, v in tmp_graphs.items()}}
    paths["headline"] = str(tmp_path_factory.mktemp("own_launch") / "den_20000_218.fst")
    fst.write_fst(paths["headline"], fst.make_synthetic_den(20000, 24, 218, seed=7))
    out = {(k, n): Plan(p, n) for k, p in paths.items() for n in CTAS}
    yield out
    for p in out.values():
        p.close()


# own_smem per batch width in WIDTHS ('1' on, '0' off), forward / backward: everything fits on the small graphs but for
# the widest batches on one CTA; the benchmark's graph fits up to N = 128 at 132 CTAs (156 KB of own rows at Npad = 128)
# and to 64 backwards at 114, and from 78 CTAs down its plans have no own-row terms (den_graph.cc BuildDenPlan)
PINNED = {
    "fixture": {n: ("111111", "111111") for n in CTAS},
    "tlm_small": {**{n: ("111111", "111111") for n in CTAS}, 1: ("111111", "111110")},
    "random_split": {**{n: ("111111", "111111") for n in CTAS}, 1: ("111110", "111110")},
    "tlm_mid": {**{n: ("111111", "111111") for n in CTAS}, 4: ("111100", "111100"), 1: ("000000", "000000")},
    "headline": {**{n: ("000000", "000000") for n in CTAS}, 132: ("111100", "111100"), 114: ("111100", "111000")},
}


def test_where_own_rows_are_on_chip(plans):
    for (name, n), p in plans.items():
        got = tuple("".join("1" if p.launch(N, backward)["own_smem"] else "0" for N in WIDTHS) for backward in (False, True))
        assert got == PINNED[name][n], (name, n, got)


def test_own_rows_fit_the_budget(plans):
    """Every layout with the own rows on chip fits the opt-in budget, and they sit behind the arc tile and close it; a launch
    keeps them off chip only when a plan without own-row terms, a TMA tier or the budget says so.  (The benchmark's plan for
    one CTA has no own-row terms, and its backward tile metadata alone passes the budget: no launch runs that pass.)"""
    for (name, n), p in plans.items():
        own_rows = p.own_rows()
        for N in WIDTHS:
            for backward in (False, True):
                L = p.launch(N, backward)
                where = (name, n, N, backward, L)
                if L["own_smem"]:
                    assert L["total"] <= BUDGET, where
                    assert own_rows and L["tier"] in (TIER_SHARED, TIER_GLOBAL), where
                    assert L["own_off"] >= L["arcs_off"] and L["own_off"] % 16 == 0, where
                    assert L["total"] == L["own_off"] + L["tile_rows"] * L["Npad"] * 4, where
                else:
                    fits = ((L["total"] + 15) // 16 * 16 + L["tile_rows"] * L["Npad"] * 4 <= BUDGET)
                    assert not own_rows or L["tier"] in (TIER_STREAMED, TIER_SMALL) or not fits, where
                # without the own rows the launch is the one it would be otherwise
                off = p.launch(N, backward, OWN_IN_L2)
                assert not off["own_smem"], where
                assert off["total"] <= L["own_off"] if L["own_smem"] else off["total"] == L["total"], where
                assert {k: off[k] for k in FIELDS if k != "total"} == {k: L[k] for k in FIELDS if k != "total"}, where


def test_small_batches_and_hooks(plans):
    """Batches of <= 16 utterances run the small-batch kernels, which keep nothing on chip; the test hooks that force the
    large-graph tiers leave the own rows on chip where a register tier remains (forward with arcs from L2) and off in the
    streamed-arc backward tier; CCB_OWN_IN_L2 turns them off everywhere."""
    p = plans[("tlm_mid", 132)]
    for N in (1, 5, 16):
        for backward in (False, True):
            L = p.launch(N, backward)
            assert L["tier"] == TIER_SMALL and not L["own_smem"], (N, L)
    for N in (40, 130):
        f, b = p.launch(N, False, ARCS_IN_GLOBAL), p.launch(N, True, ARCS_IN_GLOBAL)
        assert (f["tier"], f["own_smem"], b["tier"], b["own_smem"]) == (TIER_GLOBAL, True, TIER_STREAMED, False), N
        b = p.launch(N, True, ARCS_IN_GLOBAL | NO_TMA)
        assert (b["tier"], b["own_smem"]) == (TIER_GLOBAL, True), N
        b = p.launch(N, True, W1_IN_GLOBAL)
        assert (b["tier"], b["w1_smem"], b["own_smem"]) == (TIER_SHARED, 0, True), N
        for hooks in (OWN_IN_L2, ARCS_IN_GLOBAL | OWN_IN_L2, ARCS_IN_GLOBAL | NO_TMA | OWN_IN_L2, W1_IN_GLOBAL | OWN_IN_L2):
            for backward in (False, True):
                assert not p.launch(N, backward, hooks)["own_smem"], (N, hooks, backward)


@pytest.mark.parametrize("hook,own", [("CCB_NO_OWN", False), ("CCB_NO_MERGE", False), ("HUBS", False), ("CCB_NO_PAIRS", True)])
def test_plans_the_hooks_build(tmp_graphs, monkeypatch, hook, own):
    """Plans built without own-row terms (the hook itself, unmerged pairs, hub rows summed in parts) never keep rows on
    chip; without pairs every row is a group of one whose self loop is an own-row term, and those plans keep them."""
    if hook == "HUBS":
        monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
        monkeypatch.setenv("CCB_PART_ARCS", "7")
    else:
        monkeypatch.setenv(hook, "1")
    p = Plan(tmp_graphs["tlm_mid"][0], 132)
    try:
        assert p.own_rows() == own
        for N in WIDTHS:
            for backward in (False, True):
                assert p.launch(N, backward)["own_smem"] == own, (hook, N, backward)
                assert not p.launch(N, backward, OWN_IN_L2)["own_smem"]
    finally:
        p.close()
