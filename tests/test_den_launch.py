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

    def close(self):
        self.L.ccb_plan_destroy(self.h)


# Large-vocabulary T-compose-LM graphs: few states per label, so a CTA's tile spans many labels and the backward label
# accumulator ([labels][Npad] floats, at most 64 KB) stops fitting at some batch width
WIDE_LABEL_GRAPHS = {"G4k": (3000, 8, 4000), "G20k": (6000, 8, 20000)}


@pytest.fixture(scope="module")
def plans(tmp_graphs, fixture_fst, tmp_path_factory):
    paths = {"fixture": fixture_fst, **{k: v[0] for k, v in tmp_graphs.items()}}
    d = tmp_path_factory.mktemp("launch")
    big = str(d / "big.fst")
    fst.write_fst(big, fst.make_synthetic_den(4000, 24, 60, seed=7))
    paths["synthetic_4000"] = big
    for name, (H, deg, V) in WIDE_LABEL_GRAPHS.items():
        paths[name] = str(d / f"{name}.fst")
        fst.write_fst(paths[name], fst.make_synthetic_den(H, deg, V, seed=7))
    out = {k: Plan(p) for k, p in paths.items()}
    yield out
    for p in out.values():
        p.close()


def test_every_batch_width_gets_a_launch_that_fits(plans):
    for name, plan in plans.items():
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
