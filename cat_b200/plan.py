"""Host-side view of the den-graph kernel plan (``ccb_plan_*``): no GPU needed.

Used by the CPU tests (a numpy emulation of the kernels' arithmetic runs on these exact arrays) and by
tooling that wants to inspect how a den graph is cut for the persistent grid.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib

QUAD = 4            # arc segments are padded to whole quads (den_graph.h kQuad)
CHUNK_ARC_PAD = 16  # chunk arc counts are padded to a multiple of this (kChunkArcPad)
EV_ROW, EV_ROW_POS0, EV_ROW_POS1, EV_PARTIAL = 0, 1, 2, 3   # den_graph.h kEv*
EV_COMMON = EV_PARTIAL   # (old name)
EV_PAIR_MERGED = 3        # forward, plans without hub rows: ONE segment ends both rows of a pair (kEvPairMerged)
ARC_DTYPE = np.dtype([("peer", "<u4"), ("w", "<f4")])


@dataclass
class PassView:
    arcs: np.ndarray          # ARC_DTYPE [A]
    chunk_state: np.ndarray   # int32 [n_chunks+1]
    chunk_arc: np.ndarray     # int32 [n_chunks+1]
    chunk_pair: np.ndarray    # int32 [n_chunks+1]
    cta_labels: np.ndarray    # int32 [n_ctas, 4]
    w1: np.ndarray = None     # float32 [A] backward pass only: second weight per slot

    def weights(self) -> np.ndarray:
        return np.abs(self.arcs["w"])

    def segments(self):
        """Decode the stream the way the kernels walk it: yields (arc_begin, arc_end, event, label_changed) per
        segment.  Chunk-tail padding quads (unflagged, weight 0) attach to the following segment.
        Forward: event = kEv* code, label_changed = bool.  Backward (dual-weight groups): event = EV_ROW (one row) or
        EV_ROW_POS1 (a pair: two rows), label_changed = (flag of the first row, flag of the second row)."""
        w = self.arcs["w"].reshape(-1, QUAD)
        sign = np.signbit(w)
        ends = np.nonzero(sign[:, 3])[0]
        begin = 0
        for e in ends:
            if self.w1 is None:
                ev = (int(sign[e, 2]) << 1) | int(sign[e, 1])
                yield begin * QUAD, (e + 1) * QUAD, ev, bool(sign[e, 0])
            else:
                ev = EV_ROW_POS1 if sign[e, 2] else EV_ROW
                yield begin * QUAD, (e + 1) * QUAD, ev, (bool(sign[e, 0]), bool(sign[e, 1]))
            begin = e + 1


@dataclass
class PlanView:
    file_states: int
    file_arcs: int
    num_states: int
    num_pairs: int
    start: int
    num_labels: int
    n_ctas: int
    n_warps: int
    max_tile_arcs: int
    state_label: np.ndarray
    state_pos: np.ndarray
    final_lin: np.ndarray
    orig_state: np.ndarray
    start_arcs: np.ndarray
    hub_states: np.ndarray
    fwd: PassView
    bwd: PassView
    own_fwd: np.ndarray = None      # float32 [S, 2]: own-row coefficients of the forward pass (den_graph.h DenPlan::own_fwd)
    own_bwd: np.ndarray = None      # float32 [S, 2]

    @property
    def own_rows(self) -> bool:
        """DenPlan::own_rows: arcs from a group's own rows are coefficients (own_fwd / own_bwd), not gathered slots."""
        return bool(self.own_fwd.any() or self.own_bwd.any())

    @property
    def fwd_merged(self) -> bool:
        """DenPlan::fwd_merged: every pair is one forward segment (its second member's in-arcs, padding, then -- unless the plan
        carries own-row terms -- the first member's single arc in the last slot).  Event code 3 means kEvPairMerged in a plan
        without hub rows."""
        if len(self.hub_states):
            return False
        sign = np.signbit(self.fwd.arcs["w"].reshape(-1, QUAD))
        return bool((sign[:, 3] & sign[:, 2] & sign[:, 1]).any())


def load_plan(path: str, n_ctas: int = 132, n_warps: int = 16) -> PlanView:
    L = _lib.lib()
    h = L.ccb_plan_create(path.encode(), n_ctas, n_warps)
    if not h:
        raise RuntimeError(_lib.last_error())
    try:
        info = (C.c_long * 13)()
        assert L.ccb_plan_info(h, info) == 0
        S0, A0, S, Af, Ab, start, nl, nc, nw, mta, P, nsa, nh = [int(x) for x in info]
        n_chunks = nc * nw

        def get(which, dtype, count):
            a = np.empty(count, dtype=dtype)
            rc = L.ccb_plan_copy(h, which, a.ctypes.data_as(C.c_void_p), a.nbytes)
            assert rc == 0, f"ccb_plan_copy({which}) -> {rc}"
            return a

        return PlanView(S0, A0, S, P, start, nl, nc, nw, mta,
                        get(0, np.int32, S), get(9, np.int32, S), get(1, np.float32, S), get(2, np.int32, S),
                        get(12, ARC_DTYPE, nsa), get(16, np.int32, nh),
                        PassView(get(3, ARC_DTYPE, Af), get(4, np.int32, n_chunks + 1), get(5, np.int32, n_chunks + 1),
                                 get(10, np.int32, n_chunks + 1), get(13, np.int32, nc * 4).reshape(nc, 4)),
                        PassView(get(6, ARC_DTYPE, Ab), get(7, np.int32, n_chunks + 1), get(8, np.int32, n_chunks + 1),
                                 get(11, np.int32, n_chunks + 1), get(14, np.int32, nc * 4).reshape(nc, 4),
                                 get(15, np.float32, Ab)),
                        get(17, np.float32, 2 * S).reshape(S, 2), get(18, np.float32, 2 * S).reshape(S, 2))
    finally:
        L.ccb_plan_destroy(h)
