"""Word decoding through a TLG decoding graph on the GPU (``ctc_crf.fst_decode``): the 1-best step of CAT's
``cat/ctc/fst_decode.sh`` (Kaldi ``latgen-faster`` + ``lattice-best-path``) without the lattice.

``DecodingGraph`` wraps the native loader (``cat_b200/csrc/wfst.cc``); ``fst_decode`` runs the frame-synchronous Viterbi
beam search (``cat_b200/csrc/wfst_decode.cu``, DESIGN.md §7 "TLG decoding").
"""
from __future__ import annotations

import ctypes as C
import math
from collections import namedtuple
from typing import List, Optional

import numpy as np
import torch

from . import _lib
from ._C import _DTYPES, _PinnedRing, _budget_cache, _check, _check_sample_args, _rings, _scratch_budget, _stream

MAX_ACTIVE = 1 << 20

# ccb_wfst_copy codes (include/ctc_crf_b200.h) and their dtypes
_TABLES = {"arc_off": (0, np.int32), "eps_off": (1, np.int32), "dst": (2, np.int32), "token": (3, np.int32),
           "olabel": (4, np.int32), "weight": (5, np.float32), "fid": (6, np.int32), "final": (7, np.float32),
           "level": (8, np.int32)}

WfstResult = namedtuple("WfstResult", ["words", "num_words", "align", "ac_logp", "graph_cost", "cost", "reached_final"])


class DecodingGraph:
    """A TLG decoding graph, read from an OpenFst ``vector``/``standard`` binary file in CAT's conventions: ilabel = token
    + 1 (blank = token 0), ilabel 0 = epsilon, olabel = word id (0 = no word), tropical weights (what
    ``cat/utils/tool/build_decoding_graph.sh`` writes as ``TLG.fst``).  words: CAT's ``words.txt`` or ``r_words.txt``
    (lines "word id"), used by ``to_text``.

    A file whose epsilon arcs form a cycle, a const FST, one with embedded symbol tables or with aligned fields raises
    RuntimeError saying what is wrong.  The tables live on the host until a search uses the graph on a device; dropping the
    object frees both (on the device with ``cudaFree``, which waits for the device).  Attributes: num_states, num_arcs,
    start, L (the longest epsilon path), E (the most states one state reaches through epsilon arcs), max_out (the largest
    emitting out-degree), max_ilabel, eps_arcs."""

    def __init__(self, path: str, words: Optional[str] = None):
        L = _lib.lib()
        h = L.ccb_wfst_create(str(path).encode())
        if not h:
            raise RuntimeError(f"DecodingGraph: {_lib.last_error()}")
        self._h = h
        self.path = str(path)
        info = (C.c_long * 8)()
        L.ccb_wfst_info(h, info)
        (self.num_states, self.num_arcs, self.start, self.L, self.E, self.max_out, self.max_ilabel,
         self.eps_arcs) = (int(x) for x in info)
        self.words = None
        if words is not None:
            self.words = {}
            with open(words, encoding="utf-8") as f:
                for line in f:
                    p = line.split()
                    if len(p) == 2 and p[1].lstrip("-").isdigit():
                        self.words[int(p[1])] = p[0]

    @property
    def handle(self) -> int:
        return self._h

    def tables(self) -> dict:
        """The host tables as numpy arrays: each state's arcs are arc_off[s] .. arc_off[s+1]-1, emitting ones (in file
        order) up to eps_off[s], then epsilon ones; per arc dst, token (-1: epsilon), olabel, weight, fid (its position in
        the file); per state final (+inf: not final) and level (the longest epsilon path into it)."""
        L = _lib.lib()
        S, A = self.num_states, self.num_arcs
        sizes = {"arc_off": S + 1, "eps_off": S, "dst": A, "token": A, "olabel": A, "weight": A, "fid": A, "final": S,
                 "level": S}
        out = {}
        for name, (which, dt) in _TABLES.items():
            a = np.empty(sizes[name], dt)
            if L.ccb_wfst_copy(self._h, which, a.ctypes.data_as(C.c_void_p), a.nbytes) != 0:
                raise RuntimeError(f"ccb_wfst_copy({name}) failed")
            out[name] = a
        return out

    def to_text(self, words: torch.Tensor, num_words: torch.Tensor) -> List[Optional[List[str]]]:
        """The word strings of ``fst_decode``'s words and num_words, one list per utterance (None for an utterance without a
        path).  One device-to-host copy.  Ids the word table does not list are written as their number."""
        N, W = words.shape
        host = torch.cat([num_words.reshape(N, 1).to(torch.int32), words.to(torch.int32)], 1).cpu().numpy()
        table = self.words or {}
        return [None if r[0] < 0 else [table.get(int(w), str(int(w))) for w in r[1:1 + r[0]]] for r in host]

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                _lib.lib().ccb_wfst_destroy(h)
            except Exception:      # interpreter shutdown: module globals may already be gone
                pass


def check_decode_args(graph, V, acwt, lmwt, wip, beam, max_active) -> None:
    """The search arguments of ``fst_decode`` (ValueError), checked before anything touches a device."""
    if not isinstance(graph, DecodingGraph):
        raise ValueError(f"fst_decode: graph must be a DecodingGraph, not {type(graph).__name__}")
    if isinstance(max_active, bool) or not isinstance(max_active, int) or not 1 <= max_active <= MAX_ACTIVE:
        raise ValueError(f"fst_decode: max_active must be an int in [1, {MAX_ACTIVE}], not {max_active!r}")
    for name, v in (("acwt", acwt), ("lmwt", lmwt), ("wip", wip), ("beam", beam)):
        if isinstance(v, bool) or not isinstance(v, (int, float)) or math.isnan(v):
            raise ValueError(f"fst_decode: {name} must be a number, not {v!r}")
    if not beam > 0:
        raise ValueError(f"fst_decode: beam must be > 0 (inf is allowed), not {beam!r}")
    if not (math.isfinite(acwt) and acwt >= 0):
        raise ValueError(f"fst_decode: acwt must be finite and >= 0, not {acwt!r}")
    if not (math.isfinite(lmwt) and lmwt > 0):
        raise ValueError(f"fst_decode: lmwt must be finite and > 0, not {lmwt!r}")
    if not math.isfinite(wip):
        raise ValueError(f"fst_decode: wip must be finite, not {wip!r}")
    if graph.max_ilabel > V:
        raise ValueError(f"fst_decode: the graph has ilabels up to {graph.max_ilabel} (tokens up to {graph.max_ilabel - 1}), "
                         f"the logits have V = {V}")


def fst_decode(logits: torch.Tensor, lx: torch.Tensor, graph: DecodingGraph, acwt: float = 1.0, lmwt: float = 1.0,
               wip: float = 0.0, beam: float = 17.0, max_active: int = 7000) -> WfstResult:
    """The 1-best word sequence per utterance through ``graph`` by a frame-synchronous Viterbi beam search on the GPU
    (DESIGN.md §7 "TLG decoding"): the search ``latgen-faster --beam=beam --max-active=max_active
    --acoustic-scale=acwt/lmwt`` + ``lattice-best-path --lm-scale=lmwt --word-ins-penalty=wip`` performs, without the
    lattice.  With acs = acwt / lmwt and wps = wip / lmwt, an emitting arc adds its weight, -acs * y[t][token] and wps per
    word; an epsilon arc its weight and wps per word.  Each frame keeps the tokens within best + beam, recombines per state,
    closes over epsilon arcs and keeps the max_active cheapest.

    logits (N,T,V) fp32, bf16 or fp16 on the GPU: log-probs or raw logits (a per-frame shift does not change the search in
    exact arithmetic); frames t >= lx[n] are never read.  lx (N,) int32 on the CPU.  max_active in [1, 2^20], beam > 0
    (inf allowed), acwt finite >= 0, lmwt finite > 0, wip finite (ValueError otherwise).

    Returns a ``WfstResult`` of device tensors, without synchronising the host: words (N, (T+1)(1+L)) int32 padded with -1,
    num_words (N,) int32, align (N,T) int32 (the token of each frame's emitting arc, -1 past lx), ac_logp (N,) =
    sum_t y[t][align[t]], graph_cost (N,) = the path's graph weights plus its final cost, cost (N,) = lmwt graph_cost -
    acwt ac_logp + wip num_words, reached_final (N,) int32 (0: no final state among the kept tokens; the best token's path
    is returned, as ``--allow-partial=true``).  An utterance without a path of finite cost gets num_words -1, rows of -1
    and cost +inf.  ``graph.to_text(words, num_words)`` gives the word strings.  One launch per slice of the batch; the
    batch is sliced when its workspace does not fit the free device memory."""
    N, T, V = _check_sample_args(logits, lx, 1)
    check_decode_args(graph, V, acwt, lmwt, wip, beam, max_active)
    L = _lib.lib()
    dev = logits.device
    K = int(max_active)
    Wcap = (T + 1) * (1 + graph.L)
    with torch.no_grad(), torch.cuda.device(dev):
        y = logits.detach().contiguous()
        esz = y.element_size()
        lens = _rings.setdefault(torch.device(dev).index, _PinnedRing()).stage([lx], dev)
        words = torch.empty((N, Wcap), dtype=torch.int32, device=dev)
        num_words = torch.empty((N,), dtype=torch.int32, device=dev)
        align = torch.empty((N, T), dtype=torch.int32, device=dev)
        ac_logp = torch.empty((N,), dtype=torch.float32, device=dev)
        graph_cost = torch.empty((N,), dtype=torch.float32, device=dev)
        cost = torch.empty((N,), dtype=torch.float32, device=dev)
        reached = torch.empty((N,), dtype=torch.int32, device=dev)
        per = int(L.ccb_wfst_decode_ws_bytes(graph.handle, 1, T, K))
        stream = _stream(dev)

        def run_slices():
            step = max(1, min(N, _scratch_budget(dev, per) // max(per, 1)))
            for n0 in range(0, N, step):
                n = min(step, N - n0)
                ws = torch.empty(int(L.ccb_wfst_decode_ws_bytes(graph.handle, n, T, K)), dtype=torch.uint8, device=dev)
                rc = L.ccb_wfst_decode(y.data_ptr() + n0 * T * V * esz, _DTYPES[y.dtype], n, T, V, lens.data_ptr() + 4 * n0,
                                       graph.handle, float(acwt), float(lmwt), float(wip), float(beam), K, ws.data_ptr(),
                                       words.data_ptr() + n0 * Wcap * 4, num_words.data_ptr() + n0 * 4,
                                       align.data_ptr() + n0 * T * 4, ac_logp.data_ptr() + n0 * 4,
                                       graph_cost.data_ptr() + n0 * 4, cost.data_ptr() + n0 * 4,
                                       reached.data_ptr() + n0 * 4, stream)
                _check(rc, "fst_decode")
                del ws

        try:
            run_slices()
        except torch.cuda.OutOfMemoryError:       # as in ctc_crf_loss_fwd
            _budget_cache.pop(torch.device(dev).index, None)
            torch.cuda.empty_cache()
            run_slices()
        lens.record_stream(torch.cuda.current_stream(dev))
    return WfstResult(words, num_words, align, ac_logp, graph_cost, cost, reached)
