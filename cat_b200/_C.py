"""``ctc_crf._C`` -- host-side mirror of the reference's pybind module (src/ctc_crf/binding.cpp:51-126).

Same four entry points, same argument meaning and placement (``gpu_ctc`` takes CPU labels/lengths/costs and
(T,N,V) activations; ``gpu_den`` takes CUDA lengths and pre-zeroed gradients), implemented by calling the C ABI
of ``libctc_crf_b200.so`` through ctypes.  As in binding.cpp, scratch is taken from torch's caching allocator
and the work is enqueued on the current CUDA stream of the tensors' device.  Differences: a device guard is
installed (binding.cpp has none, SURVEY.md 8b) and native errors raise ``RuntimeError`` instead of being
ignored (binding.cpp:105,111) or exiting the process (den_calculate.cu:16-25).

Addition: ``ctc_crf_loss_fwd`` -- the fused, synchronisation-free entry used by ``CTC_CRF_LOSS``; ``ctc_crf_loss_fwd_only``
and ``ctc_loss_fwd_only`` -- the losses without a gradient, used when grad mode is off.  Every loss function takes
``reduction`` (None: the scalar of ``size_average``; 'none': one cost per utterance) and ``zero_infinity``;
``grad_rows_scale`` is the backward of the per-utterance costs.  ``ctc_crf_loss_seqs``, ``ctc_crf_loss_seqs_fwd_only``,
``ctc_loss_seqs`` and ``ctc_align_seqs`` take several label sequences per utterance (``utt``: the logits row of each), with the
den passes run once per utterance; ``seqs_backward`` is the backward of their per-sequence costs.  ``crf_sample`` draws paths
from the CTC-CRF posterior and ``samples_to_labels`` packs them for the ``utt=`` loss.  ``ctc_beam_search`` returns N-best
lists by CTC prefix beam search, over the logits or over the den graph, optionally with a token n-gram LM fused in.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import ctcOptions

# logits dtype -> CCB_DTYPE_* code (include/ctc_crf_b200.h).  The fused entries read the logits in place in this type and
# compute in fp32; gpu_den / gpu_ctc keep the reference's fp32 contract.
_DTYPES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def check_reduction(reduction) -> bool:
    """reduction None keeps the scalar loss of ``size_average`` (the sum, or the mean over the batch); 'none' returns the
    (N,) costs.  There is no second spelling of the sum or the mean.  Returns whether the costs are returned ('none')."""
    if reduction is not None and reduction != "none":
        raise ValueError(f"reduction must be None or 'none', not {reduction!r}: for the batch sum or mean leave it None and "
                         f"choose with size_average (False: sum, True: mean over the batch)")
    return reduction == "none"


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed: {_lib.last_error() or rc}")


def _raise_if_error(what: str) -> None:
    msg = _lib.last_error()
    if msg:
        raise RuntimeError(f"{what} failed: {msg}")


def _stream(device: torch.device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _iptr(t: torch.Tensor):
    return C.cast(t.data_ptr(), C.POINTER(C.c_int))


def _ptr(t: Optional[torch.Tensor]):
    """The device address of an optional buffer: NULL for None."""
    return None if t is None else t.data_ptr()


def init_env(fst_name: str, gpus: torch.Tensor) -> None:
    """binding.cpp:51-56"""
    assert gpus.dtype == torch.int32 and not gpus.is_cuda
    g = gpus.contiguous()
    _lib.lib().Init(fst_name.encode(), int(g.numel()), _iptr(g))
    _raise_if_error("init_env")


def release_env(gpus: torch.Tensor) -> None:
    """binding.cpp:58-63"""
    g = gpus.contiguous()
    _lib.lib().Release(int(g.numel()), _iptr(g))


def den_num_states() -> int:
    return C.c_int.in_dll(_lib.lib(), "DEN_NUM_STATES").value


def den_info() -> dict:
    """Sizes of the loaded den graph and of its kernel plan."""
    info = (C.c_long * 8)()
    if _lib.lib().ccb_den_info(info) != 0:
        raise RuntimeError("den graph not loaded")
    keys = ("file_states", "file_arcs", "states", "pairs", "fwd_slots", "bwd_slots", "fwd_arcs", "bwd_arcs")
    return dict(zip(keys, [int(x) for x in info]))


def den_num_arcs() -> int:
    return C.c_int.in_dll(_lib.lib(), "DEN_NUM_ARCS").value


def gpu_den(logits: torch.Tensor, grad_net: torch.Tensor, input_lengths: torch.Tensor,
            costs_alpha: torch.Tensor, costs_beta: torch.Tensor) -> None:
    """binding.cpp:65-84.  logits (N,T,V) fp32 CUDA contiguous; grad_net pre-zeroed, filled in place;
    input_lengths (N,) int32 CUDA; costs_* (N,) fp32 CUDA."""
    L = _lib.lib()
    assert logits.is_cuda and logits.dtype == torch.float32 and logits.is_contiguous()
    assert grad_net.is_cuda and grad_net.dtype == torch.float32 and grad_net.is_contiguous()
    assert input_lengths.is_cuda and input_lengths.dtype == torch.int32
    N, T, V = logits.shape
    dev = logits.device
    with torch.cuda.device(dev):
        stream = _stream(dev)
        S = den_num_states()
        # binding.cpp:77-79 sizes; alpha is padded to whole 32-lane groups here
        # the library states its need through ccb_den_alpha_floats (lane padding, parked pair rows); alpha_size is the
        # per-(frame, utterance) row count binding.cpp would pass, rounded UP so that (T+1)*N*alpha_size covers the need
        per = (T + 1) * N
        alpha_states = max(S, -(-int(L.ccb_den_alpha_floats(N, T)) // per))
        alpha = torch.empty(per * alpha_states, dtype=torch.float32, device=dev)
        beta = torch.empty(1, dtype=torch.float32, device=dev)
        grad_storage = torch.empty(1, dtype=torch.float32, device=dev)
        L.compute_alpha(alpha.data_ptr(), logits.data_ptr(), N, T, alpha_states, V, input_lengths.data_ptr(),
                        costs_alpha.data_ptr(), stream)
        _raise_if_error("gpu_den/compute_alpha")
        L.compute_beta_and_grad(beta.data_ptr(), alpha.data_ptr(), logits.data_ptr(), costs_alpha.data_ptr(),
                                grad_storage.data_ptr(), grad_net.data_ptr(), N, T, alpha_states, V,
                                input_lengths.data_ptr(), costs_beta.data_ptr(), stream)
        _raise_if_error("gpu_den/compute_beta_and_grad")


def gpu_ctc(probs: torch.Tensor, grads: torch.Tensor, labels: torch.Tensor, label_sizes: torch.Tensor,
            sizes: torch.Tensor, minibatch_size: int, costs: torch.Tensor, blank_label: int) -> None:
    """binding.cpp:86-117.  probs/grads (T,N,V) fp32 CUDA (grads pre-zeroed); labels/label_sizes/sizes int32 CPU;
    costs (N,) fp32 CPU, receives log p(l|x) per utterance."""
    L = _lib.lib()
    assert probs.is_cuda and probs.dtype == torch.float32 and probs.is_contiguous()
    assert not labels.is_cuda and not label_sizes.is_cuda and not sizes.is_cuda and not costs.is_cuda
    assert labels.dtype == torch.int32 and label_sizes.dtype == torch.int32 and sizes.dtype == torch.int32
    assert costs.dtype == torch.float32 and costs.is_contiguous()
    labels, label_sizes, sizes = labels.contiguous(), label_sizes.contiguous(), sizes.contiguous()
    V = probs.size(2)
    dev = probs.device
    with torch.cuda.device(dev):
        opts = ctcOptions(stream=torch.cuda.current_stream(dev).cuda_stream, blank_label=int(blank_label))
        nbytes = C.c_size_t(0)
        st = L.get_workspace_size(_iptr(label_sizes), _iptr(sizes), V, minibatch_size, opts, C.byref(nbytes))
        if st != 0:
            raise RuntimeError(f"gpu_ctc/get_workspace_size: {L.ctcGetStatusString(st).decode()}")
        ws = torch.empty((nbytes.value + 3) // 4, dtype=torch.float32, device=dev)
        gptr = grads.data_ptr() if grads is not None and grads.numel() > 0 else None
        st = L.compute_ctc_loss(probs.data_ptr(), gptr, _iptr(labels), _iptr(label_sizes), _iptr(sizes), V,
                                minibatch_size, C.cast(costs.data_ptr(), C.POINTER(C.c_float)), ws.data_ptr(), opts)
        if st != 0:
            raise RuntimeError(f"gpu_ctc/compute_ctc_loss: {L.ctcGetStatusString(st).decode()} {_lib.last_error()}")


# ---------------------------------------------------------------------------------------------------
# fused entry
# ---------------------------------------------------------------------------------------------------
class _PinnedRing:
    """Small ring of pinned int32 staging buffers so the label/length upload is a true async H2D copy."""

    def __init__(self, slots: int = 4):
        self.bufs = [None] * slots
        self.events = [None] * slots
        self.i = 0

    def stage(self, parts, device) -> torch.Tensor:
        n = sum(int(p.numel()) for p in parts)
        i = self.i
        self.i = (i + 1) % len(self.bufs)
        if self.events[i] is not None:
            self.events[i].synchronize()
        if self.bufs[i] is None or self.bufs[i].numel() < n:
            self.bufs[i] = torch.empty(max(n, 1024), dtype=torch.int32, pin_memory=True)
        buf = self.bufs[i][:n]
        torch.cat(parts, out=buf)
        dev = buf.to(device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        self.events[i] = ev
        return dev


_rings = {}


class _Meta:
    """An int32 meta block: its named parts packed into one pinned buffer of the device's staging ring and uploaded with one
    asynchronous copy.  `buf` is the device tensor; each part's device address is the attribute of its name."""

    def __init__(self, device, **parts):
        self.buf = _rings.setdefault(torch.device(device).index, _PinnedRing()).stage(list(parts.values()), device)
        addr = self.buf.data_ptr()
        for name, p in parts.items():
            setattr(self, name, addr)
            addr += 4 * int(p.numel())


def _label_off(ly: torch.Tensor) -> torch.Tensor:
    """Where each label sequence starts in the flat labels, and their total at the end: (len(ly) + 1,) int32."""
    off = torch.zeros(int(ly.numel()) + 1, dtype=torch.int32)
    off[1:].copy_(torch.cumsum(ly.to(torch.int64), 0))
    return off


def upload_meta(labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor, device) -> Tuple[_Meta, int]:
    """Stage [labels | label_off (N+1) | ly | lx] as one meta block.  Returns (the block, max(ly))."""
    off = _label_off(ly)
    sum_l = int(off[-1])
    if sum_l != int(labels.numel()):
        raise RuntimeError(f"labels has {labels.numel()} entries but label lengths sum to {sum_l}")
    return _Meta(device, labels=labels, label_off=off, ly=ly, lx=lx), int(ly.max()) if ly.numel() else 0


MAX_UTTS_PER_CALL = 64           # utterances per native call: the den kernels are fastest per utterance at two utterances
                                 # per lane (N=64: 35 us per frame; N=128 in one call: 79 us), and a slice of a
                                 # length-sorted batch walks only its own longest utterance (N=256, len~U{200..3000}:
                                 # 7.8 k frame steps in four slices instead of 12 k in one).  Hard limit of the kernels: 512.
_WS_FRACTION = 0.85              # of the currently free device memory a call may use for scratch


_budget_cache = {}    # device index -> [calls until the next refresh, budget in bytes]


def _scratch_budget(dev, need: int = 0) -> int:
    """What a torch allocation can get now: free device memory plus what the caching allocator holds but is not using.
    cudaMemGetInfo costs ~0.6 ms, so the answer is reused for a few calls unless the request does not fit it."""
    key = torch.device(dev).index
    ent = _budget_cache.get(key)
    if ent is not None and ent[0] > 0 and need <= ent[1]:
        ent[0] -= 1
        return ent[1]
    free, _ = torch.cuda.mem_get_info(dev)
    free += max(0, torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev))
    budget = int(free * _WS_FRACTION)
    _budget_cache[key] = [16, budget]
    return budget


CKPT_WIDTH = 32                  # a slice whose alpha spill does not fit is halved while it is wider than this (and halving
                                 # shrinks its lane padding); at or below it, it runs with checkpointed alpha instead
                                 # (DESIGN.md "Checkpointed α": on an H100, config 4's graph, T=2000, one checkpointed slice
                                 # of 64 took 0.90 s against 0.87 s for two full-spill halves; of 32, 0.61 s against 0.80 s)
_ckpt_k_override = None          # test hook: run every slice checkpointed with this interval K


def ckpt_interval(tmax: int) -> int:
    """Checkpoint interval of a slice walking `tmax` frames: ceil(sqrt(tmax)), which about minimises checkpoints + segment."""
    return max(1, math.isqrt(max(1, tmax) - 1) + 1)


def _slice_need(L, n, tmax, maxl, k, m=None, ws_bytes=None):
    """Scratch bytes of a slice of n utterances; m: its label sequences when they are not one per utterance; ws_bytes(n, tmax):
    the workspace that takes the numerator's place (the sampler's)."""
    alpha = L.ccb_den_ckpt_alpha_floats(n, tmax, k) if k else L.ccb_den_alpha_floats(n, tmax)
    ws = ws_bytes(n, tmax) if ws_bytes is not None else L.ccb_ctc_workspace_bytes(n if m is None else m, tmax, maxl)
    return int(alpha) * 4 + int(L.ccb_den_aux_bytes(n, tmax)) + int(ws)


def _slice_seqs(ly, n0, n1, seq_off):
    """(label sequences, longest one) of utterances [n0, n1): one per utterance (seq_off None), or those of a grouping."""
    if seq_off is None:
        return n1 - n0, int(ly[n0:n1].max())
    s0, s1 = int(seq_off[n0]), int(seq_off[n1])
    return s1 - s0, int(ly[s0:s1].max()) if s1 > s0 else 0


def _plan_slices(L, lx, ly, N, V, dev, seq_off=None, ws_bytes=None):
    """Split the batch into contiguous slices whose scratch (alpha spill etc.) fits the free device memory.
    Each slice walks only max(lx[slice]) frames.  Returns (n0, n1, tmax, maxl, K) per slice; K = 0 keeps every alpha
    frame, K > 0 keeps every K-th and recomputes the rest in the backward pass.
    A slice whose full alpha spill does not fit is halved while it is wider than CKPT_WIDTH and halving shrinks its lane
    padding (the spill is proportional to the padding); otherwise it runs checkpointed with K = ceil(sqrt(tmax)), and is
    halved further only if that does not fit either.
    seq_off (N+1,): several label sequences per utterance -- ly holds their lengths grouped by utterance, those of utterance
    n at seq_off[n] .. seq_off[n+1]-1, and a slice's numerator workspace is sized by its sequences.
    ws_bytes(n, tmax): the bytes of the workspace a slice needs in place of the numerator's (the posterior sampler: ly unused)."""
    budget = _scratch_budget(dev)
    slices, n0 = [], 0
    while n0 < N:
        n1 = min(N, n0 + MAX_UTTS_PER_CALL)
        while True:
            n = n1 - n0
            half = max(1, n // 2)
            tmax = max(1, int(lx[n0:n1].max()))
            m, maxl = _slice_seqs(ly, n0, n1, seq_off) if ws_bytes is None else (n, 0)
            k = 0 if _ckpt_k_override is None else int(_ckpt_k_override)
            need = _slice_need(L, n, tmax, maxl, k, m, ws_bytes)
            if need > budget:
                budget = _scratch_budget(dev, need)     # a stale (cached) figure must not split a batch needlessly
            if need <= budget:
                break
            full = need
            if k == 0 and n > CKPT_WIDTH and int(L.ccb_den_alpha_floats(half, tmax)) < int(L.ccb_den_alpha_floats(n, tmax)):
                n1 = n0 + half
                continue
            if k == 0:
                k = ckpt_interval(tmax)
                need = _slice_need(L, n, tmax, maxl, k, m, ws_bytes)
                if need > budget:
                    budget = _scratch_budget(dev, need)
                if need <= budget:
                    break
            if n == 1:
                raise RuntimeError(f"CTC-CRF scratch for a single utterance of {tmax} frames needs {full >> 20} MiB with every "
                                   f"alpha frame kept and {need >> 20} MiB checkpointed every {k} frames, "
                                   f"only {budget >> 20} MiB free")
            n1 = n0 + half
        slices.append((n0, n1, tmax, maxl, k))
        n0 = n1
    return slices


def _fwd_only_need(L, n, tmax, m=None):
    return (int(L.ccb_den_fwd_alpha_floats(n)) * 4 + int(L.ccb_den_aux_bytes(n, tmax))
            + int(L.ccb_num_fwd_only_bytes(n if m is None else m)))


def _plan_fwd_only_slices(L, lx, ly, N, dev, seq_off=None):
    """Slices of the forward-only loss: contiguous runs of at most MAX_UTTS_PER_CALL utterances, each walking its own
    max(lx).  Its alpha is a ring of a few frames whose size does not depend on the length, so a slice is never halved or
    checkpointed; one whose scratch does not fit the free device memory is an error.  Returns (n0, n1, tmax, maxl).
    seq_off: as for _plan_slices."""
    budget = _scratch_budget(dev)
    slices = []
    for n0 in range(0, N, MAX_UTTS_PER_CALL):
        n1 = min(N, n0 + MAX_UTTS_PER_CALL)
        tmax = max(1, int(lx[n0:n1].max()))
        m, maxl = _slice_seqs(ly, n0, n1, seq_off)
        need = _fwd_only_need(L, n1 - n0, tmax, m)
        if need > budget:
            budget = _scratch_budget(dev, need)
        if need > budget:
            raise RuntimeError(f"forward-only CTC-CRF scratch for {n1 - n0} utterances of up to {tmax} frames needs "
                               f"{need >> 20} MiB (alpha ring {int(L.ccb_den_fwd_alpha_floats(n1 - n0)) * 4 >> 20} MiB), "
                               f"only {budget >> 20} MiB free")
        slices.append((n0, n1, tmax, maxl))
    return slices


def _den_slices(L, dev, slices, fwd_only=False):
    """The den scratch of each slice, allocated when its turn comes: yields (i, slice, alpha_ws, aux_ws).  alpha is the
    frame ring of the forward-only loss (fwd_only; slices of _plan_fwd_only_slices), or else the full or the checkpointed
    spill by the slice's K (slices of _plan_slices).  The caller drops its references to a slice's scratch before asking for
    the next one, so that the caching allocator reuses the blocks in stream order."""
    for i, s in enumerate(slices):
        n, tmax = s[1] - s[0], s[2]
        if fwd_only:
            alpha_floats = L.ccb_den_fwd_alpha_floats(n)
        else:
            k = s[4]
            alpha_floats = L.ccb_den_ckpt_alpha_floats(n, tmax, k) if k else L.ccb_den_alpha_floats(n, tmax)
        alpha_ws = torch.empty(int(alpha_floats), dtype=torch.float32, device=dev)
        aux_ws = torch.empty(int(L.ccb_den_aux_bytes(n, tmax)), dtype=torch.uint8, device=dev)
        yield i, s, alpha_ws, aux_ws
        del alpha_ws, aux_ws


def _retry_oom(dev, run):
    """run(), and once more if it runs out of device memory: the cached memory figure was stale, so it is measured again
    and run() plans finer slices.  The retry starts after the failed attempt's buffers have been released."""
    try:
        return run()
    except torch.cuda.OutOfMemoryError:
        _budget_cache.pop(torch.device(dev).index, None)
    torch.cuda.empty_cache()
    return run()


def _batch_loss(losses: torch.Tensor) -> torch.Tensor:
    """The (1,) loss of a call from the loss of each of its slices (a single slice's is the call's)."""
    return losses.sum().reshape(1) if losses.numel() > 1 else losses


def ctc_crf_loss_fwd(logits: torch.Tensor, labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor,
                     lamb: float, size_average: bool, want_parts: bool = False, from_logits: bool = False,
                     reduction: Optional[str] = None, zero_infinity: bool = False
                     ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """Fused CTC-CRF loss.  logits (N,T,V) fp32, bf16 or fp16 CUDA contiguous log-probs; labels/lx/ly int32 CPU.
    Returns (loss[1] fp32 CUDA, grad (N,T,V) fp32 CUDA, parts[2N] or None).  Never synchronises the host.
    Batches whose scratch does not fit the free memory (or > 512 utterances) are processed in slices.
    from_logits: `logits` are the RAW encoder outputs; log_softmax and its Jacobian are applied inside
    (grad = d loss / d raw logits), replacing cat/ctc/train.py:173-174.
    reduction 'none': the first result is costs (N,) fp32 CUDA, cost[n] = logZ_den[n] - (1+lamb) log p_ctc[n], and grad is
    unscaled (grad[n] = d cost[n] / d logits[n]); size_average is then ignored.
    zero_infinity: an utterance whose cost is not finite gets cost 0 and zero gradient rows (the divisor of size_average
    stays N)."""
    return _ctc_crf_loss(logits, labels, lx, ly, lamb, size_average, want_parts, from_logits, reduction, zero_infinity, True)


def ctc_crf_loss_fwd_only(logits: torch.Tensor, labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor,
                          lamb: float, size_average: bool, want_parts: bool = False, from_logits: bool = False,
                          reduction: Optional[str] = None, zero_infinity: bool = False
                          ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """The loss of ``ctc_crf_loss_fwd`` without its gradient, for evaluation: (loss[1] fp32 CUDA, parts[2N] or None).
    The den forward pass keeps alpha on a ring of frames, the numerator writes no cells, and no (N,T,V) buffer is
    allocated, so the scratch is a few frames of the den graph per slice whatever the lengths.  Never synchronises the
    host.  Arguments as for ``ctc_crf_loss_fwd`` (reduction 'none': the first result is the (N,) costs)."""
    loss, _, parts = _ctc_crf_loss(logits, labels, lx, ly, lamb, size_average, want_parts, from_logits, reduction,
                                   zero_infinity, False)
    return loss, parts


def _ctc_crf_loss(logits, labels, lx, ly, lamb, size_average, want_parts, from_logits, reduction, zero_infinity, with_grad):
    """ctc_crf_loss_fwd (with_grad) or ctc_crf_loss_fwd_only: (loss or costs, grad or None, parts or None).  The two differ
    in the slice planner, the alpha and numerator workspaces and the native entry only."""
    per_utt = check_reduction(reduction)
    L = _lib.lib()
    N, T, V = _check_batch_args(logits, labels, lx, ly)
    dev = logits.device
    esz = logits.element_size()
    scale = 1.0 if per_utt else 1.0 / N if size_average else 1.0
    with torch.cuda.device(dev):
        meta, _ = upload_meta(labels, lx, ly, dev)
        grad = torch.empty((N, T, V), dtype=torch.float32, device=dev) if with_grad else None
        costs = torch.empty(N, dtype=torch.float32, device=dev) if per_utt else None
        parts = torch.empty(2 * N, dtype=torch.float32, device=dev) if want_parts else None
        stream = _stream(dev)

        def run_slices():
            slices = _plan_slices(L, lx, ly, N, V, dev) if with_grad else _plan_fwd_only_slices(L, lx, ly, N, dev)
            losses = torch.empty(len(slices), dtype=torch.float32, device=dev)
            for i, s, alpha_ws, aux_ws in _den_slices(L, dev, slices, fwd_only=not with_grad):
                n0, n1, tmax, maxl = s[:4]
                n = n1 - n0
                # the numerator's cells and log-likelihoods, or its log-likelihoods alone
                num_bytes = L.ccb_ctc_workspace_bytes(n, tmax, maxl) if with_grad else L.ccb_num_fwd_only_bytes(n)
                num_ws = torch.empty(int(num_bytes), dtype=torch.uint8, device=dev)
                sub_parts = torch.empty(2 * n, dtype=torch.float32, device=dev) if want_parts else None
                y = (logits.data_ptr() + n0 * T * V * esz, _DTYPES[logits.dtype], int(from_logits), n, T, V, tmax)
                ins = (meta.labels, meta.label_off + 4 * n0, meta.ly + 4 * n0, meta.lx + 4 * n0, maxl, float(lamb),
                       float(scale), alpha_ws.data_ptr(), aux_ws.data_ptr(), num_ws.data_ptr())
                # each slice writes its own costs[n0:n1] (and grad[n0:n1]) in place
                outs = (losses.data_ptr() + 4 * i, _ptr(sub_parts), costs.data_ptr() + 4 * n0 if per_utt else None,
                        int(zero_infinity), stream)
                if with_grad:
                    rc = L.ccb_ctc_crf_loss_costs(*y, s[4], *ins, grad.data_ptr() + n0 * T * V * 4, *outs)
                else:
                    rc = L.ccb_ctc_crf_loss_costs_fwd_only(*y, *ins, *outs)
                _check(rc, "ctc_crf_loss_fwd" if with_grad else "ctc_crf_loss_fwd_only")
                if want_parts:
                    parts[n0:n1] = sub_parts[:n]
                    parts[N + n0:N + n1] = sub_parts[n:]
                del alpha_ws, aux_ws, num_ws      # stream-ordered reuse by the caching allocator for the next slice
            return losses

        # the forward-only planner never reslices: there is nothing to retry
        losses = _retry_oom(dev, run_slices) if with_grad else run_slices()
        loss = _batch_loss(losses)
        meta.buf.record_stream(torch.cuda.current_stream(dev))
    return (costs if per_utt else loss), grad, parts


def _check_batch_args(logits, labels, lx, ly):
    assert logits.is_cuda and logits.dim() == 3 and logits.is_contiguous()
    if logits.dtype not in _DTYPES:
        raise RuntimeError(f"unsupported logits dtype {logits.dtype}")
    N, T, V = logits.shape
    if N == 0:
        raise RuntimeError("empty batch")
    if int(lx.numel()) != N or int(ly.numel()) != N:
        raise RuntimeError("lx / ly must have one entry per utterance")
    if int(lx.max()) > T or int(lx.min()) < 0:
        raise RuntimeError("input lengths must lie in [0, T]")
    if int(ly.min()) < 0:
        raise RuntimeError("label lengths must be non-negative")
    if labels.numel() and (int(labels.min()) < 0 or int(labels.max()) >= V):
        raise RuntimeError("label out of range")
    return N, T, V


def ctc_loss_fwd(logits: torch.Tensor, labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor,
                 size_average: bool, blank: int = 0, reduction: Optional[str] = None, zero_infinity: bool = False
                 ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """CTC-only loss on the (N,T,V) log-probs in place (the native counterpart of ``_WARP_CTC_GPU``,
    ctc_crf/__init__.py:25-56): no (T,N,V) transpose copy, no zero fill, no host round trip for the costs.
    Returns (loss[1], grad (N,T,V) fp32 = d loss / d logits, logp[N]) on the device; never synchronises the host.
    reduction 'none': the first result is costs (N,), cost[n] = -log p[n], and grad is unscaled; zero_infinity: a cost
    that is not finite becomes 0 and its gradient rows zeros (as in ``ctc_crf_loss_fwd``)."""
    return _ctc_loss(logits, labels, lx, ly, size_average, blank, reduction, zero_infinity, True)


def ctc_loss_fwd_only(logits: torch.Tensor, labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor,
                      size_average: bool, blank: int = 0, reduction: Optional[str] = None, zero_infinity: bool = False
                      ) -> Tuple[torch.Tensor, torch.Tensor]:
    """The loss of ``ctc_loss_fwd`` without its gradient: (loss[1], logp[N]) on the device, the same values, from one alpha
    chain per utterance that writes no cells.  No workspace, no (N,T,V) buffer, no host synchronisation.
    reduction and zero_infinity as for ``ctc_loss_fwd``."""
    loss, _, logp = _ctc_loss(logits, labels, lx, ly, size_average, blank, reduction, zero_infinity, False)
    return loss, logp


def _ctc_loss(logits, labels, lx, ly, size_average, blank, reduction, zero_infinity, with_grad):
    """ctc_loss_fwd (with_grad) or ctc_loss_fwd_only: (loss or costs, grad or None, logp)."""
    per_utt = check_reduction(reduction)
    L = _lib.lib()
    N, T, V = _check_batch_args(logits, labels, lx, ly)
    dev = logits.device
    scale = 1.0 if per_utt else 1.0 / N if size_average else 1.0
    with torch.cuda.device(dev):
        meta, maxl = upload_meta(labels, lx, ly, dev)
        tmax = max(1, int(lx.max()))
        grad = torch.empty((N, T, V), dtype=torch.float32, device=dev) if with_grad else None
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        logp = torch.empty(N, dtype=torch.float32, device=dev)
        ws = torch.empty(int(L.ccb_ctc_workspace_bytes(N, tmax, maxl)), dtype=torch.uint8, device=dev) if with_grad else None
        costs = torch.empty(N, dtype=torch.float32, device=dev) if per_utt else None
        rc = L.ccb_ctc_loss_costs(logits.data_ptr(), _DTYPES[logits.dtype], N, T, V, tmax, meta.labels, meta.label_off,
                                  meta.ly, meta.lx, maxl, int(blank), float(scale), _ptr(ws), _ptr(grad), loss.data_ptr(),
                                  logp.data_ptr(), _ptr(costs), int(zero_infinity), _stream(dev))
        _check(rc, "ctc_loss_fwd" if with_grad else "ctc_loss_fwd_only")
        meta.buf.record_stream(torch.cuda.current_stream(dev))
    return (costs if per_utt else loss), grad, logp


def ctc_align(logits: torch.Tensor, labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor, blank: int = 0
              ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Best-path (Viterbi) forced alignment over the numerator lattice (SURVEY 8f-4).  logits (N,T,V) fp32/bf16/fp16
    CUDA log-probs; labels/lx/ly int32 CPU as for the loss.  Returns (align (N,T) int32 CUDA: the token of every frame
    t < lx[n], blank included, -1 beyond; score (N,) fp32 CUDA: log-probability of that path, -inf if infeasible)."""
    L = _lib.lib()
    N, T, V = _check_batch_args(logits, labels, lx, ly)
    dev = logits.device
    with torch.cuda.device(dev):
        meta, maxl = upload_meta(labels, lx, ly, dev)
        align = torch.empty((N, T), dtype=torch.int32, device=dev)
        score = torch.empty(N, dtype=torch.float32, device=dev)
        ws = torch.empty(int(L.ccb_ctc_align_workspace_bytes(N, T, maxl)), dtype=torch.uint8, device=dev)
        rc = L.ccb_ctc_align(logits.data_ptr(), _DTYPES[logits.dtype], T * V, V, N, T, V, meta.labels, meta.label_off, meta.ly,
                             meta.lx, maxl, int(blank), ws.data_ptr(), align.data_ptr(), score.data_ptr(), _stream(dev))
        _check(rc, "ctc_align")
        meta.buf.record_stream(torch.cuda.current_stream(dev))
    return align, score


def grad_rows_scale(grad: torch.Tensor, w: torch.Tensor, lx: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Backward of the per-utterance costs: out[n] = w[n] * grad[n] in `dtype` (fp32, bf16 or fp16), rows t >= lx[n] zero,
    in one pass over the (N,T,V) fp32 `grad` of a loss function called with reduction 'none'.  w: (N,) the gradient with
    respect to each cost; lx: the int32 CPU input lengths of the forward call (uploaded asynchronously)."""
    L = _lib.lib()
    assert grad.is_cuda and grad.dtype == torch.float32 and grad.dim() == 3 and grad.is_contiguous()
    if dtype not in _DTYPES:
        raise RuntimeError(f"unsupported gradient dtype {dtype}")
    N, T, V = grad.shape
    dev = grad.device
    with torch.cuda.device(dev):
        w = w.to(device=dev, dtype=torch.float32).reshape(N).contiguous()
        lens = _rings.setdefault(torch.device(dev).index, _PinnedRing()).stage([lx.to(torch.int32)], dev)
        out = torch.empty((N, T, V), dtype=dtype, device=dev)
        rc = L.ccb_grad_rows_scale(grad.data_ptr(), w.data_ptr(), lens.data_ptr(), N, T, V, out.data_ptr(), _DTYPES[dtype],
                                   _stream(dev))
        _check(rc, "grad_rows_scale")
        lens.record_stream(torch.cuda.current_stream(dev))
    return out


# ---------------------------------------------------------------------------------------------------
# several label sequences per utterance (utt=)
# ---------------------------------------------------------------------------------------------------
class SeqGroups:
    """M label sequences grouped by the logits row they are scored against, in the caller's order within a row.
    pos[j]: the caller's index of grouped sequence j; row[j]: its logits row; labels / ly: the grouped sequences;
    off (N+1,) int64: the sequences of row n are off[n] .. off[n+1]-1."""

    def __init__(self, pos, row, labels, ly, off):
        self.pos, self.row, self.labels, self.ly, self.off = pos, row, labels, ly, off
        self.M = int(pos.numel())


def group_seqs(utt: torch.Tensor, labels: torch.Tensor, ly: torch.Tensor, N: int) -> SeqGroups:
    """Check `utt` ((M,) int32 CPU, entries in [0, N), one per label sequence of `ly`) and group the sequences by row with a
    stable sort.  Host work only: the labels are on the CPU already."""
    if not isinstance(utt, torch.Tensor) or utt.dtype != torch.int32 or utt.is_cuda or utt.dim() != 1:
        what = f"{utt.dtype} {utt.device} of shape {tuple(utt.shape)}" if isinstance(utt, torch.Tensor) else type(utt).__name__
        raise RuntimeError(f"utt must be a 1-D int32 CPU tensor (the logits row of each label sequence), not {what}")
    M = int(utt.numel())
    if int(ly.numel()) != M:
        raise RuntimeError(f"utt has {M} entries but ly has {int(ly.numel())}: both need one entry per label sequence")
    if M == 0:
        raise RuntimeError("utt names no label sequence")
    if int(utt.min()) < 0 or int(utt.max()) >= N:
        raise RuntimeError(f"utt entries must lie in [0, N) = [0, {N}): they name logits rows")
    if int(ly.min()) < 0:
        raise RuntimeError("label lengths must be non-negative")
    u = utt.to(torch.int64)
    pos = torch.sort(u, stable=True).indices
    ly64 = ly.to(torch.int64)
    total = int(ly64.sum())
    if total != int(labels.numel()):
        raise RuntimeError(f"labels has {labels.numel()} entries but label lengths sum to {total}")
    gly = ly64[pos]
    src = (torch.cumsum(ly64, 0) - ly64)[pos]          # where each grouped sequence starts in the caller's labels
    dst = torch.cumsum(gly, 0) - gly                   # ... and in the grouped labels
    idx = torch.repeat_interleave(src - dst, gly, output_size=total) + torch.arange(total)
    off = torch.zeros(N + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.bincount(u, minlength=N), 0)
    return SeqGroups(pos.to(torch.int32), u[pos].to(torch.int32), labels.reshape(-1)[idx].to(torch.int32),
                     gly.to(torch.int32), off)


def _check_seq_args(logits, labels, lx, ly, utt):
    assert logits.is_cuda and logits.dim() == 3 and logits.is_contiguous()
    if logits.dtype not in _DTYPES:
        raise RuntimeError(f"unsupported logits dtype {logits.dtype}")
    N, T, V = logits.shape
    if N == 0:
        raise RuntimeError("empty batch")
    if int(lx.numel()) != N:
        raise RuntimeError("lx must have one entry per utterance (logits row)")
    if int(lx.max()) > T or int(lx.min()) < 0:
        raise RuntimeError("input lengths must lie in [0, T]")
    if labels.numel() and (int(labels.min()) < 0 or int(labels.max()) >= V):
        raise RuntimeError("label out of range")
    return N, T, V, group_seqs(utt, labels, ly, N)


class _SeqMeta(_Meta):
    """The meta block of a grouped call:
    [labels | label_off (M+1) | ly (M) | lx (N) | row (M) | pos (M) | seq_off, (n1-n0+1) entries per slice]
    row and seq_off are relative to the slice that holds the sequence (its logits pointer and first sequence); pos is the
    caller's index.  Slice i of utterances [n0, n1) finds its offsets at seq_off + n0 + i."""

    def __init__(self, grp: SeqGroups, lx: torch.Tensor, bounds, device):
        N = int(lx.numel())
        first = torch.empty(N, dtype=torch.int64)            # first utterance of the slice of each utterance
        offs = []
        for n0, n1 in bounds:
            first[n0:n1] = n0
            offs.append(grp.off[n0:n1 + 1] - grp.off[n0])
        row = (grp.row.to(torch.int64) - first[grp.row.to(torch.int64)]).to(torch.int32)
        super().__init__(device, labels=grp.labels, label_off=_label_off(grp.ly), ly=grp.ly, lx=lx.to(torch.int32),
                         row=row, pos=grp.pos, seq_off=torch.cat(offs).to(torch.int32))

    def slice_args(self, i, n0, s0):
        """(labels, label_off, label_len, len, row, pos, seq_off) of slice i, utterances from n0, sequences from s0."""
        return (self.labels, self.label_off + 4 * s0, self.ly + 4 * s0, self.lx + 4 * n0, self.row + 4 * s0,
                self.pos + 4 * s0, self.seq_off + 4 * (n0 + i))


class SeqsGradState:
    """What the backward of a grouped call with reduction 'none' needs: the logits, the meta block, and per slice the numerator
    cells (and the den aux block) of the forward call, plus the unscaled den occupancies `den` (None for CTC)."""

    def __init__(self, logits, meta, slices, den, from_logits, zero_infinity, num_coef, blank, M):
        self.logits, self.meta, self.slices, self.den = logits, meta, slices, den
        self.from_logits, self.zero_infinity, self.num_coef, self.blank, self.M = from_logits, zero_infinity, num_coef, blank, M


def ctc_crf_loss_seqs(logits: torch.Tensor, labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor, utt: torch.Tensor,
                      lamb: float, size_average: bool, from_logits: bool = False, reduction: Optional[str] = None,
                      zero_infinity: bool = False) -> Tuple[torch.Tensor, torch.Tensor, Optional[SeqsGradState]]:
    """``ctc_crf_loss_fwd`` for M label sequences, sequence m scored against logits row utt[m]: labels / ly describe the M
    sequences, lx stays (N,).  The den passes run once per utterance, every numerator of a slice in one launch.
    cost[m] = logZ_den[utt[m]] - (1+lamb) log p_ctc[m]; reduction None: the sum over the sequences (/ M with size_average) and
    grad = its gradient.  reduction 'none': the (M,) costs in the caller's order; grad then holds the unscaled den occupancies
    and the third result is the state ``seqs_backward`` turns into the gradient for given per-sequence weights."""
    per_seq = check_reduction(reduction)
    L = _lib.lib()
    N, T, V, grp = _check_seq_args(logits, labels, lx, ly, utt)
    M = grp.M
    dev = logits.device
    esz = logits.element_size()
    scale = 1.0 if per_seq else 1.0 / M if size_average else 1.0
    with torch.cuda.device(dev):
        grad = torch.empty((N, T, V), dtype=torch.float32, device=dev)
        costs = torch.empty(M, dtype=torch.float32, device=dev) if per_seq else None
        stream = _stream(dev)

        def run_slices():
            slices = _plan_slices(L, lx, grp.ly, N, V, dev, seq_off=grp.off)
            meta = _SeqMeta(grp, lx, [(s[0], s[1]) for s in slices], dev)
            losses = torch.empty(len(slices), dtype=torch.float32, device=dev)
            kept = []
            for i, (n0, n1, tmax, maxl, k), alpha_ws, aux_ws in _den_slices(L, dev, slices):
                n = n1 - n0
                s0, m = int(grp.off[n0]), int(grp.off[n1] - grp.off[n0])
                ctc_ws = torch.empty(int(L.ccb_ctc_workspace_bytes(m, tmax, maxl)), dtype=torch.uint8, device=dev)
                lab, loff, lly, llx, row, pos, soff = meta.slice_args(i, n0, s0)
                rc = L.ccb_ctc_crf_loss_seqs(logits.data_ptr() + n0 * T * V * esz, _DTYPES[logits.dtype], int(from_logits),
                                             n, T, V, tmax, k, lab, loff, lly, llx, m, row, pos, soff, maxl, float(lamb),
                                             float(scale), alpha_ws.data_ptr(), aux_ws.data_ptr(), ctc_ws.data_ptr(),
                                             grad.data_ptr() + n0 * T * V * 4, losses.data_ptr() + 4 * i,
                                             costs.data_ptr() if per_seq else None, int(zero_infinity), int(per_seq), stream)
                _check(rc, "ctc_crf_loss_seqs")
                if per_seq:    # the backward reads this slice's numerator cells and den aux block (logZ, normalisers)
                    kept.append((n0, n1, tmax, maxl, s0, m, i, aux_ws, ctc_ws))
                del alpha_ws, aux_ws, ctc_ws
            return losses, meta, kept

        losses, meta, kept = _retry_oom(dev, run_slices)
        loss = _batch_loss(losses)
        meta.buf.record_stream(torch.cuda.current_stream(dev))
    state = (SeqsGradState(logits, meta, kept, grad, from_logits, zero_infinity, -(1.0 + float(lamb)), 0, M)
             if per_seq else None)
    return (costs if per_seq else loss), grad, state


def ctc_crf_loss_seqs_fwd_only(logits: torch.Tensor, labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor,
                               utt: torch.Tensor, lamb: float, size_average: bool, from_logits: bool = False,
                               reduction: Optional[str] = None, zero_infinity: bool = False) -> torch.Tensor:
    """The loss of ``ctc_crf_loss_seqs`` without a gradient (the passes of ``ctc_crf_loss_fwd_only``): the scalar, or the (M,)
    costs with reduction 'none'."""
    per_seq = check_reduction(reduction)
    L = _lib.lib()
    N, T, V, grp = _check_seq_args(logits, labels, lx, ly, utt)
    M = grp.M
    dev = logits.device
    esz = logits.element_size()
    scale = 1.0 if per_seq else 1.0 / M if size_average else 1.0
    with torch.cuda.device(dev):
        costs = torch.empty(M, dtype=torch.float32, device=dev) if per_seq else None
        stream = _stream(dev)
        slices = _plan_fwd_only_slices(L, lx, grp.ly, N, dev, seq_off=grp.off)
        meta = _SeqMeta(grp, lx, [(s[0], s[1]) for s in slices], dev)
        losses = torch.empty(len(slices), dtype=torch.float32, device=dev)
        for i, (n0, n1, tmax, maxl), alpha_ws, aux_ws in _den_slices(L, dev, slices, fwd_only=True):
            n = n1 - n0
            s0, m = int(grp.off[n0]), int(grp.off[n1] - grp.off[n0])
            num_ws = torch.empty(max(4, int(L.ccb_num_fwd_only_bytes(m))), dtype=torch.uint8, device=dev)
            lab, loff, lly, llx, row, pos, _ = meta.slice_args(i, n0, s0)
            rc = L.ccb_ctc_crf_loss_seqs_fwd_only(logits.data_ptr() + n0 * T * V * esz, _DTYPES[logits.dtype],
                                                  int(from_logits), n, T, V, tmax, lab, loff, lly, llx, m, row, pos, maxl,
                                                  float(lamb), float(scale), alpha_ws.data_ptr(), aux_ws.data_ptr(),
                                                  num_ws.data_ptr(), losses.data_ptr() + 4 * i,
                                                  costs.data_ptr() if per_seq else None, int(zero_infinity), stream)
            _check(rc, "ctc_crf_loss_seqs_fwd_only")
            del alpha_ws, aux_ws, num_ws
        loss = _batch_loss(losses)
        meta.buf.record_stream(torch.cuda.current_stream(dev))
    return costs if per_seq else loss


def ctc_loss_seqs(logits: torch.Tensor, labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor, utt: torch.Tensor,
                  size_average: bool, blank: int = 0, reduction: Optional[str] = None, zero_infinity: bool = False,
                  with_grad: bool = True) -> Tuple[torch.Tensor, Optional[torch.Tensor], Optional[SeqsGradState]]:
    """``ctc_loss_fwd`` for M label sequences (sequence m on logits row utt[m]), every numerator in one launch: the loss
    (reduction None: the sum over the sequences, / M with size_average; 'none': the (M,) costs -log p[m] in the caller's
    order), then grad = d loss / d logits (None without with_grad, or with reduction 'none', whose gradient comes from
    ``seqs_backward`` on the returned state)."""
    per_seq = check_reduction(reduction)
    defer = per_seq and with_grad
    L = _lib.lib()
    N, T, V, grp = _check_seq_args(logits, labels, lx, ly, utt)
    M = grp.M
    dev = logits.device
    scale = 1.0 if per_seq else 1.0 / M if size_average else 1.0
    with torch.cuda.device(dev):
        meta = _SeqMeta(grp, lx, [(0, N)], dev)
        tmax = max(1, int(lx.max()))
        maxl = int(grp.ly.max())
        grad = torch.empty((N, T, V), dtype=torch.float32, device=dev) if with_grad and not defer else None
        ws = torch.empty(int(L.ccb_ctc_workspace_bytes(M, tmax, maxl)), dtype=torch.uint8, device=dev) if with_grad else None
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        logp = torch.empty(M, dtype=torch.float32, device=dev)
        costs = torch.empty(M, dtype=torch.float32, device=dev) if per_seq else None
        lab, loff, lly, llx, row, pos, soff = meta.slice_args(0, 0, 0)
        rc = L.ccb_ctc_loss_seqs(logits.data_ptr(), _DTYPES[logits.dtype], N, T, V, tmax, lab, loff, lly, llx, M, row, pos,
                                 soff, maxl, int(blank), float(scale), _ptr(ws), _ptr(grad), loss.data_ptr(),
                                 logp.data_ptr(), _ptr(costs), int(zero_infinity), int(defer), _stream(dev))
        _check(rc, "ctc_loss_seqs")
        meta.buf.record_stream(torch.cuda.current_stream(dev))
    state = (SeqsGradState(logits, meta, [(0, N, tmax, maxl, 0, M, 0, None, ws)], None, False, zero_infinity, -1.0,
                           int(blank), M) if defer else None)
    return (costs if per_seq else loss), grad, state


def seqs_backward(state: SeqsGradState, w: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Backward of a grouped call with reduction 'none': the gradient of sum_m w[m] cost[m] with respect to the logits, in
    `dtype`.  One pass per slice over the rows of its utterances: W_n * den + num_coef * sum_m w[m] gamma_m (then the
    log_softmax Jacobian for from_logits); w (M,) in the caller's order."""
    L = _lib.lib()
    y = state.logits
    N, T, V = y.shape
    dev, esz = y.device, y.element_size()
    meta = state.meta
    with torch.cuda.device(dev):
        w = w.to(device=dev, dtype=torch.float32).reshape(state.M).contiguous()
        out = torch.empty((N, T, V), dtype=torch.float32, device=dev)
        stream = _stream(dev)
        for n0, n1, tmax, maxl, s0, m, i, aux_ws, ctc_ws in state.slices:
            lab, loff, lly, llx, _, pos, soff = meta.slice_args(i, n0, s0)
            rc = L.ccb_seqs_grad(y.data_ptr() + n0 * T * V * esz, _DTYPES[y.dtype], int(state.from_logits), n1 - n0, T, V,
                                 tmax, lab, loff, lly, llx, m, pos, soff, maxl, state.blank, float(state.num_coef),
                                 w.data_ptr(), state.den.data_ptr() + n0 * T * V * 4 if state.den is not None else None,
                                 aux_ws.data_ptr() if aux_ws is not None else None, ctc_ws.data_ptr(),
                                 int(state.zero_infinity), out.data_ptr() + n0 * T * V * 4, stream)
            _check(rc, "seqs_backward")
        meta.buf.record_stream(torch.cuda.current_stream(dev))
    return out if dtype == torch.float32 else out.to(dtype)


def ctc_align_seqs(logits: torch.Tensor, labels: torch.Tensor, lx: torch.Tensor, ly: torch.Tensor, utt: torch.Tensor,
                   blank: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """``ctc_align`` of M label sequences, sequence m aligned to logits row utt[m]: (align (M,T) int32, score (M,) fp32) in
    the caller's order."""
    L = _lib.lib()
    N, T, V, grp = _check_seq_args(logits, labels, lx, ly, utt)
    M = grp.M
    dev = logits.device
    with torch.cuda.device(dev):
        meta = _SeqMeta(grp, lx, [(0, N)], dev)
        maxl = int(grp.ly.max())
        align = torch.empty((M, T), dtype=torch.int32, device=dev)
        score = torch.empty(M, dtype=torch.float32, device=dev)
        ws = torch.empty(int(L.ccb_ctc_align_workspace_bytes(M, T, maxl)), dtype=torch.uint8, device=dev)
        lab, loff, lly, llx, row, pos, _ = meta.slice_args(0, 0, 0)
        rc = L.ccb_ctc_align_seqs(logits.data_ptr(), _DTYPES[logits.dtype], T * V, V, N, T, V, lab, loff, lly, llx, M, row,
                                  pos, maxl, int(blank), ws.data_ptr(), align.data_ptr(), score.data_ptr(), _stream(dev))
        _check(rc, "ctc_align_seqs")
        meta.buf.record_stream(torch.cuda.current_stream(dev))
    return align, score


# ---------------------------------------------------------------------------------------------------
# samples from the CTC-CRF posterior
# ---------------------------------------------------------------------------------------------------
def draw_seed(generator: Optional[torch.Generator] = None) -> int:
    """The call's 64-bit Philox key: two 32-bit draws from `generator` (a CPU torch.Generator; None: torch's default one)."""
    gen = torch.default_generator if generator is None else generator
    if not isinstance(gen, torch.Generator) or gen.device.type != "cpu":
        raise RuntimeError(f"generator must be a CPU torch.Generator, not {gen!r}")
    hi, lo = (int(x) for x in torch.randint(0, 1 << 32, (2,), generator=gen, dtype=torch.int64))
    return (hi << 32) | lo


def _check_sample_args(logits, lx, num_samples):
    if not isinstance(logits, torch.Tensor) or not logits.is_cuda or logits.dim() != 3:
        raise RuntimeError("logits must be an (N,T,V) CUDA tensor")
    if logits.dtype not in _DTYPES:
        raise RuntimeError(f"unsupported logits dtype {logits.dtype}: fp32, bf16 or fp16")
    N, T, V = logits.shape
    if N == 0 or T == 0 or V == 0:
        raise RuntimeError(f"empty logits of shape {tuple(logits.shape)}")
    if not isinstance(lx, torch.Tensor) or lx.dtype != torch.int32 or lx.is_cuda or lx.dim() != 1 or int(lx.numel()) != N:
        raise RuntimeError("lx must be an (N,) int32 CPU tensor, one input length per utterance")
    if int(lx.max()) > T or int(lx.min()) < 0:
        raise RuntimeError("input lengths must lie in [0, T]")
    if isinstance(num_samples, bool) or not isinstance(num_samples, int) or num_samples < 1:
        raise RuntimeError(f"num_samples must be an int >= 1, not {num_samples!r}")
    return N, T, V


def crf_sample(logits: torch.Tensor, lx: torch.Tensor, num_samples: int = 1, generator: Optional[torch.Generator] = None
               ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """K = num_samples paths per utterance drawn exactly from the CTC-CRF posterior over the loaded den graph.  Returns device
    tensors (tokens (N,K,T) int32, lengths (N,K) int32, align (N,K,T) int32, path_logp (N,K) fp32); see
    ``ctc_crf.crf_sample``.  Batches are sliced as for the loss, the sampler's workspace in the numerator's place; never
    synchronises the host."""
    N, T, V = _check_sample_args(logits, lx, num_samples)
    K = num_samples
    seed = draw_seed(generator)
    L = _lib.lib()
    dev = logits.device
    with torch.no_grad(), torch.cuda.device(dev):
        y = logits.detach().contiguous()
        esz = y.element_size()
        lens = _rings.setdefault(torch.device(dev).index, _PinnedRing()).stage([lx], dev)
        tokens = torch.empty((N, K, T), dtype=torch.int32, device=dev)
        lengths = torch.empty((N, K), dtype=torch.int32, device=dev)
        align = torch.empty((N, K, T), dtype=torch.int32, device=dev)
        path_logp = torch.empty((N, K), dtype=torch.float32, device=dev)
        stream = _stream(dev)

        def run_slices():
            slices = _plan_slices(L, lx, None, N, V, dev, ws_bytes=lambda n, tmax: L.ccb_crf_sample_ws_bytes(n, K, tmax))
            for _, (n0, n1, tmax, _, k), alpha_ws, aux_ws in _den_slices(L, dev, slices):
                n = n1 - n0
                sample_ws = torch.empty(int(L.ccb_crf_sample_ws_bytes(n, K, tmax)), dtype=torch.uint8, device=dev)
                rc = L.ccb_crf_sample(y.data_ptr() + n0 * T * V * esz, _DTYPES[y.dtype], n, T, V, tmax, k,
                                      lens.data_ptr() + 4 * n0, K, seed, n0, alpha_ws.data_ptr(), aux_ws.data_ptr(),
                                      sample_ws.data_ptr(), tokens.data_ptr() + n0 * K * T * 4,
                                      lengths.data_ptr() + n0 * K * 4, align.data_ptr() + n0 * K * T * 4,
                                      path_logp.data_ptr() + n0 * K * 4, stream)
                _check(rc, "crf_sample")
                del alpha_ws, aux_ws, sample_ws

        _retry_oom(dev, run_slices)
        lens.record_stream(torch.cuda.current_stream(dev))
    return tokens, lengths, align, path_logp


def samples_to_labels(tokens: torch.Tensor, lengths: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(labels, ly, utt) int32 CPU tensors of the feasible samples (lengths >= 0), utterance by utterance, sample by sample:
    the arguments ``CTC_CRF_LOSS(...)(logits, labels, lx, ly, utt=utt)`` takes.  One device-to-host copy (lengths and tokens
    together), which waits for the sampler to finish."""
    if tokens.dim() != 3 or lengths.shape != tokens.shape[:2]:
        raise RuntimeError(f"tokens must be (N,K,T) and lengths (N,K), not {tuple(tokens.shape)} and {tuple(lengths.shape)}")
    N, K, T = tokens.shape
    host = torch.cat([lengths.reshape(N * K, 1).to(torch.int32), tokens.reshape(N * K, T).to(torch.int32)], 1).cpu()
    ly = host[:, 0]
    keep = ly >= 0
    rows = host[keep, 1:]
    ly = ly[keep]
    labels = rows[torch.arange(T).unsqueeze(0) < ly.unsqueeze(1)]
    utt = torch.arange(N, dtype=torch.int32).repeat_interleave(K)[keep]
    return labels.to(torch.int32).contiguous(), ly.to(torch.int32).contiguous(), utt.contiguous()


# ---------------------------------------------------------------------------------------------------
# prefix beam search
# ---------------------------------------------------------------------------------------------------
MAX_BEAM = 128


def _check_beam_args(logits, lx, beam_size, cutoff_top_n):
    N, T, V = _check_sample_args(logits, lx, 1)
    for name, v, hi in (("beam_size", beam_size, MAX_BEAM), ("cutoff_top_n", cutoff_top_n, V)):
        if isinstance(v, bool) or not isinstance(v, int) or not 1 <= v <= hi:
            raise RuntimeError(f"{name} must be an int in [1, {hi}], not {v!r}")
    return N, T, V


def _check_lm_args(lm, alpha, beta, crf, V):
    """The LM arguments of ``ctc_beam_search`` (ValueError), checked before anything touches a device."""
    if lm is None:
        return
    if crf:
        raise ValueError("ctc_beam_search: an n-gram LM cannot be combined with crf=True (the den graph has its own LM, "
                         "and two LMs would count twice)")
    for name, v in (("alpha", alpha), ("beta", beta)):
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
            raise ValueError(f"ctc_beam_search: {name} must be a finite number, not {v!r}")
    if alpha < 0:
        raise ValueError(f"ctc_beam_search: alpha must be >= 0, not {alpha!r}")
    if lm.V != V:
        raise ValueError(f"ctc_beam_search: the LM was loaded for {lm.V} labels, the logits have V = {V}")


def ctc_beam_search(logits: torch.Tensor, lx: torch.Tensor, beam_size: int, cutoff_top_n: int, crf: bool, lm=None,
                    alpha: float = 1.0, beta: float = 0.0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """The beam_size best label sequences per utterance by CTC prefix beam search, over the logits alone (crf False) or over
    the loaded den graph (crf True), with the token n-gram LM ``lm`` (an ``ngram.NGramLM``) fused in at weight alpha and
    token bonus beta when given.  Returns device tensors (tokens (N,B,T) int32, lengths (N,B) int32, timesteps (N,B,T)
    int32, scores (N,B) fp32); see ``ctc_crf.ctc_beam_search``.  One native call for the batch; never synchronises the
    host."""
    N, T, V = _check_beam_args(logits, lx, beam_size, cutoff_top_n)
    _check_lm_args(lm, alpha, beta, crf, V)
    B = beam_size
    L = _lib.lib()
    dev = logits.device
    with torch.no_grad(), torch.cuda.device(dev):
        y = logits.detach().contiguous()
        lens = _rings.setdefault(torch.device(dev).index, _PinnedRing()).stage([lx], dev)
        tokens = torch.empty((N, B, T), dtype=torch.int32, device=dev)
        lengths = torch.empty((N, B), dtype=torch.int32, device=dev)
        timesteps = torch.empty((N, B, T), dtype=torch.int32, device=dev)
        scores = torch.empty((N, B), dtype=torch.float32, device=dev)
        ws = torch.empty(int(L.ccb_ctc_beam_search_ws_bytes(N, T, B)), dtype=torch.uint8, device=dev)
        if lm is None:
            rc = L.ccb_ctc_beam_search(y.data_ptr(), _DTYPES[y.dtype], N, T, V, lens.data_ptr(), B, int(cutoff_top_n),
                                       int(bool(crf)), ws.data_ptr(), tokens.data_ptr(), lengths.data_ptr(),
                                       timesteps.data_ptr(), scores.data_ptr(), _stream(dev))
        else:
            rc = L.ccb_ctc_beam_search_lm(y.data_ptr(), _DTYPES[y.dtype], N, T, V, lens.data_ptr(), B, int(cutoff_top_n), 0,
                                          ws.data_ptr(), tokens.data_ptr(), lengths.data_ptr(), timesteps.data_ptr(),
                                          scores.data_ptr(), lm.handle, float(alpha), float(beta), _stream(dev))
        _check(rc, "ctc_beam_search")
        lens.record_stream(torch.cuda.current_stream(dev))
    return tokens, lengths, timesteps, scores


def launch_count() -> int:
    return int(_lib.lib().ccb_launch_count())
