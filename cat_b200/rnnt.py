"""RNN-T loss on the GPU over CAT's compact joint layout or the padded one, and the compact joiner's gather ops: the drop-ins
for ``warp_rnnt.rnnt_loss`` and ``gather.cat`` / ``gather.sum`` that CAT's transducer recipes import (``cat/rnnt/train.py``,
``cat/rnnt/joiner.py``).  Kernels: ``cat_b200/csrc/rnnt_kernels.cu``; definition and numbers: DESIGN.md §7 "RNN-T loss".
"""
from __future__ import annotations

from typing import Tuple

import torch
from torch.autograd import Function

from . import _lib
from ._C import _DTYPES, _PinnedRing, _check, _rings, _stream

REDUCTIONS = ("mean", "sum", "none")
_INT32_MAX = 2 ** 31 - 1


def check_rnnt_args(log_probs, labels, frames_lengths, labels_lengths, reduction, blank, compact,
                    name="rnnt_loss") -> Tuple[int, int, int, int, int]:
    """The arguments of ``rnnt_loss`` (or of the loss called `name` that shares them), checked before anything touches a
    device: dtypes (AssertionError, as the CTC entries assert theirs), then reduction, blank, shapes and -- for lengths on
    the CPU -- the row and label counts they imply (ValueError).  Returns (N, rows, V, Tmax, Umax); Tmax and Umax are 0 for
    the compact layout."""
    assert log_probs.dtype in _DTYPES, f"log_probs must be fp32, bf16 or fp16, not {log_probs.dtype}"
    for arg, t in (("labels", labels), ("frames_lengths", frames_lengths), ("labels_lengths", labels_lengths)):
        assert t.dtype == torch.int32, f"{arg} must be int32, not {t.dtype}"
    if reduction not in REDUCTIONS:
        raise ValueError(f"{name}: reduction must be one of {REDUCTIONS}, not {reduction!r}")
    V = int(log_probs.shape[-1]) if log_probs.dim() else 0
    if isinstance(blank, bool) or not isinstance(blank, int) or not 0 <= blank < max(V, 1) or V == 0:
        raise ValueError(f"{name}: blank must be an int in [0, V) with V = {V}, not {blank!r}")
    if frames_lengths.dim() != 1 or labels_lengths.shape != frames_lengths.shape or frames_lengths.numel() == 0:
        raise ValueError(f"{name}: frames_lengths and labels_lengths must both be (N,) with N >= 1, not "
                         f"{tuple(frames_lengths.shape)} and {tuple(labels_lengths.shape)}")
    N = int(frames_lengths.numel())
    if compact:
        if log_probs.dim() != 2 or labels.dim() != 1:
            raise ValueError(f"{name}(compact=True): log_probs must be (sum T(U+1), V) and labels (sum U,), not "
                             f"{tuple(log_probs.shape)} and {tuple(labels.shape)}")
        rows, Tmax, Umax = int(log_probs.shape[0]), 0, 0
    else:
        if log_probs.dim() != 4 or log_probs.shape[0] != N or log_probs.shape[2] < 1:
            raise ValueError(f"{name}: log_probs must be (N, Tmax, Umax+1, V) with N = {N}, not {tuple(log_probs.shape)}")
        Tmax, Umax = int(log_probs.shape[1]), int(log_probs.shape[2]) - 1
        if tuple(labels.shape) != (N, Umax):
            raise ValueError(f"{name}: labels must be (N, Umax) = {(N, Umax)}, not {tuple(labels.shape)}")
        rows = N * Tmax * (Umax + 1)
    if not frames_lengths.is_cuda and not labels_lengths.is_cuda:
        T, U = frames_lengths.long(), labels_lengths.long()
        if int(T.min()) < 1 or int(U.min()) < 0:
            raise ValueError(f"{name}: every frames_length must be >= 1 and every labels_length >= 0")
        if compact:
            need, n_lab = int((T * (U + 1)).sum()), int(U.sum())
            if need != rows:
                raise ValueError(f"{name}(compact=True): the lengths give sum T(U+1) = {need} rows, log_probs has {rows}")
            if n_lab != labels.numel():
                raise ValueError(f"{name}(compact=True): the label lengths sum to {n_lab}, labels has {labels.numel()}")
        elif int(T.max()) > Tmax or int(U.max()) > Umax:
            raise ValueError(f"{name}: lengths up to T = {int(T.max())}, U = {int(U.max())} overrun log_probs "
                             f"(Tmax = {Tmax}, Umax = {Umax})")
        if not labels.is_cuda:
            used = labels if compact else labels[torch.arange(Umax)[None, :] < U[:, None]]
            if used.numel() and (int(used.min()) < 0 or int(used.max()) >= V or bool((used == blank).any())):
                raise ValueError(f"{name}: labels must lie in [0, {V}) and differ from blank = {blank}")
    return N, rows, V, Tmax, Umax


def _on_device(dev, *ts) -> list:
    """The int32 tensors on `dev`: device ones as they are (contiguous), host ones staged together through the pinned ring
    (one asynchronous copy, no host synchronisation)."""
    out, host = list(ts), [i for i, t in enumerate(ts) if not t.is_cuda]
    for i, t in enumerate(ts):
        if t.is_cuda:
            if t.device != dev:
                raise ValueError(f"rnnt_loss: a CUDA-resident length or label tensor is on {t.device}, log_probs on {dev}")
            out[i] = t.contiguous()
    if host:
        buf = _rings.setdefault(dev.index, _PinnedRing()).stage([ts[i].reshape(-1) for i in host], dev)
        o = 0
        for i in host:
            n = int(ts[i].numel())
            out[i] = buf[o:o + n]
            o += n
    return out


def _int32(t: torch.Tensor) -> torch.Tensor:
    """int32 labels or lengths, on t's device and without a synchronisation.  int64 values outside the int32 range are
    clamped to -1 or the int32 maximum first, so that the kernels see them as invalid instead of wrapped round."""
    if t.dtype == torch.int32:
        return t
    return t.clamp(-1, _INT32_MAX).to(torch.int32)


def _forward(x, labels, lx, ly, blank, compact, from_logits, want_beta, shape, family="rnnt"):
    """One native forward of the ccb_<family>_* entries ("rnnt", or "ctct" for the CTC-T loss, which takes the same
    arguments).  Returns (costs (N,) fp32, costs from beta or None, workspace, device labels)."""
    N, rows, V, Tmax, Umax = shape
    L = _lib.lib()
    dev = x.device
    labels_d, lx_d, ly_d = _on_device(dev, labels, lx, ly)
    ws = torch.empty(int(getattr(L, f"ccb_{family}_workspace_bytes")(N, rows)), dtype=torch.uint8, device=dev)
    costs = torch.empty(N, dtype=torch.float32, device=dev)
    costs_b = torch.empty(N, dtype=torch.float32, device=dev) if want_beta else None
    rc = getattr(L, f"ccb_{family}_forward")(x.data_ptr(), _DTYPES[x.dtype], int(from_logits), int(compact), N, rows, V,
                                             Tmax, Umax, labels_d.data_ptr(), int(labels_d.numel()), lx_d.data_ptr(),
                                             ly_d.data_ptr(), int(blank), int(want_beta), ws.data_ptr(), costs.data_ptr(),
                                             None if costs_b is None else costs_b.data_ptr(), _stream(dev))
    _check(rc, f"{family}_loss")
    return costs, costs_b, ws, labels_d


def _reduce(costs, reduction):
    if reduction == "mean":
        return costs.mean()
    return costs.sum() if reduction == "sum" else costs


def _weights(grad_output, N, reduction, dev):
    """The per-utterance weights w_n of the backward: grad_output, / N for 'mean', expanded to (N,) fp32."""
    g = grad_output.to(device=dev, dtype=torch.float32)
    w = (g / N).expand(N) if reduction == "mean" else g.expand(N) if reduction == "sum" else g
    return w.contiguous()


class _Loss(Function):
    """The RNN-T or CTC-T loss (family "rnnt" or "ctct") with its gradient.  The forward runs the row pass and alpha ||
    beta, keeping only the O(rows) workspace; the backward writes w_n d cost_n / d x in one pass, in x's dtype."""

    @staticmethod
    def forward(ctx, x, labels, lx, ly, reduction, blank, compact, from_logits, shape, family, name):
        x = x.contiguous()
        costs, _, ws, labels_d = _forward(x, labels, lx, ly, blank, compact, from_logits, True, shape, family)
        ctx.ws, ctx.labels, ctx.shape, ctx.reduction, ctx.blank, ctx.from_logits = ws, labels_d, shape, reduction, blank, from_logits
        ctx.family, ctx.name = family, name
        ctx.x = x if from_logits else None
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        return _reduce(costs, reduction)

    @staticmethod
    def backward(ctx, grad_output):
        N, rows, V = ctx.shape[:3]
        dev = ctx.ws.device
        w = _weights(grad_output, N, ctx.reduction, dev)
        grad = torch.empty(ctx.x_shape, dtype=ctx.x_dtype, device=dev)
        x = ctx.x
        L = _lib.lib()
        with torch.cuda.device(dev):
            rc = getattr(L, f"ccb_{ctx.family}_backward")(None if x is None else x.data_ptr(), _DTYPES[ctx.x_dtype],
                                                          int(ctx.from_logits), N, rows, V, ctx.labels.data_ptr(),
                                                          int(ctx.blank), ctx.ws.data_ptr(), w.data_ptr(), grad.data_ptr(),
                                                          _stream(dev))
        _check(rc, f"{ctx.name} backward")
        ctx.ws = ctx.x = ctx.labels = None
        return (grad,) + (None,) * 10


def _loss(family, name, log_probs, labels, frames_lengths, labels_lengths, reduction, blank, compact, from_logits):
    """The loss `name` of the ccb_<family>_* entries over the joint tensor: the argument checks, the forward alone under
    ``torch.no_grad`` (or for an input that does not require grad), else the autograd Function."""
    shape = check_rnnt_args(log_probs, labels, frames_lengths, labels_lengths, reduction, blank, compact, name)
    if not log_probs.is_cuda:
        raise ValueError(f"{name}: log_probs must be on a CUDA device")
    with torch.cuda.device(log_probs.device):
        if torch.is_grad_enabled() and log_probs.requires_grad:
            return _Loss.apply(log_probs, labels, frames_lengths, labels_lengths, reduction, blank, bool(compact),
                               bool(from_logits), shape, family, name)
        costs = _forward(log_probs.detach().contiguous(), labels, frames_lengths, labels_lengths, blank, compact, from_logits,
                         False, shape, family)[0]
        return _reduce(costs, reduction)


def _costs_both_ways(family, name, log_probs, labels, frames_lengths, labels_lengths, blank, compact, from_logits):
    shape = check_rnnt_args(log_probs, labels, frames_lengths, labels_lengths, "none", blank, compact, name)
    with torch.no_grad(), torch.cuda.device(log_probs.device):
        costs, costs_b, _, _ = _forward(log_probs.contiguous(), labels, frames_lengths, labels_lengths, blank, compact,
                                        from_logits, True, shape, family)
    return costs, costs_b


def rnnt_loss(log_probs: torch.Tensor, labels: torch.Tensor, frames_lengths: torch.Tensor, labels_lengths: torch.Tensor,
              reduction: str = "mean", blank: int = 0, compact: bool = False, from_logits: bool = False) -> torch.Tensor:
    """The RNN-T loss (DESIGN.md §7 "RNN-T loss"): cost_n = -log P(y_n | x_n) over the transducer lattice of utterance n,
    as ``torchaudio.functional.rnnt_loss`` defines it, on the GPU and without a host synchronisation.

    log_probs: fp32, bf16 or fp16 on the GPU, read in place.  compact=True (CAT's layout): (sum_n T_n (U_n+1), V), utterance
    n's row (t, u) at off_n + t (U_n+1) + u, and labels (sum_n U_n,) concatenated; compact=False: (N, Tmax, Umax+1, V) and
    labels (N, Umax), where rows outside t < T_n, u <= U_n are never read.  Log-probs by default (what CAT's
    ``AbsJointNet.forward`` returns, gradient -posterior at the blank and label entries); ``from_logits=True`` takes the raw
    joiner output (``JointNet.impl_forward``) and applies the log-softmax inside, with its Jacobian, without a normalised copy.
    labels, frames_lengths (T_n >= 1), labels_lengths (U_n >= 0): int32, on the CPU or on log_probs' device.  Host lengths
    are checked against the shapes (ValueError); with device lengths an utterance that overruns the tensors, or a label outside
    [0, V) or equal to blank, gets cost NaN and zero gradient instead.  reduction: 'mean' (default) of the N costs, 'sum' or
    'none' (the (N,) fp32 costs).  The gradient comes back in log_probs' dtype.  Under ``torch.no_grad`` (or for an input
    that does not require grad) only the forward recursion runs."""
    return _loss("rnnt", "rnnt_loss", log_probs, labels, frames_lengths, labels_lengths, reduction, blank, compact, from_logits)


def rnnt_costs_both_ways(log_probs, labels, frames_lengths, labels_lengths, blank=0, compact=False, from_logits=False):
    """The (N,) costs from alpha and from beta, which agree up to rounding (a check of the two recursions)."""
    return _costs_both_ways("rnnt", "rnnt_loss", log_probs, labels, frames_lengths, labels_lengths, blank, compact,
                            from_logits)


# ---------------------------------------------------------------------------------------------------
# the compact joiner's gather ops
# ---------------------------------------------------------------------------------------------------
def gather_cat(x: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
    """``gather.cat``: the first lengths[n] entries of x[n] for each n, concatenated: (N, T, *) -> (sum lengths, *).  Plain
    indexing (autograd differentiates it); the mask costs one host synchronisation, as ``torch-gather`` does."""
    mask = torch.arange(x.shape[1], device=x.device)[None, :] < lengths.to(x.device)[:, None]
    return x[mask]


class _GatherSum(Function):
    @staticmethod
    def forward(ctx, a, b, la, lb, rows_out):
        L = _lib.lib()
        dev = a.device
        N, H = int(la.numel()), int(a.shape[1])
        out = torch.empty((rows_out, H), dtype=a.dtype, device=dev)
        ws = torch.empty(int(L.ccb_gather_ws_bytes(N)), dtype=torch.uint8, device=dev)
        _check(L.ccb_gather_sum(a.data_ptr(), b.data_ptr(), _DTYPES[a.dtype], N, rows_out, H, la.data_ptr(), lb.data_ptr(),
                                ws.data_ptr(), out.data_ptr(), _stream(dev)), "gather_sum")
        ctx.save_for_backward(la, lb)
        ctx.rows = (int(a.shape[0]), int(b.shape[0]))
        return out

    @staticmethod
    def backward(ctx, grad_out):
        la, lb = ctx.saved_tensors
        L = _lib.lib()
        dev = la.device
        g = grad_out.contiguous()
        N, H = int(la.numel()), int(g.shape[1])
        ga = torch.empty((ctx.rows[0], H), dtype=g.dtype, device=dev)
        gb = torch.empty((ctx.rows[1], H), dtype=g.dtype, device=dev)
        ws = torch.empty(int(L.ccb_gather_ws_bytes(N)), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _check(L.ccb_gather_sum_backward(g.data_ptr(), _DTYPES[g.dtype], N, ctx.rows[0], ctx.rows[1], H, la.data_ptr(),
                                             lb.data_ptr(), ws.data_ptr(), ga.data_ptr(), gb.data_ptr(), _stream(dev)),
                   "gather_sum backward")
        return ga, gb, None, None, None


def gather_sum(a: torch.Tensor, b: torch.Tensor, la: torch.Tensor, lb: torch.Tensor) -> torch.Tensor:
    """``gather.sum``: the compact broadcast sum of CAT's joiner, out[off_n + t lb_n + u] = a[ta_n + t] + b[ub_n + u] with
    a (sum la, H), b (sum lb, H) and out (sum la lb, H), where ta_n, ub_n and off_n are the running sums over the earlier
    utterances.  fp32, bf16 or fp16 (a and b alike); la, lb integer lengths on the CPU or the GPU.  With both on the CPU the
    sizes are taken on the host and the lengths uploaded asynchronously, so the call does not synchronise; sizing the output
    costs one host synchronisation when the lengths are on the GPU.  The backward sums in fp32 without atomics."""
    if a.dtype not in _DTYPES or b.dtype != a.dtype:
        raise ValueError(f"gather_sum: a and b must share one of fp32, bf16, fp16, not {a.dtype} and {b.dtype}")
    if a.dim() != 2 or b.dim() != 2 or a.shape[1] != b.shape[1] or a.shape[1] == 0:
        raise ValueError(f"gather_sum: a and b must be (rows, H) with the same H >= 1, not {tuple(a.shape)} and {tuple(b.shape)}")
    if la.dim() != 1 or lb.shape != la.shape or la.numel() == 0:
        raise ValueError(f"gather_sum: la and lb must both be (N,) with N >= 1, not {tuple(la.shape)} and {tuple(lb.shape)}")
    if not a.is_cuda or b.device != a.device:
        raise ValueError("gather_sum: a and b must be on one CUDA device")
    dev = a.device
    host = not la.is_cuda and not lb.is_cuda
    with torch.cuda.device(dev):
        la64, lb64 = (la.long(), lb.long()) if host else (la.to(dev, torch.int64), lb.to(dev, torch.int64))
        rows_out, sa, sb, lo = (int(v) for v in torch.stack([(la64 * lb64).sum(), la64.sum(), lb64.sum(),
                                                              torch.minimum(la64.min(), lb64.min())]).tolist())
        if lo < 0 or sa != a.shape[0] or sb != b.shape[0]:
            raise ValueError(f"gather_sum: the lengths (sums {sa}, {sb}, min {lo}) do not match a {tuple(a.shape)} and "
                             f"b {tuple(b.shape)}")
        la32, lb32 = _on_device(dev, la64.to(torch.int32), lb64.to(torch.int32))
        return _GatherSum.apply(a.contiguous(), b.contiguous(), la32, lb32, rows_out)
