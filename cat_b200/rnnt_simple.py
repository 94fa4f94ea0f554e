"""RNN-T loss of CAT's ``LogAdd`` joiner on the GPU, from the encoder and predictor outputs without building the joint
tensor: the drop-in for ``warp_rnnt.rnnt_loss_simple`` that ``cat/rnnt/train.py`` calls when the joiner is ``LogAdd``.
Kernels: ``cat_b200/csrc/rnnt_kernels.cu``; definition, precision and numbers: DESIGN.md §7 "RNN-T loss, LogAdd joiner".
"""
from __future__ import annotations

from typing import Tuple

import torch
from torch.autograd import Function

from . import _lib
from ._C import _DTYPES, _check, _stream
from .rnnt import _INT32_MAX, REDUCTIONS, _int32, _on_device, _reduce, _weights


def check_rnnt_simple_args(f_enc, g_pred, labels, frames_lengths, labels_lengths, reduction, blank,
                           name="rnnt_loss_simple") -> Tuple[int, int, int, int]:
    """The arguments of ``rnnt_loss_simple`` (or of the loss called `name` that shares them), checked before anything
    touches a device: dtypes (AssertionError), then reduction, blank, shapes and -- for lengths on the CPU -- the lengths and
    the labels they select (ValueError).  Returns (N, Tmax, Umax, V)."""
    assert f_enc.dtype in _DTYPES, f"f_enc must be fp32, bf16 or fp16, not {f_enc.dtype}"
    assert g_pred.dtype == f_enc.dtype, f"g_pred must have f_enc's dtype {f_enc.dtype}, not {g_pred.dtype}"
    for arg, t in (("labels", labels), ("frames_lengths", frames_lengths), ("labels_lengths", labels_lengths)):
        assert t.dtype in (torch.int32, torch.int64), f"{arg} must be int32 or int64, not {t.dtype}"
    if reduction not in REDUCTIONS:
        raise ValueError(f"{name}: reduction must be one of {REDUCTIONS}, not {reduction!r}")
    if f_enc.dim() != 3 or g_pred.dim() != 3:
        raise ValueError(f"{name}: f_enc must be (N, Tmax, V) and g_pred (N, Umax+1, V), not "
                         f"{tuple(f_enc.shape)} and {tuple(g_pred.shape)}")
    N, Tmax, V = (int(s) for s in f_enc.shape)
    if g_pred.shape[0] != N or g_pred.shape[2] != V or g_pred.shape[1] < 1 or Tmax < 1 or N < 1 or V < 1:
        raise ValueError(f"{name}: f_enc (N, Tmax, V) and g_pred (N, Umax+1, V) must share N >= 1 and V >= 1, with "
                         f"Tmax >= 1, not {tuple(f_enc.shape)} and {tuple(g_pred.shape)}")
    Umax = int(g_pred.shape[1]) - 1
    if isinstance(blank, bool) or not isinstance(blank, int) or not 0 <= blank < V:
        raise ValueError(f"{name}: blank must be an int in [0, V) with V = {V}, not {blank!r}")
    if frames_lengths.dim() != 1 or labels_lengths.shape != frames_lengths.shape or frames_lengths.numel() != N:
        raise ValueError(f"{name}: frames_lengths and labels_lengths must both be (N,) with N = {N}, not "
                         f"{tuple(frames_lengths.shape)} and {tuple(labels_lengths.shape)}")
    if tuple(labels.shape) != (N, Umax):
        raise ValueError(f"{name}: labels must be (N, Umax) = {(N, Umax)} with g_pred (N, Umax+1, V), not "
                         f"{tuple(labels.shape)}")
    if not frames_lengths.is_cuda and not labels_lengths.is_cuda:
        T, U = frames_lengths.long(), labels_lengths.long()
        if int(T.max()) > _INT32_MAX or int(U.max()) > _INT32_MAX:
            raise ValueError(f"{name}: lengths beyond the int32 range")
        if int(T.min()) < 1 or int(U.min()) < 0:
            raise ValueError(f"{name}: every frames_length must be >= 1 and every labels_length >= 0")
        if int(T.max()) > Tmax or int(U.max()) > Umax:
            raise ValueError(f"{name}: lengths up to T = {int(T.max())}, U = {int(U.max())} overrun f_enc and "
                             f"g_pred (Tmax = {Tmax}, Umax = {Umax})")
        if not labels.is_cuda:
            used = labels[torch.arange(Umax)[None, :] < U[:, None]]
            if used.numel() and (int(used.min()) < 0 or int(used.max()) >= V or bool((used == blank).any())):
                raise ValueError(f"{name}: labels must lie in [0, {V}) and differ from blank = {blank}")
    return N, Tmax, Umax, V


def _forward(f, g, labels, lx, ly, blank, want_beta, shape, family="rnnt"):
    """One native forward of the ccb_<family>_simple_* entries ("rnnt", or "ctct" for the CTC-T loss, which takes the same
    arguments).  Returns (costs (N,) fp32, workspace, device labels)."""
    N, Tmax, Umax, V = shape
    L = _lib.lib()
    dev = f.device
    labels_d, lx_d, ly_d = _on_device(dev, _int32(labels), _int32(lx), _int32(ly))
    ws = torch.empty(int(getattr(L, f"ccb_{family}_simple_workspace_bytes")(N, Tmax, Umax)), dtype=torch.uint8, device=dev)
    costs = torch.empty(N, dtype=torch.float32, device=dev)
    rc = getattr(L, f"ccb_{family}_simple_forward")(f.data_ptr(), g.data_ptr(), _DTYPES[f.dtype], N, Tmax, Umax, V,
                                                    labels_d.data_ptr(), lx_d.data_ptr(), ly_d.data_ptr(), int(blank),
                                                    int(want_beta), ws.data_ptr(), costs.data_ptr(), _stream(dev))
    _check(rc, "rnnt_loss_simple" if family == "rnnt" else f"{family}_simple_loss")
    return costs, ws, labels_d


class _SimpleLoss(Function):
    """The LogAdd joiner's RNN-T or CTC-T loss (family "rnnt" or "ctct") with its gradients on f and g.  The forward keeps
    only the O(cells + rows) workspace; the backward writes w_n d cost_n / d f and d g in f's dtype."""

    @staticmethod
    def forward(ctx, f, g, labels, lx, ly, reduction, blank, shape, family, name):
        f, g = f.contiguous(), g.contiguous()
        costs, ws, labels_d = _forward(f, g, labels, lx, ly, blank, True, shape, family)
        ctx.f, ctx.g, ctx.ws, ctx.labels, ctx.shape, ctx.reduction, ctx.blank = f, g, ws, labels_d, shape, reduction, blank
        ctx.family, ctx.name = family, name
        return _reduce(costs, reduction)

    @staticmethod
    def backward(ctx, grad_output):
        N, Tmax, Umax, V = ctx.shape
        f, g = ctx.f, ctx.g
        dev = f.device
        w = _weights(grad_output, N, ctx.reduction, dev)
        grad_f = torch.empty(f.shape, dtype=f.dtype, device=dev)
        grad_g = torch.empty(g.shape, dtype=g.dtype, device=dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            rc = getattr(L, f"ccb_{ctx.family}_simple_backward")(f.data_ptr(), g.data_ptr(), _DTYPES[f.dtype], N, Tmax, Umax,
                                                                 V, ctx.labels.data_ptr(), int(ctx.blank), ctx.ws.data_ptr(),
                                                                 w.data_ptr(), grad_f.data_ptr(), grad_g.data_ptr(),
                                                                 _stream(dev))
        _check(rc, f"{ctx.name} backward")
        ctx.f = ctx.g = ctx.ws = ctx.labels = None
        return (grad_f if ctx.needs_input_grad[0] else None, grad_g if ctx.needs_input_grad[1] else None) + (None,) * 8


def _simple_loss(family, name, f_enc, g_pred, labels, frames_lengths, labels_lengths, reduction, blank):
    """The loss `name` of the ccb_<family>_simple_* entries: the argument checks, the forward alone under
    ``torch.no_grad`` (or for inputs that do not require grad), else the autograd Function."""
    shape = check_rnnt_simple_args(f_enc, g_pred, labels, frames_lengths, labels_lengths, reduction, blank, name)
    if not f_enc.is_cuda or g_pred.device != f_enc.device:
        raise ValueError(f"{name}: f_enc and g_pred must be on one CUDA device")
    with torch.cuda.device(f_enc.device):
        if torch.is_grad_enabled() and (f_enc.requires_grad or g_pred.requires_grad):
            return _SimpleLoss.apply(f_enc, g_pred, labels, frames_lengths, labels_lengths, reduction, blank, shape, family,
                                     name)
        costs = _forward(f_enc.detach().contiguous(), g_pred.detach().contiguous(), labels, frames_lengths, labels_lengths,
                         blank, False, shape, family)[0]
        return _reduce(costs, reduction)


def rnnt_loss_simple(f_enc: torch.Tensor, g_pred: torch.Tensor, labels: torch.Tensor, frames_lengths: torch.Tensor,
                     labels_lengths: torch.Tensor, reduction: str = "mean", blank: int = 0) -> torch.Tensor:
    """The RNN-T loss of CAT's ``LogAdd`` joiner (DESIGN.md §7 "RNN-T loss, LogAdd joiner"): ``rnnt_loss`` over the
    log-probs log_softmax(f_enc[n, t] + g_pred[n, u]), computed without the (N, Tmax, Umax+1, V) joint tensor.

    f_enc (N, Tmax, V) and g_pred (N, Umax+1, V): fp32, bf16 or fp16 of one dtype on one CUDA device, read in place; rows
    t >= T_n of f_enc and u > U_n of g_pred are never read and get zero gradient.  labels (N, Umax), padded;
    frames_lengths (T_n >= 1) and labels_lengths (U_n >= 0): int32 or int64, on the CPU or on the inputs' device.  Host
    lengths (and host labels with them) are checked against the shapes (ValueError); with device lengths an utterance that
    overruns the tensors, or a label outside [0, V) or equal to blank, gets cost NaN and zero gradient instead.
    reduction: 'mean' (default) of the N costs, 'sum' or 'none' (the (N,) fp32 costs).  No host synchronisation; the
    gradients come back in the inputs' dtype; under ``torch.no_grad`` only the forward recursion runs."""
    return _simple_loss("rnnt", "rnnt_loss_simple", f_enc, g_pred, labels, frames_lengths, labels_lengths, reduction, blank)
