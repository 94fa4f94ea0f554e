"""CTC-T (CTC-Transducer) loss on the GPU: the drop-ins for ``warp_ctct.ctct_loss`` and ``warp_ctct.ctct_simple_loss`` that
CAT's transducer trainer calls with ``"trainer": {"topo": "ctct"}`` (``cat/rnnt/train.py``), for the ``JointNet`` and the
``LogAdd`` joiner.  Kernels: ``cat_b200/csrc/rnnt_kernels.cu``; definition, precision and numbers: DESIGN.md §7 "CTC-T loss".

Every frame emits exactly one symbol, as in CTC, and reads the joint row of the labels emitted so far, as in RNN-T.  With
lp(t,u,k) the log-prob of token k at row (t,u) and logaddexp written (+), over the states (u, b) (u labels emitted, the last
emission blank or none yet) and (u, l) (the last emission y_u):
    alpha_{t+1}(u,b) = [alpha_t(u,b) (+) alpha_t(u,l)] + lp(t,u,blank)
    alpha_{t+1}(u,l) = [alpha_t(u,l) + lp(t,u,y_u)] (+) [alpha_t(u-1,b) + lp(t,u-1,y_u)]
                       (+) [alpha_t(u-1,l) + lp(t,u-1,y_u)]   (only if u = 1 or y_u != y_{u-1})
    cost = -(alpha_T(U,b) (+) alpha_T(U,l)),  alpha_0(0,b) = 0 and every other alpha_0 = -inf.
"""
from __future__ import annotations

import torch
from torch.autograd import Function

from . import _lib
from ._C import _DTYPES, _check, _stream
from . import rnnt as _rnnt
from . import rnnt_simple as _simple
from .rnnt import _reduce


def _weights(grad_output, N, reduction, dev):
    """The per-utterance weights w_n of the backward: grad_output, / N for 'mean', expanded to (N,) fp32."""
    g = grad_output.to(device=dev, dtype=torch.float32)
    w = (g / N).expand(N) if reduction == "mean" else g.expand(N) if reduction == "sum" else g
    return w.contiguous()


class _CTCT(Function):
    """The CTC-T loss with its gradient.  The forward runs the row pass and alpha || beta, keeping only the O(rows)
    workspace; the backward writes w_n d cost_n / d x in one pass, in x's dtype."""

    @staticmethod
    def forward(ctx, x, labels, lx, ly, reduction, blank, compact, from_logits, shape):
        x = x.contiguous()
        costs, _, ws, labels_d = _rnnt._forward(x, labels, lx, ly, blank, compact, from_logits, True, shape, "ctct")
        ctx.ws, ctx.labels, ctx.shape, ctx.reduction, ctx.blank, ctx.from_logits = ws, labels_d, shape, reduction, blank, from_logits
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
            rc = L.ccb_ctct_backward(None if x is None else x.data_ptr(), _DTYPES[ctx.x_dtype], int(ctx.from_logits), N, rows, V,
                                     ctx.labels.data_ptr(), int(ctx.blank), ctx.ws.data_ptr(), w.data_ptr(), grad.data_ptr(),
                                     _stream(dev))
        _check(rc, "ctct_loss backward")
        ctx.ws = ctx.x = ctx.labels = None
        return (grad,) + (None,) * 8


def _layout(log_probs, compact) -> bool:
    """compact=None takes the layout from log_probs' rank: 2 -> compact, 4 -> padded (CAT's call passes no flag and hands
    the compact joiner's 2-D output when the trainer has ``compact: true``).  An explicit value is checked against the
    shape by the argument checks."""
    if compact is not None:
        return bool(compact)
    if log_probs.dim() not in (2, 4):
        raise ValueError(f"ctct_loss: log_probs must be (sum T(U+1), V) (compact) or (N, Tmax, Umax+1, V) (padded), not "
                         f"{tuple(log_probs.shape)}")
    return log_probs.dim() == 2


def ctct_loss(log_probs: torch.Tensor, labels: torch.Tensor, frames_lengths: torch.Tensor, labels_lengths: torch.Tensor,
              reduction: str = "mean", blank: int = 0, compact=None, from_logits: bool = False) -> torch.Tensor:
    """The CTC-T loss (DESIGN.md §7 "CTC-T loss"): cost_n = -log P(y_n | x_n) over the CTC-T lattice of utterance n, on the
    GPU and without a host synchronisation.  If lp(t,u,k) does not depend on u, this is the CTC cost.

    Every convention is ``rnnt_loss``'s: log_probs fp32, bf16 or fp16 on the GPU, read in place, in the compact layout
    (sum_n T_n (U_n+1), V) with labels (sum_n U_n,), or the padded one (N, Tmax, Umax+1, V) with labels (N, Umax), whose
    rows outside t < T_n, u <= U_n are never read; compact=None (default) takes the layout from log_probs' rank, an
    explicit value must agree with it.  Log-probs by default, raw joiner output with ``from_logits=True``.  labels and
    lengths int32 on the CPU or on log_probs' device; host lengths are checked (ValueError), and with device lengths a bad
    utterance gets cost NaN and zero gradient.  An infeasible utterance (T_n < U_n + the number of adjacent repeats in its
    labels) gets cost +inf and zero gradient.  reduction 'mean' (default), 'sum' or 'none'.  The gradient comes back in
    log_probs' dtype; under ``torch.no_grad`` (or for an input that does not require grad) only alpha runs."""
    compact = _layout(log_probs, compact)
    shape = _rnnt.check_rnnt_args(log_probs, labels, frames_lengths, labels_lengths, reduction, blank, compact, "ctct_loss")
    if not log_probs.is_cuda:
        raise ValueError("ctct_loss: log_probs must be on a CUDA device")
    with torch.cuda.device(log_probs.device):
        if torch.is_grad_enabled() and log_probs.requires_grad:
            return _CTCT.apply(log_probs, labels, frames_lengths, labels_lengths, reduction, blank, compact, bool(from_logits),
                               shape)
        costs = _rnnt._forward(log_probs.detach().contiguous(), labels, frames_lengths, labels_lengths, blank, compact,
                               from_logits, False, shape, "ctct")[0]
        return _reduce(costs, reduction)


def ctct_costs_both_ways(log_probs, labels, frames_lengths, labels_lengths, blank=0, compact=None, from_logits=False):
    """The (N,) costs from alpha and from beta, which agree up to rounding (a check of the two recursions)."""
    compact = _layout(log_probs, compact)
    shape = _rnnt.check_rnnt_args(log_probs, labels, frames_lengths, labels_lengths, "none", blank, compact, "ctct_loss")
    with torch.no_grad(), torch.cuda.device(log_probs.device):
        costs, costs_b, _, _ = _rnnt._forward(log_probs.contiguous(), labels, frames_lengths, labels_lengths, blank, compact,
                                              from_logits, True, shape, "ctct")
    return costs, costs_b


class _CTCTSimple(Function):
    """The LogAdd joiner's CTC-T loss with its gradients on f and g, in f's dtype."""

    @staticmethod
    def forward(ctx, f, g, labels, lx, ly, reduction, blank, shape):
        f, g = f.contiguous(), g.contiguous()
        costs, ws, labels_d = _simple._forward(f, g, labels, lx, ly, blank, True, shape, "ctct")
        ctx.f, ctx.g, ctx.ws, ctx.labels, ctx.shape, ctx.reduction, ctx.blank = f, g, ws, labels_d, shape, reduction, blank
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
            rc = L.ccb_ctct_simple_backward(f.data_ptr(), g.data_ptr(), _DTYPES[f.dtype], N, Tmax, Umax, V,
                                            ctx.labels.data_ptr(), int(ctx.blank), ctx.ws.data_ptr(), w.data_ptr(),
                                            grad_f.data_ptr(), grad_g.data_ptr(), _stream(dev))
        _check(rc, "ctct_simple_loss backward")
        ctx.f = ctx.g = ctx.ws = ctx.labels = None
        return (grad_f if ctx.needs_input_grad[0] else None, grad_g if ctx.needs_input_grad[1] else None) + (None,) * 6


def ctct_simple_loss(f_enc: torch.Tensor, g_pred: torch.Tensor, labels: torch.Tensor, frames_lengths: torch.Tensor,
                     labels_lengths: torch.Tensor, reduction: str = "mean", blank: int = 0) -> torch.Tensor:
    """The CTC-T loss of CAT's ``LogAdd`` joiner: ``ctct_loss`` over log_softmax(f_enc[n, t] + g_pred[n, u]), computed
    without the (N, Tmax, Umax+1, V) joint tensor.  Every convention is ``rnnt_loss_simple``'s: f_enc (N, Tmax, V) and
    g_pred (N, Umax+1, V) of one dtype on one CUDA device, labels (N, Umax), lengths and labels int32 or int64 on the CPU or
    the device, NaN cost and zero gradients for a bad utterance with device lengths; +inf cost and zero gradients for an
    infeasible one.  No host synchronisation; under ``torch.no_grad`` only the forward recursion runs."""
    shape = _simple.check_rnnt_simple_args(f_enc, g_pred, labels, frames_lengths, labels_lengths, reduction, blank,
                                           "ctct_simple_loss")
    if not f_enc.is_cuda or g_pred.device != f_enc.device:
        raise ValueError("ctct_simple_loss: f_enc and g_pred must be on one CUDA device")
    with torch.cuda.device(f_enc.device):
        if torch.is_grad_enabled() and (f_enc.requires_grad or g_pred.requires_grad):
            return _CTCTSimple.apply(f_enc, g_pred, labels, frames_lengths, labels_lengths, reduction, blank, shape)
        costs = _simple._forward(f_enc.detach().contiguous(), g_pred.detach().contiguous(), labels, frames_lengths,
                                 labels_lengths, blank, False, shape, "ctct")[0]
        return _reduce(costs, reduction)
