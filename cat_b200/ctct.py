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

from .rnnt import _costs_both_ways, _loss
from .rnnt_simple import _simple_loss


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
    return _loss("ctct", "ctct_loss", log_probs, labels, frames_lengths, labels_lengths, reduction, blank,
                 _layout(log_probs, compact), from_logits)


def ctct_costs_both_ways(log_probs, labels, frames_lengths, labels_lengths, blank=0, compact=None, from_logits=False):
    """The (N,) costs from alpha and from beta, which agree up to rounding (a check of the two recursions)."""
    return _costs_both_ways("ctct", "ctct_loss", log_probs, labels, frames_lengths, labels_lengths, blank,
                            _layout(log_probs, compact), from_logits)


def ctct_simple_loss(f_enc: torch.Tensor, g_pred: torch.Tensor, labels: torch.Tensor, frames_lengths: torch.Tensor,
                     labels_lengths: torch.Tensor, reduction: str = "mean", blank: int = 0) -> torch.Tensor:
    """The CTC-T loss of CAT's ``LogAdd`` joiner: ``ctct_loss`` over log_softmax(f_enc[n, t] + g_pred[n, u]), computed
    without the (N, Tmax, Umax+1, V) joint tensor.  Every convention is ``rnnt_loss_simple``'s: f_enc (N, Tmax, V) and
    g_pred (N, Umax+1, V) of one dtype on one CUDA device, labels (N, Umax), lengths and labels int32 or int64 on the CPU or
    the device, NaN cost and zero gradients for a bad utterance with device lengths; +inf cost and zero gradients for an
    infeasible one.  No host synchronisation; under ``torch.no_grad`` only the forward recursion runs."""
    return _simple_loss("ctct", "ctct_simple_loss", f_enc, g_pred, labels, frames_lengths, labels_lengths, reduction, blank)
