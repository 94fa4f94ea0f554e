"""Python surface of the CTC-CRF loss -- drop-in for the reference's ``ctc_crf`` package
(src/ctc_crf/ctc_crf/__init__.py:25-171): same class names, constructor arguments, argument placement
(logits on the GPU, labels / lx / ly int32 on the CPU), dtype asserts and error behaviour.

What changed underneath (SURVEY.md 8a row a1): the reference's forward makes ~11 passes over (N,T,V)
(transpose copy, two zero fills, combine, scale, backward multiply) and synchronises the host three times;
here ``_CTC_CRF.forward`` is ONE native call that writes the final gradient once and never synchronises.
"""
from __future__ import annotations

import os
from typing import List, Optional, Union

import torch
from torch.autograd import Function
from torch.nn import Module

from . import _C as core

__version__ = "0.1.0"


def _assert_no_grad(tensor):
    assert not tensor.requires_grad, "shouldn't require grads"


class _WARP_CTC_GPU(Function):
    """__init__.py:25-56: CTC loss on log-softmax inputs.  Same arguments, result and gradient as the reference's
    Function; underneath it is ONE native call on the (N,T,V) tensor in place -- no (T,N,V) transpose copy (:31), no
    zero-filled gradient (:32), no host round trip for the per-utterance costs (:33-35) -- see ``_C.ctc_loss_fwd``.
    (``_C.gpu_ctc`` keeps the reference's pybind signature for callers that use it directly.)
    reduction and zero_infinity (additions, after the reference's arguments) as for ``_CTC_CRF``, cost[n] = -log p[n]."""

    @staticmethod
    def forward(ctx, logits, labels, input_lengths, label_lengths, size_average=True, reduction=None, zero_infinity=False):
        logits = logits.contiguous()
        out, grads, _ = core.ctc_loss_fwd(logits, labels, input_lengths, label_lengths, size_average,
                                          **_loss_options(reduction, zero_infinity))
        ctx.grads, ctx.lx, ctx.in_dtype, ctx.reduction = grads, input_lengths, logits.dtype, reduction
        return out

    @staticmethod
    def backward(ctx, grad_output):
        return (_loss_backward(ctx, grad_output),) + (None,) * 6


class _CTC_CRF(Function):
    """__init__.py:58-94.  loss = sum_n [logZ_den(n) - (1+lamb) log p_ctc(n)] (/N),
    grad = [gamma_den - (1+lamb) gamma_ctc] (/N); backward = grads * grad_output.
    Additions, after the reference's arguments: ``reduction='none'`` returns the (N,) costs
    cost[n] = logZ_den[n] - (1+lamb) log p_ctc[n], with the gradient kept unscaled, G[n] = d cost[n] / d logits[n], so that the
    backward is one pass that writes grad_output[n] * G[n] in the logits' dtype (``_C.grad_rows_scale``); ``zero_infinity``
    as for ``CTC_CRF_LOSS``; ``from_logits=True`` is the loss of ``_CTC_CRF_LOGITS``."""

    @staticmethod
    def forward(ctx, logits, labels, input_lengths, label_lengths, lamb=0.1, size_average=True, reduction=None,
                zero_infinity=False, from_logits=False):
        logits = logits.contiguous()
        opts = _loss_options(reduction, zero_infinity)
        if from_logits:
            opts["from_logits"] = True
        out, grads, _ = core.ctc_crf_loss_fwd(logits, labels, input_lengths, label_lengths, lamb, size_average, **opts)
        ctx.grads, ctx.lx, ctx.in_dtype, ctx.reduction = grads, input_lengths, logits.dtype, reduction
        return out

    @staticmethod
    def backward(ctx, grad_output):
        return (_loss_backward(ctx, grad_output),) + (None,) * 8


class _CTC_CRF_LOGITS(_CTC_CRF):
    """SURVEY 8f-1: the same loss taken on the RAW encoder outputs.  Replaces, in one native call,
    ``logits = net_out.float().log_softmax(-1); loss = _CTC_CRF(logits, ...)`` and the autograd backward of the cast
    and of log_softmax (cat/ctc/train.py:173-174,184-190): no normalised fp32 copy is materialised and the gradient
    comes back already chained through the softmax Jacobian, in the dtype of the input."""

    @staticmethod
    def forward(ctx, logits, labels, input_lengths, label_lengths, lamb=0.1, size_average=True, reduction=None,
                zero_infinity=False):
        return _CTC_CRF.forward(ctx, logits, labels, input_lengths, label_lengths, lamb, size_average, reduction,
                                zero_infinity, True)


def _loss_backward(ctx, grad_output):
    if ctx.reduction == "none":     # grad_logits[n] = grad_output[n] * G[n], in one pass, in the logits' dtype
        return core.grad_rows_scale(ctx.grads, grad_output, ctx.lx, ctx.in_dtype)
    return (ctx.grads * grad_output.to(ctx.grads.device)).to(ctx.in_dtype)


class _CTC_CRF_SEQS(Function):
    """CTC_CRF_LOSS with several label sequences per utterance (``utt``): cost[m] = logZ_den[utt[m]] - (1+lamb) log p_ctc[m],
    one den pass per utterance.  reduction None: the forward writes the final gradient; 'none': the forward keeps the den
    occupancies unscaled and the numerator's cells, and the backward weights them by grad_output (``_C.seqs_backward``)."""

    @staticmethod
    def forward(ctx, logits, labels, lx, ly, utt, lamb, size_average, from_logits, reduction, zero_infinity):
        logits = logits.contiguous()
        out, grads, state = core.ctc_crf_loss_seqs(logits, labels, lx, ly, utt, lamb, size_average, from_logits=from_logits,
                                                   reduction=reduction, zero_infinity=zero_infinity)
        ctx.grads, ctx.state, ctx.in_dtype = grads, state, logits.dtype
        return out

    @staticmethod
    def backward(ctx, grad_output):
        return (_seqs_backward(ctx, grad_output),) + (None,) * 9


class _WARP_CTC_SEQS(Function):
    """WARP_CTC_LOSS with several label sequences per utterance (``utt``): cost[m] = -log p[m], every numerator in one
    launch; backward as in ``_CTC_CRF_SEQS``."""

    @staticmethod
    def forward(ctx, logits, labels, lx, ly, utt, size_average, reduction, zero_infinity):
        logits = logits.contiguous()
        out, grads, state = core.ctc_loss_seqs(logits, labels, lx, ly, utt, size_average, reduction=reduction,
                                               zero_infinity=zero_infinity)
        ctx.grads, ctx.state, ctx.in_dtype = grads, state, logits.dtype
        return out

    @staticmethod
    def backward(ctx, grad_output):
        return (_seqs_backward(ctx, grad_output),) + (None,) * 7


def _seqs_backward(ctx, grad_output):
    if ctx.state is not None:       # reduction 'none': sum_m grad_output[m] * d cost[m] / d logits, in the logits' dtype
        return core.seqs_backward(ctx.state, grad_output, ctx.in_dtype)
    return (ctx.grads * grad_output.to(ctx.grads.device)).to(ctx.in_dtype)


def _check_utt(utt):
    """`utt` is placed and asserted as lx / ly are; `_C.group_seqs` checks its values."""
    assert utt.dtype == torch.int, f"expect utt to be torch.int object, instead: {utt.dtype}"
    _assert_no_grad(utt)


def _check_loss_args(logits, labels, lx, ly, utt, dtypes=True):
    """The reference's argument asserts (ctc_crf/__init__.py:115-124): flat labels, with `dtypes` the logits and int32
    labels and lengths (WARP_CTC_LOSS asserts no dtypes, as the reference's does not), and no gradient on any of them."""
    assert len(labels.size()) == 1
    if dtypes:
        assert logits.dtype in (torch.float, torch.bfloat16, torch.float16), \
            f"expect logits to be torch.float (or torch.bfloat16 / torch.float16) object, instead: {logits.dtype}"
        assert labels.dtype == torch.int, f"expect labels to be torch.int object, instead: {labels.dtype}"
        assert lx.dtype == torch.int, f"expect lx to be torch.int object, instead: {lx.dtype}"
        assert ly.dtype == torch.int, f"expect ly to be torch.int object, instead: {ly.dtype}"
    if utt is not None:
        _check_utt(utt)
    _assert_no_grad(labels)
    _assert_no_grad(lx)
    _assert_no_grad(ly)


def _loss_options(reduction, zero_infinity) -> dict:
    """The keyword arguments the `_C` loss functions get for these settings: none at the defaults, so that the default
    path calls exactly what it called before the two options existed."""
    core.check_reduction(reduction)
    if reduction is None and not zero_infinity:
        return {}
    return dict(reduction=reduction, zero_infinity=bool(zero_infinity))


class CTC_CRF_LOSS(Module):
    def __init__(self, lamb: float = 0.1, size_average: bool = True, from_logits: bool = False,
                 reduction: Optional[str] = None, zero_infinity: bool = False):
        """
        lamb (float): weight for auxiliary CTC loss, final loss = lamb * loss_ctc + loss_crf
        size_average (bool): whether to do average over batch size dimension.
        from_logits (bool): addition to the reference signature -- ``forward`` takes the raw encoder outputs and
            applies log_softmax (and its backward) inside the fused call.  Default False = reference behaviour.
        reduction (None or 'none'): addition -- None returns the scalar of the reference (the batch sum, or the mean
            over the batch with size_average); 'none' returns the (N,) fp32 costs logZ_den[n] - (1+lamb) log p_ctc[n], to be
            weighted, masked or normalised by the caller.  Any other value raises ValueError.
        zero_infinity (bool): addition -- an utterance whose cost is not finite (an infeasible label sequence, an utterance
            that cannot reach a final state of the den graph) gets cost 0 and a zero gradient instead of making the batch
            loss inf or NaN.  With size_average the divisor stays N.
        """
        super(CTC_CRF_LOSS, self).__init__()
        _loss_options(reduction, zero_infinity)      # an unknown reduction fails here, at construction
        self.ctc_crf = _CTC_CRF_LOGITS.apply if from_logits else _CTC_CRF.apply
        self.lamb = lamb
        self.size_average = size_average
        self.from_logits = from_logits
        self.reduction = reduction
        self.zero_infinity = zero_infinity

    def forward(self, logits, labels, lx, ly, utt=None) -> torch.FloatTensor:
        """
        logits (torch.FloatTensor): size (N, T, V), log-probabilities, on GPU device.
            (torch.bfloat16 and torch.float16 are accepted too, read in place with fp32 arithmetic -- the reference asserts
            fp32.  With from_logits=True this takes the fp16 output of an fp16 autocast encoder as is.)
        labels (torch.IntTensor)  : size (sum {Ui}, ) flattened without paddings, on CPU.
        lx (torch.IntTensor) : size (N, ), on CPU
        ly (torch.IntTensor) : size (N, ), on CPU
        utt (torch.IntTensor, optional): addition -- size (M, ), on CPU: several label sequences per utterance (samples,
            N-best lists, alternative pronunciations).  labels / ly then describe M sequences, sequence m scored against
            logits row utt[m] (any order); lx stays (N, ).  cost[m] = logZ_den[utt[m]] - (1+lamb) log p_ctc(l_m | x_utt[m]),
            with the den computed once per utterance.  The scalar is the sum over the M sequences (/ M with size_average);
            reduction='none' returns the (M,) costs in the caller's order; zero_infinity masks per sequence.  An utterance
            without a sequence contributes nothing and gets a zero gradient.
        """
        _check_loss_args(logits, labels, lx, ly, utt)
        if utt is not None:
            return self._forward_seqs(logits, labels, lx, ly, utt)
        opts = _loss_options(self.reduction, self.zero_infinity)    # read on every call: the attributes may be reassigned
        if not torch.is_grad_enabled():
            # evaluation (torch.no_grad / inference_mode): the loss alone, with the den alpha on a ring of frames and no
            # gradient.  Keyed on grad mode, not on logits.requires_grad: with grad mode on the gradient is always computed.
            return core.ctc_crf_loss_fwd_only(logits.contiguous(), labels, lx, ly, self.lamb, self.size_average,
                                              from_logits=self.from_logits, **opts)[0]
        if opts:
            return _CTC_CRF.apply(logits, labels, lx, ly, self.lamb, self.size_average, self.reduction,
                                  bool(self.zero_infinity), self.from_logits)
        return self.ctc_crf(logits, labels, lx, ly, self.lamb, self.size_average)

    def _forward_seqs(self, logits, labels, lx, ly, utt):
        core.check_reduction(self.reduction)
        if not torch.is_grad_enabled():
            return core.ctc_crf_loss_seqs_fwd_only(logits.contiguous(), labels, lx, ly, utt, self.lamb, self.size_average,
                                                   from_logits=self.from_logits, reduction=self.reduction,
                                                   zero_infinity=bool(self.zero_infinity))
        return _CTC_CRF_SEQS.apply(logits, labels, lx, ly, utt, self.lamb, self.size_average, self.from_logits,
                                   self.reduction, bool(self.zero_infinity))


class WARP_CTC_LOSS(Module):
    """__init__.py:128-144.  reduction and zero_infinity (additions) as for CTC_CRF_LOSS, with cost[n] = -log p[n]."""

    def __init__(self, size_average=True, reduction: Optional[str] = None, zero_infinity: bool = False):
        super(WARP_CTC_LOSS, self).__init__()
        _loss_options(reduction, zero_infinity)      # an unknown reduction fails here, at construction
        self.ctc = _WARP_CTC_GPU.apply
        self.size_average = size_average
        self.reduction = reduction
        self.zero_infinity = zero_infinity

    def forward(self, logits, labels, input_lengths, label_lengths, utt=None):
        """utt (addition): (M,) int32 on CPU, sequence m of labels / label_lengths scored against logits row utt[m], as for
        CTC_CRF_LOSS; cost[m] = -log p[m], all M numerators in one launch."""
        _check_loss_args(logits, labels, input_lengths, label_lengths, utt, dtypes=False)
        if utt is not None:
            core.check_reduction(self.reduction)
            if not torch.is_grad_enabled():
                return core.ctc_loss_seqs(logits.contiguous(), labels, input_lengths, label_lengths, utt, self.size_average,
                                          reduction=self.reduction, zero_infinity=bool(self.zero_infinity),
                                          with_grad=False)[0]
            return _WARP_CTC_SEQS.apply(logits, labels, input_lengths, label_lengths, utt, self.size_average, self.reduction,
                                        bool(self.zero_infinity))
        opts = _loss_options(self.reduction, self.zero_infinity)
        if not torch.is_grad_enabled():   # evaluation: the loss alone (see CTC_CRF_LOSS.forward)
            return core.ctc_loss_fwd_only(logits.contiguous(), labels, input_lengths, label_lengths, self.size_average,
                                          **opts)[0]
        return self.ctc(logits, labels, input_lengths, label_lengths, self.size_average, self.reduction,
                        bool(self.zero_infinity))


def ctc_align(logits, labels, input_lengths, label_lengths, utt=None):
    """Best-path forced alignment of every utterance to its label sequence over the CTC lattice -- the alignment that comes
    with the numerator (SURVEY 8f-4; cat/ctc/train_jsa.py consumes frame-level paths).  Arguments as for WARP_CTC_LOSS.
    Returns (align (N,T) int32 on the GPU, token per frame incl. blank 0, -1 past each length; score (N,) fp32).
    utt (addition, (M,) int32 CPU): align each of M label sequences to its logits row utt[m]; align (M,T), score (M,)."""
    assert len(labels.size()) == 1
    if utt is not None:
        _check_utt(utt)
        return core.ctc_align_seqs(logits.contiguous(), labels, input_lengths, label_lengths, utt)
    return core.ctc_align(logits.contiguous(), labels, input_lengths, label_lengths)


def crf_sample(logits, lx, num_samples=1, generator=None):
    """Draw label sequences from the CTC-CRF posterior of the den graph loaded by ``CRFContext``, exactly: forward filtering
    (the den forward pass) and backward sampling, for sampling-based objectives (JSA, minimum-risk training with sampled
    hypotheses, REINFORCE-style estimators).  A path is drawn with probability w(path) prod_t exp(y[t][label]) final / Z, so
    for a T-compose-LM den graph the label sequence follows p_LM(l) p_ctc(l|x) / Z, the sequence posterior the loss
    normalises by.  A per-frame multinomial on the softmax is exact only for a CTC model.

    logits (N,T,V) fp32, bf16 or fp16 on the GPU: log-probs or raw logits, which give the same distribution (every path
    emits one label per frame, so the log-softmax shift cancels); frames t >= lx[n] are never read.  lx (N,) int32 on the CPU.
    num_samples K >= 1.  generator: a CPU torch.Generator (default: torch's), from which ONE 64-bit seed is drawn per call;
    ``torch.manual_seed`` reproduces a call and successive calls differ.  The samples of an utterance depend on the seed, its
    index in the batch and its own inputs only.

    Returns device tensors, without synchronising the host and without recording autograd:
      tokens (N,K,T) int32: the CTC collapse of each path (repeats merged, blank 0 dropped), padded with -1;
      lengths (N,K) int32: tokens per sample;
      align (N,K,T) int32: the label of every frame t < lx[n] (blank included), -1 beyond, as ``ctc_align``;
      path_logp (N,K) fp32: log p(path | x), accumulated in fp64.
    An utterance with no path of finite score (lx = 0, -inf frames, no reachable final state) gets lengths -1, rows of -1
    and path_logp -inf.  ``samples_to_labels`` turns the result into the ``utt=`` arguments of ``CTC_CRF_LOSS``."""
    return core.crf_sample(logits, lx, num_samples, generator)


def samples_to_labels(tokens, lengths):
    """(labels, ly, utt) CPU int32 tensors for ``CTC_CRF_LOSS(...)(logits, labels, lx, ly, utt=utt)`` from the
    ``crf_sample`` outputs: every feasible sample (lengths >= 0), utterance by utterance, samples in order; infeasible samples
    are dropped.  It performs ONE device-to-host copy, which waits for the sampler."""
    return core.samples_to_labels(tokens, lengths)


def ctc_beam_search(logits, lx, beam_size=16, cutoff_top_n=40, crf=False, lm=None, alpha=1.0, beta=0.0):
    """N-best label sequences by CTC prefix beam search on the GPU (DESIGN.md §7 "Prefix beam search").

    crf False: plain CTC, as ``ctcdecode`` computes it without a word LM -- a hypothesis collects the paths whose CTC
    collapse it is, each path scored sum_t y[t][label].  crf True: the paths run over the den graph loaded by ``CRFContext``
    and carry its arc and final weights, so for a T-compose-LM graph a sequence's total is log p_LM(l) + log p_ctc(l|x),
    the CTC-CRF posterior up to log Z.  The graph must be CTC-shaped (both slots of a prefix step into one state on a token;
    checked at the first crf call per graph and device, RuntimeError naming the states otherwise).

    logits (N,T,V) fp32, bf16 or fp16 on the GPU, log-probs or raw logits: every path has lx[n] frames, so raw logits give the
    same hypotheses, each score shifted by sum_t logsumexp(logits[n,t]).  Frames t >= lx[n] are never read.  lx (N,) int32
    on the CPU.  beam_size B in 1..128; cutoff_top_n in 1..V: a frame extends hypotheses by its cutoff_top_n most likely
    tokens (ties: lower id), plus blank and each hypothesis's own last token.

    Returns device tensors, best first, without synchronising the host and without recording autograd:
      tokens (N,B,T) int32, padded with -1; lengths (N,B) int32;
      timesteps (N,B,T) int32: the frame at which each token's prefix first entered the beam, -1 padded;
      scores (N,B) fp32: the log-sum of the kept paths (fp64 inside), a lower bound on the sequence's log mass, exact when
      nothing was pruned.
    Rows past the hypotheses of finite score have length -1, tokens -1 and score -inf; lx = 0 gives the empty sequence.
    ``samples_to_labels(tokens, lengths)`` turns the lists into the ``utt=`` arguments of the losses.

    lm: an ``NGramLM`` (a token n-gram LM read from ARPA text) fused into the plain search (DESIGN.md §7 "N-gram LM
    fusion").  A hypothesis l_1..l_k then scores  A + alpha sum_{i=1..k+1} ln P(w_i | history) + beta k,  A the score above,
    w_i the LM word of token l_i and w_{k+1} = </s>; an extension adds its term to the candidate's rank during the search,
    and the </s> term is added after the last frame, where the hypotheses are re-ranked.  alpha = 0 does not consult the
    LM.  alpha must be finite and >= 0, beta finite, ``len(labels)`` of the LM equal to V, and crf False (ValueError)."""
    return core.ctc_beam_search(logits, lx, beam_size, cutoff_top_n, crf, lm, alpha, beta)


class CTCBeamDecoder:
    """Drop-in for ``ctcdecode.CTCBeamDecoder`` on the GPU (``ctc_beam_search``, plain CTC).  ``decode(probs, seq_lens)``
    returns (beam_results (N,B,T), beam_scores (N,B) = -log score, timesteps (N,B,T), out_lens (N,B)) as ``ctcdecode`` does,
    on the device of the input (CPU inputs run on the current CUDA device).
    model_path: a token-level n-gram LM in ARPA text (``is_token_based=True``, as CAT's ``decode.py`` passes it), loaded as
    ``NGramLM(model_path, labels)`` and fused in with ``alpha`` and ``beta``; without it alpha and beta are unused.  Word-level
    LMs (``is_token_based=False``), KenLM binaries and a missing file raise NotImplementedError, a malformed ARPA file
    RuntimeError.  blank_id != 0 and cutoff_prob != 1.0 are not supported (NotImplementedError); num_processes is accepted
    and unused."""

    def __init__(self, labels, model_path=None, alpha=0, beta=0, cutoff_top_n=40, cutoff_prob=1.0, beam_width=100,
                 num_processes=4, blank_id=0, log_probs_input=False, is_token_based=False):
        if blank_id != 0:
            raise NotImplementedError("CTCBeamDecoder: the blank must be label 0")
        if cutoff_prob != 1.0:
            raise NotImplementedError("CTCBeamDecoder: cutoff_prob must be 1.0 (use cutoff_top_n)")
        self._labels = list(labels)
        self._cutoff_top_n = min(int(cutoff_top_n), len(self._labels))
        self._beam_width = int(beam_width)
        self._log_probs_input = bool(log_probs_input)
        self._lm, self._alpha, self._beta = None, float(alpha), float(beta)
        if model_path is not None:
            if not is_token_based:
                raise NotImplementedError("CTCBeamDecoder: word-level LMs scored on spaces are not supported; pass "
                                          "is_token_based=True with a token n-gram LM")
            if not _is_arpa_text(model_path):
                raise NotImplementedError(f"CTCBeamDecoder: only ARPA text LMs are supported (`ngram.sh --arpa`), and "
                                          f"{model_path!r} is missing or is not ARPA text (a KenLM binary?)")
            from .ngram import NGramLM
            self._lm = NGramLM(model_path, self._labels)

    def decode(self, probs, seq_lens=None):
        """probs (N,T,V): probabilities, or log-probabilities with log_probs_input=True.  seq_lens (N,): frames per utterance
        (default: all T)."""
        x = probs if probs.is_cuda else probs.to(torch.device("cuda", torch.cuda.current_device()))
        if not self._log_probs_input:
            x = x.float().log()
        N, T, _ = x.shape
        lx = torch.full((N,), T, dtype=torch.int32) if seq_lens is None else torch.as_tensor(seq_lens).to("cpu", torch.int32)
        tokens, lengths, timesteps, scores = core.ctc_beam_search(x, lx, self._beam_width,
                                                                  min(self._cutoff_top_n, int(x.shape[2])), False,
                                                                  self._lm, self._alpha, self._beta)
        return tokens, -scores, timesteps, lengths


def _is_arpa_text(path) -> bool:
    """False for a missing file, a KenLM binary, a gzip file or one with NUL bytes near its start: files the ARPA loader
    does not read.  Anything else goes to the loader, which names the line of what it cannot parse."""
    if not os.path.isfile(path):
        return False
    with open(path, "rb") as f:
        head = f.read(4096)
    return not (head.startswith(b"mmap lm ") or head.startswith(b"\x1f\x8b") or b"\0" in head)


class CRFContext:
    def __init__(self, den_lm: str, gpus: Union[int, List[int]]) -> None:
        """
        den_lm (str): path to the denominator LM (OpenFst binary, see cat/utils/tool/prep_den_lm.sh)
        gpus   (int, List[int]): Specify which GPU to be used.
        """
        if not os.path.isfile(den_lm):
            raise RuntimeError(f"Denominator LM model location is invalid: {den_lm}.")
        if isinstance(gpus, int):
            gpus = [gpus]
        nprocs = torch.cuda.device_count()
        if not all([i >= 0 and i < nprocs for i in gpus]):
            raise RuntimeError(f"Available GPU={nprocs}, invalid GPU ids: {gpus}.")
        gpu_t = torch.IntTensor(gpus)
        core.init_env(den_lm, gpu_t)
        self._gpus = gpu_t

    def __del__(self):
        if hasattr(self, '_gpus'):
            try:
                core.release_env(self._gpus)
            except Exception:      # interpreter shutdown: module globals may already be gone
                pass
            del self._gpus
