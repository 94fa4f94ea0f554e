"""Beam search for CAT's RNN-T transducers (``topo: rnnt``) on the GPU: the drop-in for ``cat/rnnt/rnnt_decoder.py``'s
``RNNTDecoder`` without an external LM, ILM estimation or ``<eos>`` early stop.  The networks run in torch, under the
caller's autocast; the search (exact top-B, prefix trie, fixed-order merge) is one native launch per frame
(``cat_b200/csrc/rnnt_decode.cu``).  Definition and differences from CAT: DESIGN.md §7 "Transducer beam search".
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from . import _lib
from ._C import _DTYPES, _check, _stream
from .rnnt import _on_device
from .rnnt_simple import _int32

MAX_BEAM = 128
_MODE_LOGPROBS, _MODE_LOGITS, _MODE_LOGADD = 0, 1, 2


def _check_args(enc_out, frame_lens, beam_size, nbest, blank, name) -> Tuple[int, int, int]:
    """The arguments of the search ``name`` (ValueError), checked before anything runs.  Returns (N, Tmax, nbest)."""
    if not isinstance(enc_out, torch.Tensor) or enc_out.dim() != 3 or not enc_out.is_cuda:
        raise ValueError(f"{name}: enc_out must be an (N, T, H) CUDA tensor")
    N, Tmax = int(enc_out.shape[0]), int(enc_out.shape[1])
    if N < 1:
        raise ValueError(f"{name}: enc_out holds no utterance")
    if isinstance(beam_size, bool) or not isinstance(beam_size, int) or not 1 <= beam_size <= MAX_BEAM:
        raise ValueError(f"{name}: beam_size must be an int in [1, {MAX_BEAM}], not {beam_size!r}")
    nbest = beam_size if nbest is None else nbest
    if isinstance(nbest, bool) or not isinstance(nbest, int) or not 1 <= nbest <= beam_size:
        raise ValueError(f"{name}: nbest must be an int in [1, beam_size = {beam_size}], not {nbest!r}")
    if isinstance(blank, bool) or not isinstance(blank, int) or blank < 0:
        raise ValueError(f"{name}: blank must be an int >= 0, not {blank!r}")
    if not isinstance(frame_lens, torch.Tensor) or frame_lens.dtype not in (torch.int32, torch.int64) \
            or tuple(frame_lens.shape) != (N,):
        raise ValueError(f"{name}: frame_lens must be an int32 or int64 (N,) tensor with N = {N}")
    if frame_lens.is_cuda:
        if frame_lens.device != enc_out.device:
            raise ValueError(f"{name}: frame_lens is on {frame_lens.device}, enc_out on {enc_out.device}")
    elif N and (int(frame_lens.min()) < 0 or int(frame_lens.max()) > Tmax):
        raise ValueError(f"{name}: frame_lens must lie in [0, T = {Tmax}]")
    return N, Tmax, nbest


def _check_state(predictor, state, R: int, name):
    """The predictor states the search can carry per slot: None, or a tuple of 3-D tensors with the batch on dim 1."""
    if state is None:
        return
    if isinstance(state, tuple) and all(isinstance(s, torch.Tensor) and s.dim() == 3 and s.shape[1] == R for s in state):
        return
    raise NotImplementedError(f"{name}: the state of predictor {type(predictor).__name__} is neither None nor a "
                              "tuple of 3-D tensors with the batch on dim 1 (an LSTM's); it cannot be carried per beam slot")


class _Joiner:
    """How the joiner's rows for a frame reach the kernel: LogAdd (f and g rows), JointNet in "add" mode (raw logits from
    fc(fc_enc(enc) + fc_dec(pn)), fc_enc applied once per call) or any other joiner (log-probs of joiner(enc, pn))."""

    def __init__(self, joiner, enc_out, caller):
        name = type(joiner).__name__
        self.joiner = joiner
        self.caller = caller
        if name == "LogAdd":
            self.mode = _MODE_LOGADD
            self.f = enc_out.contiguous()
        elif name == "JointNet" and getattr(joiner, "_mode", None) == "add":
            self.mode = _MODE_LOGITS
            self.fe = joiner.fc_enc(enc_out)
        else:
            self.mode = _MODE_LOGPROBS
            self.enc = enc_out

    def rows(self, t: int, pn_out: torch.Tensor, N: int, B: int) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """(rows (N*B, V) contiguous, f (N, Tmax, V) of the rows' dtype for LogAdd else None)"""
        R = N * B
        if self.mode == _MODE_LOGADD:
            g = pn_out.reshape(R, -1)
            if g.shape[1] != self.f.shape[2]:
                raise ValueError(f"{self.caller}: the LogAdd joiner's f (N, T, {self.f.shape[2]}) and g (R, "
                                 f"{g.shape[1]}) rows differ in V")
            dt = torch.promote_types(self.f.dtype, g.dtype)
            if self.f.dtype != dt:
                self.f = self.f.to(dt)
            return g.to(dt).contiguous(), self.f
        if self.mode == _MODE_LOGITS:
            h = self.fe[:, t, None, :] + self.joiner.fc_dec(pn_out).reshape(N, B, -1)
            return self.joiner.fc(h).reshape(R, -1).contiguous(), None
        enc = self.enc[:, t, None, None, :].expand(N, B, 1, -1).reshape(R, 1, -1)
        return self.joiner(enc, pn_out).reshape(R, -1).contiguous(), None


def _beam_search(name: str, family: str, enc_out, frame_lens, predictor, joiner, beam_size, nbest, blank):
    """The frame loop of the transducer searches: ``family`` "rnnt" or "ctct" picks the native ws-bytes, init and step entries
    (``ccb_<family>_beam_*``); both are finished by ``ccb_rnnt_beam_finish``.  ``name`` is the calling function's, for its
    errors.  Each frame runs the predictor once over all N*B slots, every slot keeping its parent's output and state or
    advancing them by the token it emitted; nothing synchronises the host."""
    N, Tmax, nbest = _check_args(enc_out, frame_lens, beam_size, nbest, blank, name)
    B, R = beam_size, N * beam_size
    dev = enc_out.device
    L = _lib.lib()

    def entry(e):   # the native entry, looked up where it is called: the argument checks run before any native access
        return getattr(L, f"ccb_{family}_beam_{e}")

    with torch.no_grad(), torch.cuda.device(dev):
        lens = _on_device(dev, _int32(frame_lens))[0]
        if Tmax:
            pn_out, state = predictor(torch.full((R, 1), blank, dtype=torch.long, device=dev), None)
            _check_state(predictor, state, R, name)
            join = _Joiner(joiner, enc_out, name)
        parent = torch.empty((N, B), dtype=torch.int32, device=dev)
        token = torch.empty((N, B), dtype=torch.int32, device=dev)
        node = torch.empty((N, B), dtype=torch.int32, device=dev)
        score = torch.empty((N, B), dtype=torch.float64, device=dev)
        tokens = torch.empty((N, nbest, Tmax), dtype=torch.int32, device=dev)
        lengths = torch.empty((N, nbest), dtype=torch.int32, device=dev)
        scores = torch.empty((N, nbest), dtype=torch.float32, device=dev)
        slot_base = (torch.arange(N, device=dev, dtype=torch.long) * B)[:, None]
        ws = None

        def init():   # (after the first frame's rows: every argument error is raised before a native call)
            nonlocal ws
            ws = torch.empty(int(entry("ws_bytes")(N, Tmax, B)), dtype=torch.uint8, device=dev)
            _check(entry("init")(N, Tmax, B, ws.data_ptr(), parent.data_ptr(), token.data_ptr(), node.data_ptr(),
                                 score.data_ptr(), _stream(dev)), name)

        if Tmax == 0:
            init()
        for t in range(Tmax):
            rows, f = join.rows(t, pn_out, N, B)
            if rows.dtype not in _DTYPES:
                rows = rows.float()
                f = f.float() if f is not None else None
            V = int(rows.shape[1])
            if blank >= V:
                raise ValueError(f"{name}: blank = {blank} is not a label of the joiner's V = {V}")
            if t == 0:
                init()
            _check(entry("step")(rows.data_ptr(), f.data_ptr() if f is not None else None, _DTYPES[rows.dtype], join.mode,
                                 N, Tmax, B, V, t, lens.data_ptr(), blank, ws.data_ptr(), parent.data_ptr(),
                                 token.data_ptr(), node.data_ptr(), score.data_ptr(), _stream(dev)), name)
            if t + 1 == Tmax:
                break
            # each slot's predictor output and state: its parent's, advanced by the token it emitted (if any)
            src = (slot_base + parent.long()).reshape(R)
            tok = token.reshape(R)
            ext = tok >= 0
            pn_par = pn_out.index_select(0, src)
            st_par = None if state is None else tuple(s.index_select(1, src) for s in state)
            out_new, st_new = predictor(torch.where(ext, tok, blank).long().reshape(R, 1), st_par)
            _check_state(predictor, st_new, R, name)
            pn_out = torch.where(ext.view(R, *([1] * (out_new.dim() - 1))), out_new, pn_par.to(out_new.dtype))
            state = None if st_new is None else tuple(
                torch.where(ext.view(1, R, 1), sn, sp.to(sn.dtype)) for sn, sp in zip(st_new, st_par))
        _check(L.ccb_rnnt_beam_finish(N, Tmax, B, nbest, ws.data_ptr(), node.data_ptr(), score.data_ptr(),
                                      tokens.data_ptr(), lengths.data_ptr(), scores.data_ptr(), _stream(dev)), name)
        lens.record_stream(torch.cuda.current_stream(dev))
    return tokens, lengths, scores


def rnnt_beam_search(enc_out: torch.Tensor, frame_lens: torch.Tensor, predictor, joiner, beam_size: int = 5,
                     nbest: Optional[int] = None, blank: int = 0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The nbest (default beam_size) best label sequences of every utterance by CAT's RNA beam search (DESIGN.md §7
    "Transducer beam search"), blank = bos = ``blank``.

    enc_out (N, T, H) on a CUDA device; frame_lens (N,) int32 or int64 on the CPU or that device (T_n in [0, T]; an
    utterance with T_n = 0 gets the empty hypothesis, score 0).  ``predictor(tokens (R, 1), state)`` returns (out (R, 1, H'),
    state) with a state that is None or a tuple of 3-D tensors with the batch on dim 1; ``joiner`` is CAT's LogAdd, a
    JointNet or any module called as joiner(enc (R, 1, H), pn (R, 1, H')) returning log-probs.  Returns device tensors
    tokens (N, nbest, T) int32 -1 padded, lengths (N, nbest) int32 (-1 past the hypotheses found) and scores (N, nbest)
    fp32, best first.  The frame loop runs to T; nothing synchronises the host."""
    return _beam_search("rnnt_beam_search", "rnnt", enc_out, frame_lens, predictor, joiner, beam_size, nbest, blank)


class RNNTDecoder:
    """CAT's ``cat.rnnt.rnnt_decoder.RNNTDecoder`` with its constructor, decoding on the GPU through ``rnnt_beam_search``.
    Not supported (NotImplementedError): an LM with alpha != 0, ILM estimation with ilm_weight != 0, an ``<eos>`` early stop
    and bos_id != blank_id.  alpha == 0 drops the LM, as in CAT."""

    def __init__(self, predictor, joiner, blank_id: int = 0, bos_id: int = 0, eos_id: int = -1, beam_size: int = 5,
                 nbest: int = -1, lm_module=None, alpha: float = 0.0, beta: float = 0.0, est_ilm: bool = False,
                 ilm_weight: float = 0.0):
        if bos_id != blank_id:
            raise NotImplementedError(f"RNNTDecoder: bos_id ({bos_id}) must equal blank_id ({blank_id}), as in CAT")
        if alpha == 0.0:
            lm_module = None
        if lm_module is not None:
            raise NotImplementedError("RNNTDecoder: external LM fusion (lm_module with alpha != 0) is not supported")
        if est_ilm and ilm_weight != 0.0:
            raise NotImplementedError("RNNTDecoder: ILM estimation (est_ilm with ilm_weight != 0) is not supported")
        if eos_id not in (-1, blank_id):
            raise NotImplementedError(f"RNNTDecoder: the <eos> early stop (eos_id = {eos_id}) is not supported")
        if isinstance(beam_size, bool) or not isinstance(beam_size, int) or not 1 <= beam_size <= MAX_BEAM:
            raise ValueError(f"RNNTDecoder: beam_size must be an int in [1, {MAX_BEAM}], not {beam_size!r}")
        if nbest == -1:
            nbest = beam_size
        if isinstance(nbest, bool) or not isinstance(nbest, int) or nbest < 1:
            raise ValueError(f"RNNTDecoder: nbest must be -1 or a positive int, not {nbest!r}")
        self.predictor = predictor
        self.joiner = joiner
        self.blank_id = blank_id
        self.bos_id = bos_id
        self.eos_id = -1
        self.beam_size = beam_size
        self.nbest = min(nbest, beam_size)

    def __call__(self, enc_out: torch.Tensor, frame_lens: Optional[torch.Tensor] = None
                 ) -> List[Tuple[List[List[int]], List[float]]]:
        """[(token lists without bos, scores), ...] per utterance, best first: CAT's return value.  One host copy."""
        return _to_lists(*rnnt_beam_search(enc_out, _frame_lens(enc_out, frame_lens), self.predictor, self.joiner,
                                           self.beam_size, self.nbest, self.blank_id))


def _frame_lens(enc_out, frame_lens):
    """CAT's default: every utterance runs to T."""
    if frame_lens is None:
        return torch.full((enc_out.size(0),), enc_out.size(1), dtype=torch.int32)
    return frame_lens


def _to_lists(tokens, lengths, scores) -> List[Tuple[List[List[int]], List[float]]]:
    """[(token lists, scores), ...] per utterance from a search's device tensors, as CAT's decoders return them.  One host
    copy."""
    N, K, T = tokens.shape
    host = torch.cat([tokens.reshape(N, K * T), lengths, scores.view(torch.int32)], dim=1).cpu()
    out = []
    for n in range(N):
        toks = host[n, :K * T].view(K, T)
        lens = host[n, K * T:K * T + K].tolist()
        sc = host[n, K * T + K:].contiguous().view(torch.float32).tolist()
        hyps = [(toks[k, :lens[k]].tolist(), sc[k]) for k in range(K) if lens[k] >= 0]
        out.append(([h for h, _ in hyps], [s for _, s in hyps]))
    return out
