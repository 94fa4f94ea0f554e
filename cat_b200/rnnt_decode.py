"""Beam search for CAT's RNN-T transducers (``topo: rnnt``) on the GPU: the drop-in for ``cat/rnnt/rnnt_decoder.py``'s
``RNNTDecoder``, with CAT's external LM fusion (``alpha``, ``beta``) and ILM estimation (``ilm_weight``), without the
``<eos>`` early stop.  The networks run in torch, under the caller's autocast; the search (exact top-B, prefix trie,
fixed-order merge, the fusion terms) is one native launch per frame (``cat_b200/csrc/rnnt_decode.cu``), and an n-gram LM's
rows, or the rows of a weighted LM mix (``MultiLM``, CAT's ``MultiDecoder``, as LODR decoding uses), are one more.
Definition and differences from CAT: DESIGN.md §7 "Transducer beam search", "RNN-T beam search with LM fusion" and
"RNN-T beam search with an LM mix".
"""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Optional, Tuple

import torch

from . import _lib
from ._C import _DTYPES, _check, _stream
from .ngram import NGramLM
from .rnnt import _int32, _on_device

MAX_BEAM = 128
MAX_MIX = 8                  # members of a MultiLM (rnnt_decode.cu kLmMixMax)
_MIX_SMEM = 200 * 1024       # the mix rows kernel's shared memory: 8 (largest n-gram word count + V) bytes at most
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


def _check_state(predictor, state, R: int, name, what="predictor"):
    """The predictor (or LM) states the search can carry per slot: None, or a tuple of 3-D tensors with the batch on dim 1."""
    if state is None:
        return
    if isinstance(state, tuple) and all(isinstance(s, torch.Tensor) and s.dim() == 3 and s.shape[1] == R for s in state):
        return
    raise NotImplementedError(f"{name}: the state of {what} {type(predictor).__name__} is neither None nor a "
                              "tuple of 3-D tensors with the batch on dim 1 (an LSTM's); it cannot be carried per beam slot")


def _carry(step, out, state, src, tok, ext, blank: int, check):
    """Each slot's network output and state after a frame: its parent's (rows ``src`` of ``out`` and of dim 1 of ``state``),
    advanced by ``step(tokens (R, 1), state)`` where the slot emitted a token (``ext``).  The predictor and a neural LM are
    carried alike; ``check`` validates the new state."""
    R = src.shape[0]
    out_par = out.index_select(0, src)
    st_par = None if state is None else tuple(s.index_select(1, src) for s in state)
    out_new, st_new = step(torch.where(ext, tok, blank).long().reshape(R, 1), st_par)
    check(st_new)
    out = torch.where(ext.view(R, *([1] * (out_new.dim() - 1))), out_new, out_par.to(out_new.dtype))
    state = None if st_new is None else tuple(
        torch.where(ext.view(1, R, 1), sn, sp.to(sn.dtype)) for sn, sp in zip(st_new, st_par))
    return out, state


# CAT's LMs the search cannot carry per slot, and what to use instead
_REFUSED_LMS = {
    "NGram": "load its ARPA file (cat/utils/pipeline/ngram.sh --arpa) as cat_b200.ngram.NGramLM(<ARPA>, labels) instead",
    "MultiDecoder": "its members (_weights, _decs) cannot be read; build a cat_b200.rnnt_decode.MultiLM(weights, lms) "
                    "from the built members instead",
    "PretrainedTransformer": "a Transformer LM's state grows with the prefix",
    "CausalTransformer": "a Transformer LM's state grows with the prefix",
}


def _check_lm(lm, caller, mix_ok=True):
    """An LM the search can fuse (NotImplementedError otherwise): an ``NGramLM``, a module with ``get_log_prob`` or, with
    ``mix_ok``, a ``MultiLM``."""
    name = type(lm).__name__
    if isinstance(lm, NGramLM) or (mix_ok and isinstance(lm, MultiLM)):
        return
    if isinstance(lm, MultiLM) or name == "MultiDecoder":
        raise NotImplementedError(f"{caller}: LM {name} is not supported as a member of a mix: mixes do not nest")
    if name in _REFUSED_LMS:
        raise NotImplementedError(f"{caller}: LM {name} is not supported: {_REFUSED_LMS[name]}")
    if not callable(getattr(lm, "get_log_prob", None)):
        raise NotImplementedError(f"{caller}: LM {name} is not supported: the LM must be a cat_b200.ngram.NGramLM or a "
                                  "module with get_log_prob(tokens (R, 1), state) -> (log-probs (R, 1, V), state)")


class MultiLM:
    """A weighted mix of LMs, the GPU stand-in for CAT's ``MultiDecoder`` (``cat/shared/decoder.py``), as LODR decoding uses
    it: ``MultiLM([0.28125, -0.3125], [NGramLM(<5-gram ARPA>, labels), NGramLM(<LODR bigram ARPA>, labels)])``.  Its row
    after a prefix is sum_i w_i LM_i, summed in fp64 in member order and rounded to fp32 once (DESIGN.md §7 "RNN-T beam
    search with an LM mix"); the search fuses it like one LM, with alpha and beta.  Members are ``NGramLM`` objects and
    neural LMs with CAT's ``get_log_prob`` and an LSTM-like state, built by the caller (CAT builds them from config files).
    As in CAT, zero-weight members are dropped.  ValueError: weights and lms of different lengths, a weight that is not a
    finite number, no member left, more than ``MAX_MIX`` members, n-gram members over different label sets, or n-gram
    members whose word rows do not fit the rows kernel's shared memory; NotImplementedError: a member the search cannot
    carry (CAT's KenLM ``NGram``, Transformers, nested mixes)."""

    def __init__(self, weights, lms):
        weights, lms = list(weights), list(lms)
        if len(weights) != len(lms):
            raise ValueError(f"MultiLM: {len(weights)} weights for {len(lms)} LMs")
        weights = [_weight(w, "every weight", "MultiLM") for w in weights]
        kept = [(w, lm) for w, lm in zip(weights, lms) if w != 0.0]
        if not kept:
            raise ValueError("MultiLM: every weight is zero, so nothing is left to fuse")
        if len(kept) > MAX_MIX:
            raise ValueError(f"MultiLM: at most {MAX_MIX} members of non-zero weight, not {len(kept)}")
        for _, lm in kept:
            _check_lm(lm, "MultiLM", mix_ok=False)
        self.weights = [w for w, _ in kept]
        self.lms = [lm for _, lm in kept]
        vs = {lm.V for lm in self.lms if isinstance(lm, NGramLM)}
        if len(vs) > 1:
            raise ValueError(f"MultiLM: the n-gram members are loaded for different numbers of labels {sorted(vs)}")
        if vs:
            self.check_smem(vs.pop(), "MultiLM")

    @property
    def has_ngram(self) -> bool:
        return any(isinstance(lm, NGramLM) for lm in self.lms)

    def check_smem(self, V: int, caller):
        """The rows kernel builds each n-gram word row and the V-wide fp64 sum in shared memory (ValueError if too big)"""
        W = max([lm.num_words for lm in self.lms if isinstance(lm, NGramLM)], default=0)
        if 8 * (W + V) > _MIX_SMEM:
            raise ValueError(f"{caller}: the mix's largest n-gram LM has {W} words and V = {V}; the mix rows are built in "
                             f"shared memory, which holds at most {_MIX_SMEM // 8} words plus labels")

    def score(self, input_ids, targets, input_lengths=None) -> torch.Tensor:
        """CAT's ``MultiDecoder.score``: sum_i w_i member_i.score(input_ids, targets, input_lengths), in member order,
        each product and sum in fp64, rounded to fp32 once.  ``NGramLM`` members score on the GPU (``NGramLM.score``); a
        neural member uses its own CAT ``score``.  The result is on input_ids' device."""
        out = None
        for w, lm in zip(self.weights, self.lms):
            x = w * lm.score(input_ids, targets, input_lengths).to(input_ids.device, torch.float64)
            out = x if out is None else out + x
        return out.float()

    def __repr__(self):
        return f"MultiLM({self.weights}, [{', '.join(type(lm).__name__ for lm in self.lms)}])"


def _as_lm(lm, caller):
    """CAT's ``MultiDecoder`` as a ``MultiLM`` when its ``_weights`` and ``_decs`` can be read (every member then checked as
    a ``MultiLM`` member); any other LM as it is."""
    if type(lm).__name__ != "MultiDecoder" or isinstance(lm, MultiLM):
        return lm
    try:
        weights, decs = list(lm._weights), list(lm._decs)
    except (AttributeError, TypeError):
        raise NotImplementedError(f"{caller}: LM MultiDecoder is not supported: {_REFUSED_LMS['MultiDecoder']}") from None
    return MultiLM(weights, decs)


def _check_ilm_joiner(joiner, caller):
    """A joiner the ILM can be estimated from (NotImplementedError otherwise): one with ``impl_forward``, except LogAdd."""
    name = type(joiner).__name__
    if name == "LogAdd":
        raise NotImplementedError(f"{caller}: ILM estimation is not supported for the LogAdd joiner (its impl_forward "
                                  "raises in CAT)")
    if not callable(getattr(joiner, "impl_forward", None)):
        raise NotImplementedError(f"{caller}: ILM estimation needs the joiner's impl_forward; {name} has none")


def _weight(x, what, caller) -> float:
    if isinstance(x, bool) or not isinstance(x, (int, float)) or not math.isfinite(x):
        raise ValueError(f"{caller}: {what} must be a finite number, not {x!r}")
    return float(x)


class _Joiner:
    """How the joiner's rows for a frame reach the kernel: LogAdd (f and g rows), JointNet in "add" mode (raw logits from
    fc(fc_enc(enc) + fc_dec(pn)), fc_enc applied once per call) or any other joiner (log-probs of joiner(enc, pn))."""

    def __init__(self, joiner, enc_out, caller, ilm=False):
        name = type(joiner).__name__
        self.joiner = joiner
        self.caller = caller
        self.ilm = ilm
        if name == "LogAdd":
            self.mode = _MODE_LOGADD
            self.f = enc_out.contiguous()
        elif name == "JointNet" and getattr(joiner, "_mode", None) == "add":
            self.mode = _MODE_LOGITS
            self.fe = joiner.fc_enc(enc_out)
            if ilm:   # impl_forward(0, pn) = fc(fc_enc(0) + fc_dec(pn)): fc_enc(0) is fc_enc's bias, once per call
                self.fe0 = joiner.fc_enc(torch.zeros_like(enc_out[:1, :1]))
        else:
            self.mode = _MODE_LOGPROBS
            self.enc = enc_out

    def ilm_rows(self, pn_out: torch.Tensor, R: int) -> torch.Tensor:
        """The ILM logits (R, V) of every slot, impl_forward(zeros, pn) (mode 0 joiners; JointNet "add" shares rows()'s
        fc_dec)"""
        enc = torch.zeros((R, 1, self.enc.shape[2]), dtype=self.enc.dtype, device=self.enc.device)
        return self.joiner.impl_forward(enc, pn_out).reshape(R, -1).contiguous()

    def rows(self, t: int, pn_out: torch.Tensor, N: int, B: int):
        """(rows (N*B, V) contiguous, f (N, Tmax, V) of the rows' dtype for LogAdd else None, and with ``ilm`` the ILM
        logits (N*B, V))"""
        R = N * B
        if self.mode == _MODE_LOGITS:
            fd = self.joiner.fc_dec(pn_out).reshape(N, B, -1)
            rows = self.joiner.fc(self.fe[:, t, None, :] + fd).reshape(R, -1).contiguous()
            if not self.ilm:
                return rows, None
            return rows, None, self.joiner.fc(self.fe0 + fd).reshape(R, -1).contiguous()
        out = self._rows(t, pn_out, N, B)
        return out + (self.ilm_rows(pn_out, R),) if self.ilm else out

    def _rows(self, t: int, pn_out: torch.Tensor, N: int, B: int) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
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
        enc = self.enc[:, t, None, None, :].expand(N, B, 1, -1).reshape(R, 1, -1)
        return self.joiner(enc, pn_out).reshape(R, -1).contiguous(), None


class _Fusion:
    """The external LM and ILM terms of the RNN-T search (DESIGN.md §7 "RNN-T beam search with LM fusion"), checked before
    anything runs.  The LM term is on iff ``lm`` is given and alpha != 0, the ILM term iff ilm_weight != 0.  Per call it
    carries the LM's per-slot state: an ``NGramLM``'s int32 states (double-buffered) and rows from
    ``ccb_ngram_slot_rows``, or a neural LM's output and state, carried like the predictor's.  A ``MultiLM`` carries
    each member so (every n-gram member double-buffered, every neural member through ``_carry``), and one
    ``ccb_lm_mix_slot_rows`` launch per frame makes the mix rows."""

    def __init__(self, lm, alpha, beta, ilm_weight, joiner, blank, caller):
        self.alpha = _weight(alpha, "alpha", caller)
        self.beta = _weight(beta, "beta", caller)
        self.ilm_weight = _weight(ilm_weight, "ilm_weight", caller)
        self.lm = _as_lm(lm, caller) if lm is not None and self.alpha != 0.0 else None
        self.ilm = self.ilm_weight != 0.0
        self.caller = caller
        if self.lm is not None:
            _check_lm(self.lm, caller)
            if (isinstance(self.lm, NGramLM) or isinstance(self.lm, MultiLM) and self.lm.has_ngram) and blank != 0:
                raise ValueError(f"{caller}: an NGramLM's label 0 is the blank, so blank must be 0, not {blank}")
        if self.ilm:
            _check_ilm_joiner(joiner, caller)

    @property
    def active(self) -> bool:
        return self.lm is not None or self.ilm

    def start(self, N: int, B: int, blank: int, dev):
        """The LM at the start of every hypothesis (no native call yet)"""
        self.N, self.B, self.R, self.blank = N, B, N * B, blank
        if isinstance(self.lm, NGramLM):
            self.state = [torch.empty((N, B), dtype=torch.int32, device=dev) for _ in range(2)]
            self.rows = None
        elif isinstance(self.lm, MultiLM):
            # per member: an n-gram's two state buffers, or a neural LM's [output, state]
            self.members = []
            for lm in self.lm.lms:
                if isinstance(lm, NGramLM):
                    self.members.append([torch.empty((N, B), dtype=torch.int32, device=dev) for _ in range(2)])
                else:
                    out, st = lm.get_log_prob(torch.full((self.R, 1), blank, dtype=torch.long, device=dev), None)
                    _check_state(lm, st, self.R, self.caller, "LM")
                    self.members.append([out, st])
            self.rows = None
        elif self.lm is not None:
            self.out, self.st = self.lm.get_log_prob(torch.full((self.R, 1), blank, dtype=torch.long, device=dev), None)
            _check_state(self.lm, self.st, self.R, self.caller, "LM")

    def check_v(self, V: int):
        """The LM's V against the joiner's (ValueError, before the first native call)"""
        if isinstance(self.lm, MultiLM):
            for i, (lm, m) in enumerate(zip(self.lm.lms, self.members)):
                lv = lm.V if isinstance(lm, NGramLM) else int(m[0].shape[-1])
                if lv != V:
                    raise ValueError(f"{self.caller}: member {i} of the LM mix has V = {lv} labels, the joiner V = {V}")
            self.lm.check_smem(V, self.caller)
            if self.rows is None:
                self.rows = torch.empty((self.R, V), dtype=torch.float32, device=self.members[0][0].device)
            return
        lv = self.lm.V if isinstance(self.lm, NGramLM) else None if self.lm is None else int(self.out.shape[-1])
        if lv is not None and lv != V:
            raise ValueError(f"{self.caller}: the LM has V = {lv} labels, the joiner V = {V}")
        if isinstance(self.lm, NGramLM) and self.rows is None:
            self.rows = torch.empty((self.R, V), dtype=torch.float32, device=self.state[0].device)

    def _ngram_rows(self, parent=None, token=None):
        # the next beam's states go to the other buffer; rows are overwritten (stream order keeps the last step's reads)
        src, dst = self.state
        _check(_lib.lib().ccb_ngram_slot_rows(
            self.lm.handle, self.N, self.B, self.rows.shape[1], None if parent is None else parent.data_ptr(),
            None if token is None else token.data_ptr(), None if parent is None else src.data_ptr(), dst.data_ptr(),
            self.rows.data_ptr(), _stream(dst.device)), self.caller)
        self.state.reverse()

    def _mix_rows(self, parent=None, token=None):
        # one launch: every n-gram member's next states (into its other buffer) and the mix rows (R, V) fp32.  The entry
        # takes the n-gram members first, then the neural ones, and the mix's order as a permutation of that list.
        lms, ws, mem = self.lm.lms, self.lm.weights, self.members
        ng = [i for i, lm in enumerate(lms) if isinstance(lm, NGramLM)]
        nn = [i for i, lm in enumerate(lms) if not isinstance(lm, NGramLM)]
        nrows = [_neural_rows(mem[i][0], self.R) for i in nn]   # (alive until the launch is enqueued)

        def arr(ctype, xs):
            return (ctype * max(len(xs), 1))(*xs)

        vp = C.c_void_p
        _check(_lib.lib().ccb_lm_mix_slot_rows(
            len(ng), arr(vp, [lms[i].handle for i in ng]), arr(C.c_double, [ws[i] for i in ng]),
            arr(vp, [mem[i][0].data_ptr() for i in ng]), arr(vp, [mem[i][1].data_ptr() for i in ng]),
            len(nn), arr(vp, [r.data_ptr() for r in nrows]), arr(C.c_int, [_DTYPES[r.dtype] for r in nrows]),
            arr(C.c_double, [ws[i] for i in nn]), arr(C.c_int, [(ng + nn).index(i) for i in range(len(lms))]),
            self.N, self.B, self.rows.shape[1], None if parent is None else parent.data_ptr(),
            None if token is None else token.data_ptr(), self.rows.data_ptr(), _stream(self.rows.device)), self.caller)
        for i in ng:
            mem[i].reverse()

    def first(self):
        """The first frame's LM rows (after the workspace's init)"""
        if isinstance(self.lm, NGramLM):
            self._ngram_rows()
        elif isinstance(self.lm, MultiLM):
            self._mix_rows()

    def lm_rows(self) -> Optional[torch.Tensor]:
        """The current beam's LM log-prob rows (R, V), or None without the LM term"""
        if self.lm is None:
            return None
        if isinstance(self.lm, (NGramLM, MultiLM)):
            return self.rows
        return _neural_rows(self.out, self.R)

    def advance(self, src, tok, ext, parent, token):
        """Every slot's LM after a frame: its parent's, advanced by the token it emitted"""
        if isinstance(self.lm, NGramLM):
            self._ngram_rows(parent, token)
        elif isinstance(self.lm, MultiLM):
            for lm, m in zip(self.lm.lms, self.members):
                if not isinstance(lm, NGramLM):
                    m[0], m[1] = _carry(lm.get_log_prob, m[0], m[1], src, tok, ext, self.blank,
                                        lambda st, lm=lm: _check_state(lm, st, self.R, self.caller, "LM"))
            self._mix_rows(parent, token)
        elif self.lm is not None:
            self.out, self.st = _carry(self.lm.get_log_prob, self.out, self.st, src, tok, ext, self.blank,
                                       lambda st: _check_state(self.lm, st, self.R, self.caller, "LM"))


def _neural_rows(out, R: int) -> torch.Tensor:
    """A neural LM's output as the (R, V) row block the kernels read: fp32, bf16 or fp16, contiguous"""
    rows = out.reshape(R, -1)
    return (rows if rows.dtype in _DTYPES else rows.float()).contiguous()


def _beam_search(name: str, family: str, enc_out, frame_lens, predictor, joiner, beam_size, nbest, blank,
                 fusion: Optional[_Fusion] = None):
    """The frame loop of the transducer searches: ``family`` "rnnt" or "ctct" picks the native ws-bytes, init and step entries
    (``ccb_<family>_beam_*``); both are finished by ``ccb_rnnt_beam_finish``.  ``name`` is the calling function's, for its
    errors.  Each frame runs the predictor once over all N*B slots, every slot keeping its parent's output and state or
    advancing them by the token it emitted; nothing synchronises the host.  With an active ``fusion`` (RNN-T only) the step
    is ``ccb_rnnt_beam_step_fused``, the LM is carried per slot like the predictor, and the returned scores are acoustic
    plus LM part."""
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
            join = _Joiner(joiner, enc_out, name, ilm=fusion is not None and fusion.ilm)
            if fusion is not None:
                fusion.start(N, B, blank, dev)
        parent = torch.empty((N, B), dtype=torch.int32, device=dev)
        token = torch.empty((N, B), dtype=torch.int32, device=dev)
        node = torch.empty((N, B), dtype=torch.int32, device=dev)
        score = torch.empty((N, B), dtype=torch.float64, device=dev)
        tokens = torch.empty((N, nbest, Tmax), dtype=torch.int32, device=dev)
        lengths = torch.empty((N, nbest), dtype=torch.int32, device=dev)
        scores = torch.empty((N, nbest), dtype=torch.float32, device=dev)
        slot_base = (torch.arange(N, device=dev, dtype=torch.long) * B)[:, None]
        lm_part = torch.zeros((N, B), dtype=torch.float64, device=dev) if fusion is not None else None
        ws = None

        def init():   # (after the first frame's rows: every argument error is raised before a native call)
            nonlocal ws
            ws = torch.empty(int(entry("ws_bytes")(N, Tmax, B)), dtype=torch.uint8, device=dev)
            _check(entry("init")(N, Tmax, B, ws.data_ptr(), parent.data_ptr(), token.data_ptr(), node.data_ptr(),
                                 score.data_ptr(), _stream(dev)), name)

        if Tmax == 0:
            init()
        for t in range(Tmax):
            rows, f, *ilm = join.rows(t, pn_out, N, B)
            if rows.dtype not in _DTYPES:
                rows = rows.float()
                f = f.float() if f is not None else None
            V = int(rows.shape[1])
            if blank >= V:
                raise ValueError(f"{name}: blank = {blank} is not a label of the joiner's V = {V}")
            if fusion is not None:
                fusion.check_v(V)
            if t == 0:
                init()
                if fusion is not None:
                    fusion.first()
            if fusion is None:
                _check(entry("step")(rows.data_ptr(), f.data_ptr() if f is not None else None, _DTYPES[rows.dtype],
                                     join.mode, N, Tmax, B, V, t, lens.data_ptr(), blank, ws.data_ptr(), parent.data_ptr(),
                                     token.data_ptr(), node.data_ptr(), score.data_ptr(), _stream(dev)), name)
            else:
                lmr = fusion.lm_rows()
                ilr = ilm[0] if ilm else None
                if ilr is not None and ilr.dtype not in _DTYPES:
                    ilr = ilr.float()
                _check(L.ccb_rnnt_beam_step_fused(
                    rows.data_ptr(), f.data_ptr() if f is not None else None, _DTYPES[rows.dtype], join.mode, N, Tmax, B, V,
                    t, lens.data_ptr(), blank, ws.data_ptr(), parent.data_ptr(), token.data_ptr(), node.data_ptr(),
                    score.data_ptr(), None if lmr is None else lmr.data_ptr(), _DTYPES[lmr.dtype] if lmr is not None else 0,
                    fusion.alpha, fusion.beta, None if ilr is None else ilr.data_ptr(),
                    _DTYPES[ilr.dtype] if ilr is not None else 0, fusion.ilm_weight, lm_part.data_ptr(), _stream(dev)), name)
            if t + 1 == Tmax:
                break
            # each slot's predictor output and state (and LM): its parent's, advanced by the token it emitted (if any)
            src = (slot_base + parent.long()).reshape(R)
            tok = token.reshape(R)
            ext = tok >= 0
            pn_out, state = _carry(predictor, pn_out, state, src, tok, ext, blank,
                                   lambda st: _check_state(predictor, st, R, name))
            if fusion is not None:
                fusion.advance(src, tok, ext, parent, token)
        if fusion is not None:
            score.add_(lm_part)   # the hypothesis score: acoustic plus LM part
        _check(L.ccb_rnnt_beam_finish(N, Tmax, B, nbest, ws.data_ptr(), node.data_ptr(), score.data_ptr(),
                                      tokens.data_ptr(), lengths.data_ptr(), scores.data_ptr(), _stream(dev)), name)
        lens.record_stream(torch.cuda.current_stream(dev))
    return tokens, lengths, scores


def rnnt_beam_search(enc_out: torch.Tensor, frame_lens: torch.Tensor, predictor, joiner, beam_size: int = 5,
                     nbest: Optional[int] = None, blank: int = 0, lm=None, alpha: float = 0.0, beta: float = 0.0,
                     ilm_weight: float = 0.0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The nbest (default beam_size) best label sequences of every utterance by CAT's RNA beam search (DESIGN.md §7
    "Transducer beam search"), blank = bos = ``blank``, with CAT's LM fusion and ILM estimation (§7 "RNN-T beam search with
    LM fusion").

    enc_out (N, T, H) on a CUDA device; frame_lens (N,) int32 or int64 on the CPU or that device (T_n in [0, T]; an
    utterance with T_n = 0 gets the empty hypothesis, score 0).  ``predictor(tokens (R, 1), state)`` returns (out (R, 1, H'),
    state) with a state that is None or a tuple of 3-D tensors with the batch on dim 1; ``joiner`` is CAT's LogAdd, a
    JointNet or any module called as joiner(enc (R, 1, H), pn (R, 1, H')) returning log-probs.  Returns device tensors
    tokens (N, nbest, T) int32 -1 padded, lengths (N, nbest) int32 (-1 past the hypotheses found) and scores (N, nbest)
    fp32, best first.  The frame loop runs to T; nothing synchronises the host.

    LM fusion (on iff ``lm`` is given and alpha != 0): every extension by token k != blank adds beta + alpha ln P_LM(k |
    prefix) to the hypothesis's LM part.  ``lm`` is a ``cat_b200.ngram.NGramLM`` loaded for the joiner's V labels (label 0
    the blank, so blank must be 0), a module whose ``get_log_prob(tokens (R, 1), state)`` returns (log-probs (R, 1, V),
    state) with a state like the predictor's (CAT's LSTM LM), or a ``MultiLM`` of such members (or CAT's ``MultiDecoder``
    with readable members), whose row sum_i w_i LM_i takes the place of ln P_LM, as in LODR decoding; any other LM raises
    NotImplementedError.  ILM estimation (on
    iff ilm_weight != 0): every extension adds ilm_weight (I[k] - logsumexp over the non-blank I), I the joiner's
    impl_forward(zeros, pn) logits (JointNet "add": fc(fc_enc's bias + fc_dec(pn))); LogAdd and joiners without
    impl_forward raise NotImplementedError.  Candidates rank by acoustic score plus LM part; merged hypotheses add only
    their acoustic scores and keep the LM part of the first; the returned scores are acoustic plus LM part.  alpha, beta
    and ilm_weight may have any sign."""
    fusion = _Fusion(lm, alpha, beta, ilm_weight, joiner, blank, "rnnt_beam_search")
    return _beam_search("rnnt_beam_search", "rnnt", enc_out, frame_lens, predictor, joiner, beam_size, nbest, blank,
                        fusion if fusion.active else None)


class RNNTDecoder:
    """CAT's ``cat.rnnt.rnnt_decoder.RNNTDecoder`` with its constructor, decoding on the GPU through ``rnnt_beam_search``.
    CAT's rules: alpha == 0 drops the LM whatever beta is, and ILM estimation is on iff est_ilm and ilm_weight != 0.
    ``lm_module`` is a ``cat_b200.ngram.NGramLM`` (in place of CAT's KenLM ``NGram``), a neural LM with CAT's
    ``get_log_prob`` and an LSTM-like state, or a weighted mix of those: a ``MultiLM``, or CAT's ``MultiDecoder`` whose
    ``_weights`` and ``_decs`` are such members (LODR decoding).  Returned scores are CAT's ``Hypothesis.score``: acoustic
    plus LM part.  Not supported (NotImplementedError, raised here): other LMs (KenLM ``NGram``, a ``MultiDecoder`` without
    readable members, Transformers), ILM estimation with LogAdd or a joiner without ``impl_forward``, an ``<eos>`` early
    stop and bos_id != blank_id."""

    def __init__(self, predictor, joiner, blank_id: int = 0, bos_id: int = 0, eos_id: int = -1, beam_size: int = 5,
                 nbest: int = -1, lm_module=None, alpha: float = 0.0, beta: float = 0.0, est_ilm: bool = False,
                 ilm_weight: float = 0.0):
        if bos_id != blank_id:
            raise NotImplementedError(f"RNNTDecoder: bos_id ({bos_id}) must equal blank_id ({blank_id}), as in CAT")
        fusion = _Fusion(lm_module, alpha, beta, ilm_weight if est_ilm else 0.0, joiner, blank_id, "RNNTDecoder")
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
        self.lm, self.alpha, self.beta = fusion.lm, fusion.alpha, fusion.beta
        self.ilm_weight = fusion.ilm_weight

    def __call__(self, enc_out: torch.Tensor, frame_lens: Optional[torch.Tensor] = None
                 ) -> List[Tuple[List[List[int]], List[float]]]:
        """[(token lists without bos, scores), ...] per utterance, best first: CAT's return value.  One host copy."""
        return _to_lists(*rnnt_beam_search(enc_out, _frame_lens(enc_out, frame_lens), self.predictor, self.joiner,
                                           self.beam_size, self.nbest, self.blank_id, self.lm, self.alpha, self.beta,
                                           self.ilm_weight))


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
