"""Beam search for CAT's CTC-T transducers (``topo: ctct``) on the GPU: the drop-in for ``cat/rnnt/ctct_decoder.py``'s
``CTCTDecoder``.  A CTC prefix beam search whose joint row depends on the prefix: every frame emits one symbol, as in the
CTC-T loss.  The networks run in torch, under the caller's autocast, in the transducer searches' shared frame loop; the
search (exact per-row top-k, prefix trie, order-free merge, ranked pruning) is one native launch per frame
(``cat_b200/csrc/ctct_decode.cu``).  Definition and differences from CAT: DESIGN.md §7 "CTC-T beam search".
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from .rnnt_decode import MAX_BEAM, _beam_search, _frame_lens, _to_lists


def ctct_beam_search(enc_out: torch.Tensor, frame_lens: torch.Tensor, predictor, joiner, beam_size: int = 5,
                     nbest: Optional[int] = None, blank: int = 0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The nbest (default beam_size) best label sequences of every utterance by CAT's CTC-T prefix beam search (DESIGN.md
    §7 "CTC-T beam search"), blank = bos = ``blank``; each frame extends every hypothesis by its row's min(beam_size, V - 1)
    most likely non-blank tokens.

    The arguments and results are ``rnnt_beam_search``'s: enc_out (N, T, H) on a CUDA device; frame_lens (N,) int32 or int64
    on the CPU or that device (T_n = 0: the empty hypothesis, score 0); ``predictor(tokens (R, 1), state)`` returns (out
    (R, 1, H'), state) with a state that is None or a tuple of 3-D tensors with the batch on dim 1; ``joiner`` is CAT's
    LogAdd, a JointNet or any module called as joiner(enc (R, 1, H), pn (R, 1, H')) returning log-probs.  Returns device
    tensors tokens (N, nbest, T) int32 -1 padded, lengths (N, nbest) int32 (-1 past the hypotheses found) and scores
    (N, nbest) fp32, best first.  Nothing synchronises the host."""
    return _beam_search("ctct_beam_search", "ctct", enc_out, frame_lens, predictor, joiner, beam_size, nbest, blank)


class CTCTDecoder:
    """CAT's ``cat.rnnt.ctct_decoder.CTCTDecoder`` with its constructor (``RNNTDecoder``'s), decoding on the GPU through
    ``ctct_beam_search``.  As in CAT: any eos_id is accepted and ignored (the search has no early stop), est_ilm and
    ilm_weight are accepted and ignored, and alpha == 0 drops the LM.  An LM with alpha != 0 raises NotImplementedError
    (CAT asserts), and so does bos_id != blank_id.  A blank_id other than 0 is excluded from the top-k, where CAT always
    excludes index 0."""

    def __init__(self, predictor, joiner, blank_id: int = 0, bos_id: int = 0, eos_id: int = -1, beam_size: int = 5,
                 nbest: int = -1, lm_module=None, alpha: float = 0.0, beta: float = 0.0, est_ilm: bool = False,
                 ilm_weight: float = 0.0):
        if bos_id != blank_id:
            raise NotImplementedError(f"CTCTDecoder: bos_id ({bos_id}) must equal blank_id ({blank_id}), as in CAT")
        if alpha == 0.0:
            lm_module = None
        if lm_module is not None:
            raise NotImplementedError("CTCTDecoder: external LM fusion (lm_module with alpha != 0) is not supported, "
                                      "as in CAT")
        if isinstance(beam_size, bool) or not isinstance(beam_size, int) or not 1 <= beam_size <= MAX_BEAM:
            raise ValueError(f"CTCTDecoder: beam_size must be an int in [1, {MAX_BEAM}], not {beam_size!r}")
        if nbest == -1:
            nbest = beam_size
        if isinstance(nbest, bool) or not isinstance(nbest, int) or nbest < 1:
            raise ValueError(f"CTCTDecoder: nbest must be -1 or a positive int, not {nbest!r}")
        self.predictor = predictor
        self.joiner = joiner
        self.blank_id = blank_id
        self.bos_id = bos_id
        self.eos_id = eos_id
        self.beam_size = beam_size
        self.nbest = min(nbest, beam_size)

    def __call__(self, enc_out: torch.Tensor, frame_lens: Optional[torch.Tensor] = None
                 ) -> List[Tuple[List[List[int]], List[float]]]:
        """[(token lists without bos, scores), ...] per utterance, best first: CAT's return value.  One host copy."""
        return _to_lists(*ctct_beam_search(enc_out, _frame_lens(enc_out, frame_lens), self.predictor, self.joiner,
                                           self.beam_size, self.nbest, self.blank_id))
