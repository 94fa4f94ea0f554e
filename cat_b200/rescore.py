"""N-best rescoring with an LM on the GPU: CAT's ``cat/lm/rescore.py`` arithmetic applied to the device outputs of
``rnnt_beam_search``, ``ctct_beam_search`` and ``ctc_beam_search``, without a host synchronisation.
"""
from __future__ import annotations

from typing import Tuple

import torch

from .rnnt_decode import _as_lm, _weight


def rescore_nbest(tokens: torch.Tensor, lengths: torch.Tensor, scores: torch.Tensor, lm, alpha: float = 0.0,
                  beta: float = 0.0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Rescore N-best lists as CAT's ``rescore.py`` does.  tokens (N, K, T) int32 padded with -1, lengths (N, K) (-1: no
    hypothesis in that row) and scores (N, K), as the beam searches return them; lm an ``NGramLM``, a ``MultiLM``, CAT's
    ``MultiDecoder`` or any LM with CAT's ``score(input_ids, targets, input_lengths)``.
    Each hypothesis l becomes CAT's rescoring input: token 0 prepended (it is scored as <s>), length len(l) + 1, and
    token 0 (</s>) as the last target.  Returns device tensors
      lm_scores (N, K) fp32: lm.score of each hypothesis (what ``--save-lm-nbest`` stores), -inf for absent rows;
      total (N, K) fp32: scores + alpha * lm_scores + beta * (len(l) + 1), in that order in fp32, -inf for absent rows;
      best (N,) int64: the first index of the largest total per utterance (0 when every row is absent).
    alpha and beta are finite numbers (ValueError otherwise)."""
    alpha = _weight(alpha, "alpha", "rescore_nbest")
    beta = _weight(beta, "beta", "rescore_nbest")
    if not (isinstance(tokens, torch.Tensor) and tokens.dim() == 3 and isinstance(lengths, torch.Tensor)
            and isinstance(scores, torch.Tensor) and tuple(lengths.shape) == tuple(tokens.shape[:2])
            and tuple(scores.shape) == tuple(tokens.shape[:2])):
        raise ValueError("rescore_nbest: tokens must be (N, K, T) and lengths and scores (N, K) tensors")
    N, K, T = (int(x) for x in tokens.shape)
    lm = _as_lm(lm, "rescore_nbest")
    present = lengths >= 0
    in_lens = lengths.clamp(min=0).to(torch.int64).reshape(-1) + 1
    in_toks = torch.zeros((N * K, T + 1), dtype=torch.int64, device=tokens.device)
    in_toks[:, 1:] = tokens.reshape(N * K, T).clamp(min=0)
    targets = torch.zeros((N * K, 1), dtype=torch.int64, device=tokens.device)
    lm_scores = lm.score(in_toks, targets, in_lens).reshape(N, K).masked_fill(~present, float("-inf"))
    total = (scores.float() + alpha * lm_scores + beta * in_lens.reshape(N, K)).masked_fill(~present, float("-inf"))
    return lm_scores, total, total.argmax(dim=1)
