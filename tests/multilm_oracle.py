"""Test infrastructure for the RNN-T beam search with an LM mix (``cat_b200.rnnt_decode.MultiLM``, DESIGN.md §7 "RNN-T beam
search with an LM mix"), written from its definition.

``CatMultiDecoder`` restates CAT's ``MultiDecoder.get_log_prob`` (``cat/shared/decoder.py``) over built members (the
``CatNGram`` and ``LSTMLM`` stand-ins of tests/rnnt_fusion_oracle.py), with a tuple state; it plugs into
``cat_decode_fused`` as its LM.  ``mix_rows`` is the mix row in the kernel's order, in numpy.
"""
from __future__ import annotations

import numpy as np
import torch


class MultiDecoder(torch.nn.Module):
    """CAT's MultiDecoder over built members (named as CAT's, which is how the search recognises it): ``_weights`` and
    ``_decs`` as CAT keeps them (zero-weight members dropped), get_log_prob(x, hidden) -> (sum_i w_i out_i, summed in
    member order as torch does, (state_1, ..., state_K)); hidden None starts every member."""

    def __init__(self, weights, decs):
        super().__init__()
        kept = [(w, d) for w, d in zip(weights, decs) if w != 0.0]
        self._weights = [w for w, _ in kept]
        mods = [d for _, d in kept]
        # CAT keeps its members in an nn.ModuleList; the CatNGram stand-in is not a module, so a plain list holds it then
        self._decs = torch.nn.ModuleList(mods) if all(isinstance(d, torch.nn.Module) for d in mods) else mods
        self._num_decs = len(kept)

    def get_log_prob(self, x, hidden=None):
        out = 0.0
        state = []
        for i in range(self._num_decs):
            part_out, part_state = self._decs[i].get_log_prob(x, None if hidden is None else hidden[i])
            out = out + part_out.to(x.device) * self._weights[i]
            state.append(part_state)
        return out, tuple(state)


CatMultiDecoder = MultiDecoder


def mix_rows(rows, weights, dtype=np.float32):
    """The mix row sum_i w_i rows[i] in the kernel's order: each member's row widened exactly to fp64, each product and sum
    rounded on its own, the first product starting the sum, in member order; -inf wherever a member is -inf; rounded to
    ``dtype`` once."""
    acc, dead = None, None
    with np.errstate(invalid="ignore"):
        for r, w in zip(rows, weights):
            r = np.asarray(r).astype(np.float64)
            x = w * r
            acc = x if acc is None else acc + x
            dead = (r == -np.inf) if dead is None else dead | (r == -np.inf)
        return np.where(dead, -np.inf, acc).astype(dtype)
