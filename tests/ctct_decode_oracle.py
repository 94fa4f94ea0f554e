"""Test infrastructure: two restatements of the CTC-T prefix beam search (``cat_b200.ctct_decode``, DESIGN.md §7 "CTC-T beam
search"), written from its definition.

``beam_ref`` is the search in fp64 numpy over a callback ``lp(t, prefix) -> row``; ``cat_decode`` is CAT's per-hypothesis,
dict-merging CTC-T decoder restated in torch over real predictor and joiner modules (its rows computed by the joiner's own
forward, its scores in fp64).  The modules are tests/rnnt_decode_oracle.py's.
"""
from __future__ import annotations

import numpy as np
import torch

NEG = -np.inf


def _lae(a: float, b: float) -> float:
    return float(np.logaddexp(a, b))


def topk(row, k: int, blank: int):
    """The k non-blank tokens with the largest row value, ties to the lower token (-inf values included)."""
    return sorted((c for c in range(len(row)) if c != blank), key=lambda c: (-row[c], c))[:k]


def beam_ref(T: int, V: int, B: int, lp, nbest=None, blank: int = 0):
    """[(prefix tuple, score)] best first, at most min(nbest, |beam|): T frames, beam B, rows lp(t, prefix) (V,) fp64.

    An entry is (prefix, b, n), the beam starting as [((), -inf, 0)].  Per frame, entry r with s = b (+) n and row lp_r:
    extension (r, j), c = topk(lp_r)[j], adds (c == last ? b : s) + lp_r[c] to n(prefix + c), key r (k + 1) + j; the stay
    adds s + lp_r[blank] to b(prefix) and, for a non-empty prefix, n + lp_r[last] to n(prefix), key r (k + 1) + k.  A
    target's key is its smallest; the min(B, #finite) best by (s desc, key asc) are the next beam, in that order."""
    k = min(B, V - 1)
    beam = [((), NEG, 0.0)]
    for t in range(T):
        tgt = {}

        def add(p, key, b=NEG, n=NEG):
            if p in tgt:
                e = tgt[p]
                tgt[p] = (_lae(e[0], b), _lae(e[1], n), min(e[2], key))
            else:
                tgt[p] = (b, n, key)

        for r, (p, b, n) in enumerate(beam):
            row = np.asarray(lp(t, p), dtype=np.float64)
            assert row.shape == (V,)
            s = _lae(b, n)
            last = p[-1] if p else None
            for j, c in enumerate(topk(row, k, blank)):
                add(p + (c,), r * (k + 1) + j, n=(b if c == last else s) + float(row[c]))
            add(p, r * (k + 1) + k, b=s + float(row[blank]), n=n + float(row[last]) if p else NEG)
        live = [(p, b, n, key) for p, (b, n, key) in tgt.items() if _lae(b, n) > NEG]
        live.sort(key=lambda e: (-_lae(e[1], e[2]), e[3]))
        beam = [(p, b, n) for p, b, n, _ in live[:B]]
    out = [(p, _lae(b, n)) for p, b, n in beam]
    return out[:len(out) if nbest is None else nbest]


@torch.no_grad()
def cat_decode(enc_out, frame_lens, predictor, joiner, beam_size, nbest=None, blank=0):
    """CAT's CTCTDecoder restated hypothesis by hypothesis: each hypothesis carries its prefix, masses b and n (fp64),
    predictor output and state; the joiner's log-probs come from joiner(enc (1, 1, H), pn (1, 1, H')).  Each frame visits
    the hypotheses in beam order, each one's top-k extensions then its stay, merging them into a dict in that order; the
    dict's hypotheses with s > -inf are ranked by s (stable) and the first beam_size kept.  Returns [(token lists,
    scores)] per utterance, as CTCTDecoder.__call__."""
    nbest = beam_size if nbest is None else nbest
    dev = enc_out.device
    res = []
    for n in range(enc_out.shape[0]):
        pn, st = predictor(torch.full((1, 1), blank, dtype=torch.long, device=dev), None)
        hyps = {(): [NEG, 0.0, pn, st]}
        for t in range(int(frame_lens[n])):
            enc = enc_out[n, t].reshape(1, 1, -1)
            nxt = {}
            for p, (b, nb_, pn, st) in hyps.items():
                row = joiner(enc, pn).reshape(-1).double().cpu().numpy()
                V = row.shape[0]
                s = _lae(b, nb_)
                for c in topk(row, min(beam_size, V - 1), blank):
                    v = (b if p and c == p[-1] else s) + float(row[c])
                    q = p + (c,)
                    if q in nxt:
                        nxt[q][1] = _lae(nxt[q][1], v)
                    else:
                        pq, sq = predictor(torch.full((1, 1), c, dtype=torch.long, device=dev), st)
                        nxt[q] = [NEG, v, pq, sq]
                vb = s + float(row[blank])
                vn = nb_ + float(row[p[-1]]) if p else NEG
                if p in nxt:
                    nxt[p][0] = _lae(nxt[p][0], vb)
                    nxt[p][1] = _lae(nxt[p][1], vn)
                else:
                    nxt[p] = [vb, vn, pn, st]
            ranked = sorted((h for h in nxt.items() if _lae(h[1][0], h[1][1]) > NEG),
                            key=lambda h: -_lae(h[1][0], h[1][1]))
            hyps = dict(ranked[:beam_size])
        out = list(hyps.items())[:nbest]
        res.append(([list(p) for p, _ in out], [_lae(h[0], h[1]) for _, h in out]))
    return res
