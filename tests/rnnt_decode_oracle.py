"""Test infrastructure: two restatements of the transducer beam search (``cat_b200.rnnt_decode``, DESIGN.md §7
"Transducer beam search"), written from its definition.

``beam_ref`` is the search in fp64 numpy over a callback ``lp(t, prefix) -> row``; ``cat_decode`` is CAT's
per-hypothesis, dict-merging RNA decoder restated in torch over real predictor and joiner modules (its rows computed by the
joiner's own forward, its scores in fp64).
"""
from __future__ import annotations

import numpy as np
import torch


def _lae(a: float, b: float) -> float:
    return float(np.logaddexp(a, b))


def beam_ref(T: int, V: int, B: int, lp, nbest=None):
    """[(prefix tuple, score)] best first, at most min(nbest, |beam|): T frames, beam B, rows lp(t, prefix) (V,) fp64,
    blank 0.  Each frame keeps the min(B, |beam| V) best candidates (value desc, flat index asc, -inf dropped), visits them
    in increasing flat index and merges those with the same target prefix by logaddexp in that order."""
    beam = [((), 0.0)]
    for t in range(T):
        cands = []
        for r, (p, s) in enumerate(beam):
            row = np.asarray(lp(t, p), dtype=np.float64)
            assert row.shape == (V,)
            for k in range(V):
                v = s + float(row[k])
                if v > -np.inf:
                    cands.append((v, r * V + k))
        cands.sort(key=lambda c: (-c[0], c[1]))
        kept = sorted(cands[:B], key=lambda c: c[1])
        nxt = {}
        for v, f in kept:
            r, k = divmod(f, V)
            q = beam[r][0] if k == 0 else beam[r][0] + (k,)
            nxt[q] = _lae(nxt[q], v) if q in nxt else v
        beam = list(nxt.items())   # insertion order: first appearance
    beam.sort(key=lambda h: -h[1])   # stable
    return beam[:len(beam) if nbest is None else nbest]


def exhaustive(T: int, V: int, lp):
    """{prefix: log-sum of every emission sequence of T frames (blank 0) that emits it}, rows depending on the prefix
    emitted before each frame."""
    out = {}

    def walk(t, p, s):
        if t == T:
            out[p] = _lae(out[p], s) if p in out else s
            return
        row = np.asarray(lp(t, p), dtype=np.float64)
        for k in range(V):
            walk(t + 1, p if k == 0 else p + (k,), s + float(row[k]))

    walk(0, (), 0.0)
    return out


@torch.no_grad()
def cat_decode(enc_out, frame_lens, predictor, joiner, beam_size, nbest=None, blank=0):
    """CAT's RNNTDecoder.batch_decode restated hypothesis by hypothesis: each hypothesis carries its prefix, score (fp64),
    predictor output and state; the joiner's log-probs come from joiner(enc (1, 1, H), pn (1, 1, H')).  Returns
    [(token lists, scores)] per utterance, as RNNTDecoder.__call__."""
    nbest = beam_size if nbest is None else nbest
    res = []
    for n in range(enc_out.shape[0]):
        pn, st = predictor(torch.full((1, 1), blank, dtype=torch.long, device=enc_out.device), None)
        hyps = {(): (0.0, pn, st)}
        for t in range(int(frame_lens[n])):
            order = list(hyps.items())
            enc = enc_out[n, t].reshape(1, 1, -1)
            rows = [joiner(enc, h[1]).reshape(-1).double().cpu().numpy() for _, h in order]
            V = rows[0].shape[0]
            flat = [(order[r][1][0] + float(rows[r][k]), r * V + k) for r in range(len(order)) for k in range(V)]
            flat = [c for c in flat if c[0] > -np.inf]
            flat.sort(key=lambda c: (-c[0], c[1]))
            nxt = {}
            for v, f in sorted(flat[:beam_size], key=lambda c: c[1]):
                r, k = divmod(f, V)
                p, (s, pn, st) = order[r]
                if k == blank:
                    q, cache = p, (pn, st)
                else:
                    q = p + (k,)
                    cache = predictor(torch.full((1, 1), k, dtype=torch.long, device=enc_out.device), st) if q not in nxt \
                        else None
                if q in nxt:
                    nxt[q] = (_lae(nxt[q][0], v),) + nxt[q][1:]
                else:
                    nxt[q] = (v,) + tuple(cache)
            hyps = nxt
        ranked = sorted(hyps.items(), key=lambda h: -h[1][0])[:nbest]
        res.append(([list(p) for p, _ in ranked], [h[0] for _, h in ranked]))
    return res


# ---- small stand-ins for CAT's modules (their call conventions and, for the joiners, their class names) ----------------
class LSTMPredictor(torch.nn.Module):
    """CAT's LSTM predictor with ``with_head: false``: embedding, one LSTM layer; forward(tokens (R, U), state) -> (out
    (R, U, H), (h, c))."""

    def __init__(self, V, H):
        super().__init__()
        self.embedding = torch.nn.Embedding(V, H)
        self.rnn = torch.nn.LSTM(H, H, batch_first=True)

    def forward(self, x, hidden=None):
        return self.rnn(self.embedding(x), hidden)


class EmbeddingPredictor(torch.nn.Module):
    """CAT's Embedding predictor with a head: forward(tokens, state) -> (classifier(relu(embed)), None)."""

    def __init__(self, V, H, out=None):
        super().__init__()
        self.embedding = torch.nn.Embedding(V, H)
        self.classifier = torch.nn.Linear(H, out or H)

    def forward(self, x, *args):
        return self.classifier(torch.relu(self.embedding(x))), None


class JointNet(torch.nn.Module):
    """CAT's JointNet in "add" mode: log_softmax(fc(fc_enc(enc) + fc_dec(pn))), fc = tanh then a linear layer."""

    def __init__(self, He, Hp, V, H):
        super().__init__()
        self.fc_enc = torch.nn.Linear(He, H)
        self.fc_dec = torch.nn.Linear(Hp, H)
        self.fc = torch.nn.Sequential(torch.nn.Tanh(), torch.nn.Linear(H, V))
        self._mode = "add"

    def forward(self, enc, pn):
        if enc.dim() == 3:
            return self.fc(self.fc_enc(enc)[:, :, None, :] + self.fc_dec(pn)[:, None, :, :]).log_softmax(-1)
        return self.fc(self.fc_enc(enc) + self.fc_dec(pn)).log_softmax(-1)


class LogAdd(torch.nn.Module):
    """CAT's LogAdd joiner: log_softmax(f + g)."""

    def forward(self, f, g):
        if f.dim() == 3:
            return (f[:, :, None, :] + g[:, None, :, :]).log_softmax(-1)
        return (f + g).log_softmax(-1)


class CatJoiner(torch.nn.Module):
    """A joiner the search calls as a black box (CAT's "cat" join mode): log_softmax(fc(cat(enc, pn)))."""

    def __init__(self, He, Hp, V):
        super().__init__()
        self.fc = torch.nn.Sequential(torch.nn.Tanh(), torch.nn.Linear(He + Hp, V))

    def forward(self, enc, pn):
        T, U = enc.shape[1], pn.shape[1]
        x = torch.cat([enc[:, :, None, :].expand(-1, -1, U, -1), pn[:, None, :, :].expand(-1, T, -1, -1)], -1)
        return self.fc(x).log_softmax(-1)


def module_lp(enc_row, predictor, joiner, blank=0):
    """lp(t, prefix) for beam_ref from the modules: the predictor run over (blank, prefix...) from scratch, then the joiner
    on enc_row(t) (1, 1, H); fp64 numpy."""
    @torch.no_grad()
    def lp(t, p):
        x = torch.tensor([[blank, *p]], dtype=torch.long, device=enc_row(t).device)
        out, _ = predictor(x, None)
        return joiner(enc_row(t), out[:, -1:]).reshape(-1).double().cpu().numpy()
    return lp
