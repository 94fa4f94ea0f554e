"""Test infrastructure for the RNN-T beam search with LM fusion and ILM estimation (``cat_b200.rnnt_decode``, DESIGN.md §7
"RNN-T beam search with LM fusion"), written from its definition.

``beam_ref_fused`` is the search in fp64 numpy over callbacks ``lp(t, prefix)`` (acoustic row) and ``term(t, prefix)``
(fusion terms), in the kernel's arithmetic order; ``cat_decode_fused`` restates CAT's ``RNNTDecoder.batch_decode`` with an
LM and ILM hypothesis by hypothesis over real modules.  The stand-ins: a ``JointNet`` with ``impl_forward`` in "add" and
"cat" mode, CAT's LSTM LM, and ``CatNGram``, CAT's KenLM ``NGram`` restated over the textbook ARPA scorer.
"""
from __future__ import annotations

import numpy as np
import torch

from rnnt_decode_oracle import _lae
from test_ngram_dispatch import LN10, Textbook


def fuse_term(lm_row, ilm_row, alpha, beta, w, blank=0):
    """The fusion term of every column, fp64, in the kernel's order: (beta + alpha LM) + w (I - lse), I - lse formed in the
    ILM row's own precision, lse over the non-blank columns; -inf where an LM or ILM entry is -inf; the blank column 0.
    Either row may be None (that term off)."""
    V = len(lm_row if lm_row is not None else ilm_row)
    term = np.zeros(V)
    dead = np.zeros(V, dtype=bool)
    if lm_row is not None:
        lm = np.asarray(lm_row, dtype=np.float64)
        term = beta + alpha * lm
        dead |= lm == -np.inf
    if ilm_row is not None:
        I = np.asarray(ilm_row)
        nb = np.delete(I.astype(np.float64), blank)
        lse = np.logaddexp.reduce(nb) if nb.size else -np.inf
        x = (I - I.dtype.type(lse)).astype(I.dtype).astype(np.float64)
        wx = w * x
        term = term + wx if lm_row is not None else wx
        dead |= I == -np.inf
    term = np.where(dead, -np.inf, term)
    term[blank] = 0.0
    return term


def beam_ref_fused(T, V, B, lp, term=None, nbest=None, blank=0):
    """[(prefix, score = acoustic + LM part)] best first: the fused search.  Candidate (r, k) ranks by
    ((s_r + lp[k]) + m_r) + [k != blank] term[k] (value desc, flat index asc, -inf dropped); the kept ones, in increasing
    flat index, merge their acoustic parts s_r + lp[k] by logaddexp per target prefix, and a target keeps the LM part of
    its first candidate (m_r for blank, m_r + term[k] for an extension).  term None: the search without fusion."""
    beam = [((), 0.0, 0.0)]
    for t in range(T):
        cands, terms = [], []
        for r, (p, s, m) in enumerate(beam):
            row = np.asarray(lp(t, p), dtype=np.float64)
            tr = None if term is None else np.asarray(term(t, p), dtype=np.float64)
            terms.append(tr)
            for k in range(V):
                a = s + float(row[k])
                v = a + m
                if tr is not None and k != blank:
                    v = -np.inf if tr[k] == -np.inf else v + float(tr[k])
                if v > -np.inf:
                    cands.append((v, r * V + k, a))
        cands.sort(key=lambda c: (-c[0], c[1]))
        nxt = {}
        for v, f, a in sorted(cands[:B], key=lambda c: c[1]):
            r, k = divmod(f, V)
            p, _, m = beam[r]
            q = p if k == blank else p + (k,)
            if q in nxt:
                nxt[q][0] = _lae(nxt[q][0], a)
            else:
                nxt[q] = [a, m if k == blank or terms[r] is None else m + float(terms[r][k])]
        beam = [(q, s, m) for q, (s, m) in nxt.items()]
    ranked = sorted(((p, s + m) for p, s, m in beam), key=lambda h: -h[1])   # stable
    return ranked[:len(ranked) if nbest is None else nbest]


def prefix_ilm(pred, joiner, He, blank=0):
    """I(prefix): the joiner's impl_forward(zeros, pn) logits for the predictor run over (blank, prefix...), fp64 numpy"""
    @torch.no_grad()
    def ilm(p):
        dev = next(pred.parameters()).device
        out, _ = pred(torch.tensor([[blank, *p]], dtype=torch.long, device=dev), None)
        zero = torch.zeros((1, 1, He), dtype=out.dtype, device=dev)
        return joiner.impl_forward(zero, out[:, -1:]).reshape(-1).double().cpu().numpy()
    return ilm


def prefix_lm(lm, blank=0):
    """LM(prefix): the LM's log-prob row after (blank, prefix...), run from its start state, fp64 numpy"""
    @torch.no_grad()
    def row(p):
        st, out = None, None
        for x in (blank, *p):
            out, st = lm.get_log_prob(torch.tensor([[x]], dtype=torch.long, device=_device(lm)), st)
        return np.asarray(out.reshape(-1).double().cpu().numpy())
    return row


def _device(m):
    ps = list(m.parameters()) if isinstance(m, torch.nn.Module) else []
    return ps[0].device if ps else torch.device("cpu")


@torch.no_grad()
def cat_decode_fused(enc_out, frame_lens, predictor, joiner, beam_size, nbest=None, lm=None, alpha=0.0, beta=0.0,
                     ilm_weight=0.0, blank=0):
    """CAT's RNNTDecoder.batch_decode (cat/rnnt/rnnt_decoder.py) with an LM (on iff lm and alpha != 0) and ILM estimation
    (on iff ilm_weight != 0), hypothesis by hypothesis: each carries its prefix, acoustic log-prob and LM part (fp64),
    predictor output and state, LM output and state.  combine = log_prob + (s + m), + beta + alpha LM and + w
    log_softmax(I[1:]) on the non-blank columns; the B best (value desc, flat asc), visited in flat order; a merged target
    adds only s_h + log_prob and keeps the LM part of the candidate that created it.  Returns [(token lists, scores)]."""
    nbest = beam_size if nbest is None else nbest
    use_lm = lm is not None and alpha != 0.0
    use_ilm = ilm_weight != 0.0
    dev = enc_out.device
    He = enc_out.shape[-1]

    def tok(x):
        return torch.full((1, 1), x, dtype=torch.long, device=dev)

    res = []
    for n in range(enc_out.shape[0]):
        pn, st = predictor(tok(blank), None)
        lmo, lms = lm.get_log_prob(tok(blank), None) if use_lm else (None, None)
        hyps = {(): (0.0, 0.0, pn, st, lmo, lms)}
        for t in range(int(frame_lens[n])):
            order = list(hyps.items())
            enc = enc_out[n, t].reshape(1, 1, -1)
            rows, combs = [], []
            for _, (s, m, pn, _, lmo, _) in order:
                row = joiner(enc, pn).reshape(-1).double().cpu().numpy()
                comb = row + (s + m)
                if use_lm:
                    comb[1:] += beta + alpha * lmo.reshape(-1).double().cpu().numpy()[1:]
                if use_ilm:
                    il = joiner.impl_forward(torch.zeros((1, 1, He), dtype=enc.dtype, device=dev), pn)
                    il = il.reshape(-1).double()
                    comb[1:] += ilm_weight * torch.log_softmax(il[1:], 0).cpu().numpy()
                rows.append(row)
                combs.append(comb)
            V = rows[0].shape[0]
            flat = [(combs[r][k], r * V + k) for r in range(len(order)) for k in range(V) if combs[r][k] > -np.inf]
            flat.sort(key=lambda c: (-c[0], c[1]))
            nxt = {}
            for v, f in sorted(flat[:beam_size], key=lambda c: c[1]):
                r, k = divmod(f, V)
                p, (s, m, pn, st, lmo, lms) = order[r]
                a = s + float(rows[r][k])
                q = p if k == blank else p + (k,)
                if q in nxt:
                    nxt[q] = (_lae(nxt[q][0], a),) + nxt[q][1:]
                    continue
                if k == blank:
                    nxt[q] = (a, m, pn, st, lmo, lms)
                    continue
                m2 = m + float(combs[r][k] - (rows[r][k] + (s + m)))   # the candidate's LM and ILM terms
                pn2, st2 = predictor(tok(k), st)
                lmo2, lms2 = lm.get_log_prob(tok(k), lms) if use_lm else (None, None)
                nxt[q] = (a, m2, pn2, st2, lmo2, lms2)
            hyps = nxt
        ranked = sorted(((p, h[0] + h[1]) for p, h in hyps.items()), key=lambda h: -h[1])[:nbest]
        res.append(([list(p) for p, _ in ranked], [s for _, s in ranked]))
    return res


# ---- stand-ins for CAT's modules -----------------------------------------------------------------------------------------
class JointNet(torch.nn.Module):
    """CAT's JointNet with impl_forward: "add" mode fc(fc_enc(enc) + fc_dec(pn)), "cat" mode fc(cat(enc, pn)), fc = tanh
    then a linear layer; forward is impl_forward's log_softmax."""

    def __init__(self, He, Hp, V, H, mode="add"):
        super().__init__()
        if mode == "add":
            self.fc_enc = torch.nn.Linear(He, H)
            self.fc_dec = torch.nn.Linear(Hp, H)
        else:
            self.fc_enc = self.fc_dec = None
            H = He + Hp
        self.fc = torch.nn.Sequential(torch.nn.Tanh(), torch.nn.Linear(H, V))
        self._mode = mode

    def impl_forward(self, enc, pn):
        if self._mode == "add":
            enc, pn = self.fc_enc(enc), self.fc_dec(pn)
            if enc.dim() == 3:
                return self.fc(enc[:, :, None, :] + pn[:, None, :, :])
            return self.fc(enc + pn)
        if enc.dim() == 3:
            T, U = enc.shape[1], pn.shape[1]
            return self.fc(torch.cat([enc[:, :, None, :].expand(-1, -1, U, -1), pn[:, None, :, :].expand(-1, T, -1, -1)], -1))
        return self.fc(torch.cat([enc, pn], -1))

    def forward(self, enc, pn):
        return self.impl_forward(enc, pn).log_softmax(-1)


class LSTMLM(torch.nn.Module):
    """CAT's LSTM LM (cat/shared/decoder.py LSTM): embedding, one LSTM layer, classifier; get_log_prob(tokens (R, U),
    state) -> (log-probs (R, U, V), (h, c))."""

    def __init__(self, V, H):
        super().__init__()
        self.embedding = torch.nn.Embedding(V, H)
        self.rnn = torch.nn.LSTM(H, H, batch_first=True)
        self.classifier = torch.nn.Linear(H, V)

    def forward(self, x, hidden=None):
        out, st = self.rnn(self.embedding(x), hidden)
        return self.classifier(out), st

    def get_log_prob(self, x, hidden=None):
        logits, st = self.forward(x, hidden)
        return logits.log_softmax(-1), st


class CatNGram:
    """CAT's KenLM NGram (cat/shared/decoder.py:516-613) over the textbook ARPA scorer: token 0 is the word </s>, token i
    the word labels[i]; get_log_prob(token (1, 1), history) appends the token's word to the history (None: empty) and
    returns ln 10 * log10 P(word(k) | last n-1 words) for every k (column 0 is 0, never used) and the new history."""

    def __init__(self, path, labels):
        self.tb = Textbook(path, labels)
        self.labels = labels
        self.V = len(labels)

    def word(self, i):
        return "</s>" if i == 0 else self.tb.word(self.labels[i])

    def row(self, hist):
        n = self.tb.order - 1
        h = tuple(hist[max(0, len(hist) - n):]) if n > 0 else ()
        out = np.zeros(self.V)
        for k in range(1, self.V):
            out[k] = self.tb.log10(h, self.word(k)) * LN10
        return out

    def get_log_prob(self, x, hist=None):
        hist = (hist or ()) + (self.word(int(x.reshape(-1)[0])),)
        return torch.tensor(self.row(hist)).reshape(1, 1, -1), hist


def ngram_rows_dense(t, state):
    """The dense-chain row construction of ngram_slot_rows_kernel, in numpy over NGramLM.tables() ``t``: ln P(. | state)
    for every label, fp32 (label without a word: 0)."""
    chain, c, s = [], [], state
    acc = 0.0
    while True:
        chain.append(s)
        c.append(acc)
        if s == 0:
            break
        acc += float(t["bow"][s])
        s = int(t["back"][s])
    wrow = c[-1] + t["root_p"].astype(np.float64)
    for j in range(len(chain) - 2, -1, -1):
        s = chain[j]
        lo, hi = int(t["arc_off"][s]), int(t["arc_off"][s + 1])
        p = t["arc_p"][lo:hi]
        ok = ~np.isnan(p)
        wrow[t["arc_word"][lo:hi][ok]] = c[j] + p[ok].astype(np.float64)
    w = t["tok2word"]
    return np.where(w < 0, 0.0, wrow[np.maximum(w, 0)] * LN10).astype(np.float32)
