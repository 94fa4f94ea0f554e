"""GPU: n-gram sentence scoring (``NGramLM.score``, ``ccb_ngram_score``) bit for bit against ``Replay``, the kernel's
numpy restatement, and within 1 fp32 ulp of the textbook sum; both launch layouts, invariances, NaN rows, CPU inputs,
``MultiLM.score`` and ``rescore_nbest`` on real beam-search outputs."""
import numpy as np
import pytest
import torch

import ctc_crf
from cat_b200 import _C
from cat_b200.ngram import NGramLM, make_random_arpa
from cat_b200.rescore import rescore_nbest
from cat_b200.rnnt_decode import MultiLM, rnnt_beam_search
from rnnt_decode_oracle import LSTMPredictor
from rnnt_fusion_oracle import JointNet, LSTMLM
from test_ngram_dispatch import Textbook, cat_labels
from test_ngram_score_dispatch import FakeLM, Replay, cat_rescore, cat_string, textbook_score

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _lm(tmp_path, V, order, seed=0, counts=None, **kw):
    path = make_random_arpa(str(tmp_path / f"lm{order}_{V}_{seed}.arpa"), V, order, counts or [4 * V] * (order - 1),
                            seed=seed, **kw)
    labels = cat_labels(V)
    return path, labels, NGramLM(path, labels)


def _batch(V, R, U, seed, lm_rows=None):
    """R rows of width U: token 0 first, random tokens (some 0) after it, lengths in [1, U]."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, V, (R, U), generator=g)
    ids[:, 0] = 0
    ids[torch.rand((R, U), generator=g) < 0.02] = 0
    lens = torch.randint(1, U + 1, (R,), generator=g)
    return ids, lens


def _check_rows(rp, tb, labels, ids, tg, lens, got, rows):
    for b in rows:
        L = int(lens[b])
        want = rp.score(ids[b].numpy(), int(tg[b, -1]), L)
        assert got[b].view(torch.int32) == torch.tensor(float(want)).float().view(torch.int32), (b, float(got[b]), want)
        t = np.float32(textbook_score(tb, cat_string(ids[b].numpy(), int(tg[b, -1]), L, labels)))
        assert abs(float(got[b]) - float(t)) <= float(np.spacing(np.abs(t))), (b, float(got[b]), t)


@pytest.mark.parametrize("order", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("R", [1, 1000, 100000])
def test_matches_replay_and_textbook(tmp_path, order, dtype, R):
    V, U = 60, 24
    path, labels, lm = _lm(tmp_path, V, order, seed=order, pruned_prefixes=0.3)
    rp, tb = Replay(lm, path, labels), Textbook(path, labels)
    ids, lens = _batch(V, R, U, seed=R + order)
    tg = torch.zeros((R, U), dtype=torch.int64)
    got = lm.score(ids.to(DEV, dtype), tg.to(DEV, dtype), lens.to(DEV, dtype)).cpu()
    rows = range(R) if R <= 1000 else np.random.default_rng(0).choice(R, 1500, replace=False)
    _check_rows(rp, tb, labels, ids, tg, lens, got, rows)


@pytest.mark.parametrize("U", [1, 255, 256, 4096, 8192])
def test_edge_lengths_and_both_layouts(tmp_path, U):
    V = 40
    path, labels, lm = _lm(tmp_path, V, 4, seed=U)
    rp, tb = Replay(lm, path, labels), Textbook(path, labels)
    R = 6
    ids, lens = _batch(V, R, U, seed=U)
    lens[0] = U
    lens[1] = 1
    tg = torch.zeros((R, 1), dtype=torch.int64)
    got = lm.score(ids.to(DEV), tg.to(DEV), lens.to(DEV)).cpu()
    _check_rows(rp, tb, labels, ids, tg, lens, got, range(R))
    # U = 1: <s> and </s> only, with input_lengths None
    if U == 1:
        full = lm.score(ids.to(DEV), tg.to(DEV)).cpu()
        assert torch.equal(full, got)


def test_invariances(tmp_path):
    V, R, U = 50, 3000, 40
    path, labels, lm = _lm(tmp_path, V, 5, seed=11)
    ids, lens = _batch(V, R, U, seed=5)
    tg = torch.zeros((R, U), dtype=torch.int64)
    d_ids, d_tg, d_lens = ids.to(DEV), tg.to(DEV), lens.to(DEV)
    a = lm.score(d_ids, d_tg, d_lens)
    # two runs, and out-of-range padding past each length
    pad = d_ids.clone()
    pad[torch.arange(U, device=DEV)[None, :] >= d_lens[:, None]] = 10 ** 9
    assert torch.equal(a, lm.score(d_ids, d_tg, d_lens)) and torch.equal(a, lm.score(pad, d_tg, d_lens))
    # a row alone, or in a batch scored by the CTA layout (U >= 256), equals the row in the batch
    wide = torch.zeros((R, 300), dtype=torch.int64, device=DEV)
    wide[:, :U] = d_ids
    assert torch.equal(a, lm.score(wide, d_tg, d_lens))
    for b in (0, 17, R - 1):
        L = int(lens[b])
        assert torch.equal(a[b:b + 1], lm.score(d_ids[b:b + 1, :L], d_tg[b:b + 1], None))
    # a side stream
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = lm.score(d_ids, d_tg, d_lens)
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(a, b)
    # no host synchronisation, and one launch per call whatever R and U are
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for x in (d_ids, wide, d_ids[:1]):
            n0 = _C.launch_count()
            lm.score(x, d_tg[:x.shape[0]], d_lens[:x.shape[0]])
            assert _C.launch_count() == n0 + 1
        n0 = _C.launch_count()
        lm.score(d_ids, d_tg, lens.int())          # host lengths staged without a synchronisation
        assert _C.launch_count() == n0 + 1
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_bad_device_values_give_nan_for_that_row_only(tmp_path):
    V, R, U = 30, 8, 12
    path, labels, lm = _lm(tmp_path, V, 3, seed=2)
    ids, lens = _batch(V, R, U, seed=9)
    tg = torch.zeros((R, 1), dtype=torch.int64)
    good = lm.score(ids.to(DEV), tg.to(DEV), lens.to(DEV)).cpu()
    ids2, lens2, tg2 = ids.clone(), lens.clone(), tg.clone()
    ids2[1, 0] = V
    ids2[2, int(lens[2]) - 1] = -3
    lens2[3] = 0
    lens2[4] = U + 1
    tg2[5, -1] = V + 7
    got = lm.score(ids2.to(DEV), tg2.to(DEV), lens2.to(DEV)).cpu()
    bad = torch.zeros(R, dtype=torch.bool)
    bad[1:6] = True
    assert bool(got[bad].isnan().all()) and torch.equal(got[~bad], good[~bad])


def test_cpu_inputs_return_cpu_result(tmp_path):
    V, R, U = 30, 50, 10
    path, labels, lm = _lm(tmp_path, V, 3, seed=4)
    ids, lens = _batch(V, R, U, seed=1)
    tg = torch.zeros((R, U), dtype=torch.int64)
    got = lm.score(ids, tg, lens)
    assert got.device.type == "cpu" and torch.equal(got, lm.score(ids.to(DEV), tg.to(DEV), lens).cpu())


def test_lms_alternated_and_replaced(tmp_path):
    V, R, U = 40, 200, 16
    ids, lens = _batch(V, R, U, seed=3)
    tg = torch.zeros((R, 1), dtype=torch.int64)
    x = (ids.to(DEV), tg.to(DEV), lens.to(DEV))
    pa, la, a = _lm(tmp_path, V, 3, seed=21)
    pb, lb, b = _lm(tmp_path, V, 4, seed=22)
    ra, rb = Replay(a, pa, la), Replay(b, pb, lb)
    for lm, rp in ((a, ra), (b, rb), (a, ra), (b, rb)):
        got = lm.score(*x).cpu()
        assert all(float(got[i]) == float(rp.score(ids[i].numpy(), 0, int(lens[i]))) for i in range(0, R, 7))
    del a
    torch.cuda.synchronize()
    pc, lc, c = _lm(tmp_path, V, 2, seed=23)
    rc = Replay(c, pc, lc)
    got = c.score(*x).cpu()
    assert all(float(got[i]) == float(rc.score(ids[i].numpy(), 0, int(lens[i]))) for i in range(0, R, 7))


def _cat_abs_score(lm, input_ids, targets, input_lengths):
    """CAT's AbsDecoder.score restated (a unidirectional LSTM's outputs at valid positions do not depend on the lengths)."""
    logits, _ = lm(input_ids)
    lp = logits.log_softmax(-1).gather(index=targets.long().unsqueeze(2), dim=-1).squeeze(-1)
    mask = torch.arange(input_ids.size(1), device=input_ids.device)[None, :] < input_lengths[:, None].to(input_ids.device)
    return (lp * mask).sum(dim=1)


class _ScoredLSTM(LSTMLM):
    def score(self, input_ids, targets, input_lengths=None):
        return _cat_abs_score(self, input_ids, targets, input_lengths)


def test_multilm_score_is_weighted_sum(tmp_path):
    V, R, U = 30, 64, 12
    pa, la, a = _lm(tmp_path, V, 5, seed=31)
    pb, lb, b = _lm(tmp_path, V, 2, seed=32)
    torch.manual_seed(0)
    nn_lm = _ScoredLSTM(V, 16).to(DEV).eval()
    ids, lens = _batch(V, R, U, seed=8)
    tg = torch.roll(ids, -1, dims=1)
    x = (ids.to(DEV), tg.to(DEV), lens.to(DEV))
    w = [0.28125, -0.3125, 0.5]
    mix = MultiLM(w, [a, b, nn_lm])
    with torch.no_grad():
        got = mix.score(*x)
        parts = [a.score(*x), b.score(*x), nn_lm.score(*x)]
    want = (w[0] * parts[0].double() + w[1] * parts[1].double() + w[2] * parts[2].double()).float()
    assert torch.equal(got, want)


def test_rescore_nbest_on_beam_search_outputs(tmp_path):
    V, N, T, H, B = 30, 6, 20, 16, 8
    path, labels, lm = _lm(tmp_path, V, 3, seed=41)
    tb = Textbook(path, labels)
    torch.manual_seed(1)
    pred, joiner = LSTMPredictor(V, H).to(DEV).eval(), JointNet(H, H, V, H).to(DEV).eval()
    enc = torch.randn(N, T, H, device=DEV)
    flen = torch.tensor([T, T - 3, 11, 5, 2, 1], device=DEV)
    with torch.no_grad():
        outs = [rnnt_beam_search(enc, flen, pred, joiner, B)]
    y = torch.randn(N, T, V, device=DEV).log_softmax(-1)
    outs.append(ctc_crf.ctc_beam_search(y, flen.int().cpu(), B, V))
    for out in outs:
        tokens, lengths, scores = out[0], out[1], out[-1]
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            lm_s, total, best = rescore_nbest(tokens, lengths, scores, lm, 0.4, 0.7)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ref = rescore_nbest(tokens.cpu(), lengths.cpu(), scores.cpu(), FakeLM(tb, labels), 0.4, 0.7)
        assert torch.allclose(lm_s.cpu(), ref[0], rtol=3e-7, atol=0)
        for n in range(N):
            k = int((lengths[n] >= 0).sum())
            texts = [tokens[n, j, :int(lengths[n, j])].tolist() for j in range(k)]
            final, keep = cat_rescore(texts, scores[n, :k].cpu(), lm_s[n, :k].cpu(), 0.4, 0.7)
            assert torch.equal(total[n, :k].cpu(), final) and int(best[n]) == keep


def test_bench_aishell_shape_sample(tmp_path):
    V = 4232
    path, labels, lm = _lm(tmp_path, V, 5, seed=5, counts=[200000] * 4)
    rp, tb = Replay(lm, path, labels), Textbook(path, labels)
    R, U = 7176 * 16, 31
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(1, V, (R, U), generator=g)
    ids[:, 0] = 0
    lens = torch.randint(9, U + 1, (R,), generator=g)
    tg = torch.zeros((R, 1), dtype=torch.int64)
    got = lm.score(ids.to(DEV), tg.to(DEV), lens.to(DEV)).cpu()
    _check_rows(rp, tb, labels, ids, tg, lens, got, np.random.default_rng(1).choice(R, 300, replace=False))
