"""GPU: the RNN-T beam search with an LM mix (``cat_b200.rnnt_decode.MultiLM``, LODR decoding): the mix rows kernel frame
by frame against ``ccb_ngram_slot_rows`` run alone and the numpy restatement (tests/multilm_oracle.py), bit for bit; a
one-member mix against today's single-LM fusion, bit for bit; and ``RNNTDecoder`` end to end against CAT's decoder with
``CatMultiDecoder`` (tests/rnnt_fusion_oracle.py ``cat_decode_fused``)."""
import ctypes as C

import numpy as np
import pytest
import torch

from cat_b200 import _lib
from cat_b200.ngram import NGramLM, make_random_arpa
from cat_b200.rnnt_decode import MultiLM, RNNTDecoder, rnnt_beam_search
from multilm_oracle import CatMultiDecoder, mix_rows
from rnnt_decode_oracle import LSTMPredictor
from rnnt_fusion_oracle import CatNGram, JointNet, LSTMLM, cat_decode_fused

pytestmark = pytest.mark.gpu

_DT = {"fp32": (torch.float32, 0), "bf16": (torch.bfloat16, 1), "fp16": (torch.float16, 2)}
LODR = (0.28125, -0.3125)   # CAT's aishell rnnt-v1 "5gram char + LODR" weights: elm, then the bigram's (ilm) weight


@pytest.fixture(autouse=True)
def _fp32_networks():
    # the search and the restatement run the networks at different batch sizes; TF32 would make their rows differ by ~1e-3
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    torch.cuda.empty_cache()


def _labels(V):
    return ["<blk>", "<unk>"] + [str(i) for i in range(2, V)]


def _arr(t, xs):
    return (t * max(len(xs), 1))(*xs)


# ---- mix rows, frame by frame ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dname", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("N, B, V", [(3, 5, 40), (2, 16, 300), (1, 128, 300), (2, 16, 4232)])
def test_mix_rows_and_states_match_slot_rows_and_restatement(tmp_path, dname, N, B, V):
    # members in the order n-gram, neural, n-gram, neural: the kernel's member order and each member's place are checked
    dt, code = _DT[dname]
    labels = _labels(V)
    counts = {40: [120, 150, 150, 150], 300: [900, 900, 900, 900], 4232: [20000] * 4}[V]
    lms = [NGramLM(make_random_arpa(str(tmp_path / "a.arpa"), V, 5, counts, seed=V, pruned_prefixes=0.3), labels),
           NGramLM(make_random_arpa(str(tmp_path / "b.arpa"), V, 2, counts[0], seed=V + 1), labels)]
    weights = [0.28125, 0.7, -0.3125, -1.3]   # (n-gram 0, neural 0, n-gram 1, neural 1)
    order = [0, 2, 1, 3]                      # the entry's list: n-grams first, then neural
    L = _lib.lib()
    dev = torch.device("cuda")
    R = N * B
    mix_st = [[torch.full((N, B), -7, dtype=torch.int32, device=dev) for _ in range(2)] for _ in lms]
    one_st = [[torch.full((N, B), -9, dtype=torch.int32, device=dev) for _ in range(2)] for _ in lms]
    one_rows = [torch.full((R, V), float("nan"), device=dev) for _ in lms]
    out = torch.full((R, V), float("nan"), device=dev)
    rng = np.random.default_rng(V + B)
    for step in range(8):
        neural = []
        for j in range(2):   # neural rows with -inf entries and values of both signs
            z = rng.standard_normal((R, V)) * 3
            z[rng.random((R, V)) < 0.02] = -np.inf
            neural.append(torch.tensor(z, dtype=torch.float32).to(dt).to(dev).contiguous())
        if step == 0:
            par_d = tok_d = None
        else:
            par = rng.integers(0, B, (N, B))
            tok = np.where(rng.random((N, B)) < 0.3, -1, rng.integers(1, V, (N, B)))
            par_d = torch.tensor(par, dtype=torch.int32, device=dev)
            tok_d = torch.tensor(tok, dtype=torch.int32, device=dev)
        pp = None if par_d is None else par_d.data_ptr()
        tp = None if tok_d is None else tok_d.data_ptr()
        for lm, st, rows in zip(lms, one_st, one_rows):
            rc = L.ccb_ngram_slot_rows(lm.handle, N, B, V, pp, tp, None if pp is None else st[0].data_ptr(),
                                       st[1].data_ptr(), rows.data_ptr(), None)
            assert rc == 0, _lib.last_error()
            st.reverse()
        rc = L.ccb_lm_mix_slot_rows(
            2, _arr(C.c_void_p, [lm.handle for lm in lms]), _arr(C.c_double, [weights[0], weights[2]]),
            _arr(C.c_void_p, [s[0].data_ptr() for s in mix_st]), _arr(C.c_void_p, [s[1].data_ptr() for s in mix_st]),
            2, _arr(C.c_void_p, [r.data_ptr() for r in neural]), _arr(C.c_int, [code, code]),
            _arr(C.c_double, [weights[1], weights[3]]), _arr(C.c_int, order), N, B, V, pp, tp, out.data_ptr(), None)
        assert rc == 0, _lib.last_error()
        for s in mix_st:
            s.reverse()
        for a, b in zip(mix_st, one_st):
            assert torch.equal(a[0], b[0]), step
        members = [one_rows[0], neural[0], one_rows[1], neural[1]]
        ref = mix_rows([m.float().cpu().numpy() for m in members], weights)
        got = out.cpu().numpy()
        assert np.array_equal(got.view(np.int32), ref.view(np.int32)), step


# ---- one member is the single-LM fusion ----------------------------------------------------------------------------------
def _build(V, H=32, mode="add", seed=0):
    torch.manual_seed(seed)
    pred = LSTMPredictor(V, H)
    joiner = JointNet(H, H, V, H, mode)
    for m in (pred, joiner):
        for p in m.parameters():
            p.data.mul_(3.0)
    return pred.cuda().eval(), joiner.cuda().eval()


def _lstm_lm(V, seed=4):
    torch.manual_seed(seed)
    lm = LSTMLM(V, 24)
    for p in lm.parameters():
        p.data.mul_(2.0)
    return lm.cuda().eval()


def _ngram(tmp_path, V, order, counts=None):
    path = make_random_arpa(str(tmp_path / f"lm{order}.arpa"), V, order, counts or [4 * V] * (order - 1), seed=order)
    return NGramLM(path, _labels(V)), CatNGram(path, _labels(V))


@pytest.mark.parametrize("kind", ["ngram", "lstm"])
@pytest.mark.parametrize("ilm_weight", [0.0, -0.3125])
def test_one_member_mix_is_the_single_lm_fusion(tmp_path, kind, ilm_weight):
    V = 37
    pred, joiner = _build(V)
    lm = _ngram(tmp_path, V, 4)[0] if kind == "ngram" else _lstm_lm(V)
    enc = torch.randn(4, 10, 32, device="cuda")
    lens = torch.tensor([10, 6, 0, 9])
    kw = dict(alpha=0.6, beta=0.4, ilm_weight=ilm_weight)
    for B in (1, 4, 16):
        a = rnnt_beam_search(enc, lens, pred, joiner, beam_size=B, lm=lm, **kw)
        b = rnnt_beam_search(enc, lens, pred, joiner, beam_size=B, lm=MultiLM([1.0], [lm]), **kw)
        for x, y in zip(a, b):
            assert torch.equal(x, y)


# ---- end to end against CAT's decoder ------------------------------------------------------------------------------------
_MIXES = {"5gram+2gram": ("ngram5", "ngram2"), "3gram+2gram": ("ngram3", "ngram2"), "lstm+2gram": ("lstm", "ngram2")}


def _mix(tmp_path, V, kinds):
    gpu, ref = [], []
    for k in kinds:
        if k == "lstm":
            m = _lstm_lm(V)
            gpu.append(m)
            ref.append(m)
        else:
            g, r = _ngram(tmp_path, V, int(k[-1]))
            gpu.append(g)
            ref.append(r)
    return gpu, ref


def _compare(got, ref, tol=1e-4):
    assert len(got) == len(ref)
    for (gh, gs), (rh, rs) in zip(got, ref):
        assert gh == rh
        for a, b in zip(gs, rs):
            assert abs(a - b) <= tol * (1 + abs(b)), (a, b)


@pytest.mark.parametrize("mix, w", [("5gram+2gram", 0.0), ("3gram+2gram", 0.0), ("lstm+2gram", 0.0),
                                    ("5gram+2gram", -0.3125)])
@pytest.mark.parametrize("mode", ["add", "cat"])
@pytest.mark.parametrize("B", [1, 4, 16])
def test_decoder_matches_cat_restatement(tmp_path, mix, w, mode, B):
    V = 29
    pred, joiner = _build(V, mode=mode)
    gpu, ref = _mix(tmp_path, V, _MIXES[mix])
    weights = [1.0, -0.3125] if mix.startswith("lstm") else [0.28125 * 3, -0.3125 * 2]
    torch.manual_seed(5)
    enc = torch.randn(5, 9, 32, device="cuda")
    lens = torch.tensor([9, 1, 0, 6, 9])
    dec = RNNTDecoder(pred, joiner, beam_size=B, lm_module=MultiLM(weights, gpu), alpha=0.9, beta=0.5, est_ilm=w != 0,
                      ilm_weight=w)
    got = dec(enc, lens)
    refd = cat_decode_fused(enc, lens, pred, joiner, B, lm=CatMultiDecoder(weights, ref), alpha=0.9, beta=0.5,
                            ilm_weight=w)
    _compare(got, refd)
    assert got[2] == ([[]], [0.0])


def test_aishell_lodr(tmp_path):
    # CAT's aishell "5gram char + LODR" configuration: the 5-gram with elm 0.28125, the pruned bigram with -0.3125
    V, H = 4232, 512
    torch.manual_seed(0)
    pred = LSTMPredictor(V, H).cuda().eval()
    joiner = JointNet(H, H, V, H).cuda().eval()
    for p in joiner.fc.parameters():
        p.data.mul_(4.0)
    g5, r5 = _ngram(tmp_path, V, 5, [8000] * 4)
    g2, r2 = _ngram(tmp_path, V, 2, [20000])
    enc = torch.randn(2, 8, H, device="cuda")
    lens = torch.tensor([8, 5])
    got = RNNTDecoder(pred, joiner, beam_size=16, lm_module=MultiLM(list(LODR), [g5, g2]), alpha=1.0, beta=0.5)(enc, lens)
    _compare(got, cat_decode_fused(enc, lens, pred, joiner, 16, lm=CatMultiDecoder(list(LODR), [r5, r2]), alpha=1.0,
                                   beta=0.5))


def test_cat_multidecoder_is_multilm(tmp_path):
    V = 31
    pred, joiner = _build(V)
    a, b = _lstm_lm(V, 4), _lstm_lm(V, 5)
    enc = torch.randn(3, 8, 32, device="cuda")
    lens = torch.tensor([8, 5, 7])
    kw = dict(beam_size=8, alpha=0.5, beta=0.2, est_ilm=True, ilm_weight=-0.2)
    x = RNNTDecoder(pred, joiner, lm_module=CatMultiDecoder([0.6, 0.0, -0.4], [a, _lstm_lm(V, 6), b]), **kw)(enc, lens)
    y = RNNTDecoder(pred, joiner, lm_module=MultiLM([0.6, -0.4], [a, b]), **kw)(enc, lens)
    assert x == y


# ---- properties ---------------------------------------------------------------------------------------------------------
def _lodr_kw(tmp_path, V, kind="ngram"):
    first = _ngram(tmp_path, V, 4)[0] if kind == "ngram" else _lstm_lm(V)
    return dict(lm=MultiLM([0.8, -0.3125], [first, _ngram(tmp_path, V, 2)[0]]), alpha=0.5, beta=0.3, ilm_weight=-0.25)


@pytest.mark.parametrize("kind", ["ngram", "lstm"])
def test_fp16_autocast(tmp_path, kind):
    V = 31
    pred, joiner = _build(V)
    first = _ngram(tmp_path, V, 3) if kind == "ngram" else (_lstm_lm(V),) * 2
    g2, r2 = _ngram(tmp_path, V, 2)
    enc = torch.randn(3, 8, 32, device="cuda")
    lens = torch.tensor([8, 5, 2])
    with torch.autocast("cuda", dtype=torch.float16):
        got = RNNTDecoder(pred, joiner, beam_size=4, lm_module=MultiLM([0.9, -0.3], [first[0], g2]), alpha=0.4, beta=0.2,
                          est_ilm=True, ilm_weight=-0.3)(enc, lens)
        ref = cat_decode_fused(enc, lens, pred, joiner, 4, lm=CatMultiDecoder([0.9, -0.3], [first[1], r2]), alpha=0.4,
                               beta=0.2, ilm_weight=-0.3)
    _compare(got, ref, 1e-3)


@pytest.mark.parametrize("kind", ["ngram", "lstm"])
def test_device_lengths_nan_past_the_end_and_repeat_bits(tmp_path, kind):
    V = 19
    pred, joiner = _build(V)
    kw = _lodr_kw(tmp_path, V, kind)
    enc = torch.randn(3, 8, 32, device="cuda")
    lens = torch.tensor([8, 4, 6])
    a = rnnt_beam_search(enc, lens, pred, joiner, beam_size=4, **kw)
    enc2 = enc.clone()
    enc2[1, 4:] = float("nan")
    enc2[2, 6:] = float("nan")
    b = rnnt_beam_search(enc2, lens.cuda(), pred, joiner, beam_size=4, **kw)
    c = rnnt_beam_search(enc, lens, pred, joiner, beam_size=4, **kw)
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_side_stream(tmp_path):
    V = 19
    pred, joiner = _build(V)
    kw = _lodr_kw(tmp_path, V, "lstm")
    enc = torch.randn(2, 6, 32, device="cuda")
    lens = torch.tensor([6, 3])
    a = rnnt_beam_search(enc, lens, pred, joiner, beam_size=4, **kw)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = rnnt_beam_search(enc, lens, pred, joiner, beam_size=4, **kw)
    torch.cuda.current_stream().wait_stream(s)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("kind", ["ngram", "lstm"])
def test_no_host_synchronisation(tmp_path, kind):
    V = 19
    pred, joiner = _build(V)
    kw = _lodr_kw(tmp_path, V, kind)
    enc = torch.randn(2, 6, 32, device="cuda")
    for lens in (torch.tensor([6, 2]), torch.tensor([6, 2], device="cuda")):
        rnnt_beam_search(enc, lens, pred, joiner, beam_size=4, **kw)   # warm-up (uploads the LMs)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            rnnt_beam_search(enc, lens, pred, joiner, beam_size=4, **kw)
        finally:
            torch.cuda.set_sync_debug_mode(0)
