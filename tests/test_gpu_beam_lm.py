"""``ctc_crf.ctc_beam_search(..., lm=NGramLM(...))`` on the GPU: hypotheses, timesteps and scores against the numpy
restatement ``beam_lm_ref`` (tests/test_ngram_dispatch.py), the search without an LM at zero weights, exactness at full beam,
the invariances (dtypes, raw logits, padding, scratch contents, synchronisation, streams, launches), LM lifetimes, the
``CTCBeamDecoder`` with CAT's LM arguments and the headline shape."""
import numpy as np
import pytest
import torch

from cat_b200 import _C
from cat_b200.ngram import NGramLM, make_random_arpa
from test_beam_dispatch import enum_plain, hyps
from test_gpu_beam import _batch, _compare, _same
from test_ngram_dispatch import Textbook, beam_lm_ref, cat_labels

pytestmark = pytest.mark.gpu

V = 218
WEIGHTS = [(0.25, -0.5), (1.0, 0.0), (1.7, 1.0), (0.5, 2.0)]


def _search(y, lens, B, cut, lm=None, alpha=1.0, beta=0.0, dtype=torch.float32):
    import ctc_crf
    logits = (y if isinstance(y, torch.Tensor) else torch.as_tensor(np.asarray(y))).to(device="cuda", dtype=dtype)
    out = ctc_crf.ctc_beam_search(logits, torch.as_tensor(np.asarray(lens), dtype=torch.int32), B, cut, lm=lm, alpha=alpha,
                                  beta=beta)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


@pytest.fixture(scope="module")
def lms(tmp_path_factory):
    """Token LMs over V = 218 labels in CAT's convention: a 2-gram and a 4-gram with pruned prefixes and missing suffixes."""
    d = tmp_path_factory.mktemp("lm")
    p2 = make_random_arpa(str(d / "lm2.arpa"), V, 2, 6000, seed=1)
    p4 = make_random_arpa(str(d / "lm4.arpa"), V, 4, [8000, 8000, 6000], seed=2, pruned_prefixes=0.3, missing_suffixes=True)
    return {2: NGramLM(p2, cat_labels(V)), 4: NGramLM(p4, cat_labels(V))}


# ---------------------------------------------------------------------------------------------------------------------
# 1. kernel against the restatement
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [2, 4])
@pytest.mark.parametrize("cut", [40, 218])
@pytest.mark.parametrize("B", [1, 4, 16, 128])
def test_kernel_equals_restatement(lms, order, cut, B):
    alpha, beta = WEIGHTS[(B + cut + order) % len(WEIGHTS)]
    y, lens = _batch(3, 24 if B < 128 else 12, V, seed=B + cut + order)
    _compare(_search(y, lens, B, cut, lms[order], alpha, beta), beam_lm_ref(y, lens, B, cut, lms[order], alpha, beta),
             min_frac=0.6)


@pytest.mark.parametrize("N", [1, 64, 130])
def test_batch_sizes(lms, N):
    y, lens = _batch(N, 16, V, seed=N)
    for order, (alpha, beta) in ((2, WEIGHTS[0]), (4, WEIGHTS[2])):
        _compare(_search(y, lens, 16, 40, lms[order], alpha, beta), beam_lm_ref(y, lens, 16, 40, lms[order], alpha, beta))


def test_zero_weights_give_the_search_without_lm_bit_for_bit(lms):
    y, lens = _batch(9, 40, V, seed=7, lens=[40, 37, 29, 20, 11, 5, 2, 1, 0])
    for B, cut in ((1, 40), (16, 40), (128, 218)):
        plain = _search(y, lens, B, cut)
        for order in (2, 4):
            assert _same(_search(y, lens, B, cut, lms[order], 0.0, 0.0), plain), (B, cut, order)


def test_full_beam_is_exact(tmp_path):
    T, Vs = 4, 4                       # at most 1 + 3 + 9 + 27 + 81 = 121 prefixes: nothing is pruned at B = 128
    y, _ = _batch(3, T, Vs, seed=9)
    lens = np.full(3, T, np.int32)
    for order in (1, 2, 3):
        path = make_random_arpa(str(tmp_path / f"t{order}.arpa"), Vs, order, [6, 10][:order - 1], seed=order,
                                pruned_prefixes=0.3)
        lm, tb = NGramLM(path, cat_labels(Vs)), Textbook(path, cat_labels(Vs))
        for alpha, beta in ((0.5, -0.5), (1.7, 1.0)):
            tk, ln, ts, sc = _search(y, lens, 128, Vs, lm, alpha, beta)
            for n in range(3):
                want = {k: v + alpha * tb.ln_seq(k)[0] + beta * len(k) for k, v in enum_plain(y[n], T).items()}
                got = hyps(tk, ln, sc, n)
                assert set(got) == set(want), (order, alpha)
                for k, v in want.items():
                    assert abs(got[k] - v) <= 1e-5 * max(1, abs(v)), (order, alpha, k)


# ---------------------------------------------------------------------------------------------------------------------
# 2. invariances
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def mid(lms):
    y, lens = _batch(9, 40, V, seed=7, lens=[40, 37, 29, 20, 11, 5, 2, 1, 0])
    return lms[4], y, lens


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_half_logits_equal_their_upcast(mid, dtype):
    lm, y, lens = mid
    yh = torch.tensor(y).to(dtype)
    assert _same(_search(yh, lens, 16, 40, lm, 0.25, -0.5, dtype), _search(yh.float(), lens, 16, 40, lm, 0.25, -0.5))


def test_raw_logits_give_the_same_hypotheses(mid):
    lm, y, lens = mid
    z = (y + np.random.default_rng(1).standard_normal((y.shape[0], y.shape[1], 1)) * 5).astype(np.float32)
    zl = torch.log_softmax(torch.tensor(z), -1).numpy()
    a, b = _search(z, lens, 16, 40, lm, 0.25, -0.5), _search(zl, lens, 16, 40, lm, 0.25, -0.5)
    ra, rb = beam_lm_ref(z, lens, 16, 40, lm, 0.25, -0.5), beam_lm_ref(zl, lens, 16, 40, lm, 0.25, -0.5)
    shift = np.array([np.logaddexp.reduce(z[n, :lens[n]].astype(np.float64), -1).sum() for n in range(len(lens))])
    ok = ~(ra[4] | rb[4])
    assert ok.sum() >= 0.9 * len(lens)
    for n in np.nonzero(ok)[0]:
        assert np.array_equal(a[0][n], b[0][n]) and np.array_equal(a[1][n], b[1][n]), n
        fin = a[1][n] >= 0
        np.testing.assert_allclose(a[3][n][fin] - shift[n], b[3][n][fin], rtol=1e-5, atol=1e-3)


def test_padding_is_never_read(mid):
    lm, y, lens = mid
    ref = _search(y, lens, 16, 40, lm, 0.25, -0.5)
    for v in (np.nan, np.inf, -np.inf):
        y2 = y.copy()
        for n, l in enumerate(lens):
            y2[n, l:] = v
        assert _same(_search(y2, lens, 16, 40, lm, 0.25, -0.5), ref), v


@pytest.mark.parametrize("byte", [0x00, 0xFF, 0x7F])
def test_scratch_contents_change_nothing(mid, monkeypatch, byte):
    from test_scratch_proxy import ScratchProxy
    lm, y, lens = mid
    clean = _search(y, lens, 16, 40, lm, 0.25, -0.5)
    proxy = ScratchProxy(byte)
    monkeypatch.setattr(_C, "torch", proxy)
    assert _same(_search(y, lens, 16, 40, lm, 0.25, -0.5), clean), byte
    L = _C._lib.lib()
    assert any(b == int(L.ccb_ctc_beam_search_ws_bytes(len(lens), y.shape[1], 16)) for b, _, d in proxy.record)


def test_no_host_synchronisation(mid):
    import ctc_crf
    lm, y, lens = mid
    logits = torch.tensor(y, device="cuda")
    lx = torch.tensor(lens)
    ctc_crf.ctc_beam_search(logits, lx, 16, 40, lm=lm)      # warm-up: the first call on a device uploads the LM's tables
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = ctc_crf.ctc_beam_search(logits, lx, 16, 40, lm=lm, alpha=0.25, beta=-0.5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(t.is_cuda for t in out)


def test_side_stream(mid):
    import ctc_crf
    lm, y, lens = mid
    ref = _search(y, lens, 16, 40, lm, 0.25, -0.5)
    s = torch.cuda.Stream()
    logits = torch.tensor(y, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out = ctc_crf.ctc_beam_search(logits, torch.tensor(lens), 16, 40, lm=lm, alpha=0.25, beta=-0.5)
    s.synchronize()
    assert _same([t.cpu().numpy() for t in out], ref)


def test_launch_count_does_not_depend_on_beam(mid):
    lm, y, lens = mid
    counts = []
    for B in (1, 16, 128):
        k0 = _C.launch_count()
        _search(y, lens, B, 40, lm, 0.25, -0.5)
        counts.append(_C.launch_count() - k0)
    assert counts == [1, 1, 1], counts


# ---------------------------------------------------------------------------------------------------------------------
# 3. LM lifetimes
# ---------------------------------------------------------------------------------------------------------------------
def test_two_lms_alternate_and_a_destroyed_one_can_be_replaced(tmp_path):
    y, lens = _batch(5, 30, V, seed=11)
    paths = [make_random_arpa(str(tmp_path / f"lm{i}.arpa"), V, 3, [3000, 3000], seed=20 + i) for i in range(2)]
    a, b = NGramLM(paths[0], cat_labels(V)), NGramLM(paths[1], cat_labels(V))
    ra, rb = _search(y, lens, 16, 40, a, 1.0, 0.5), _search(y, lens, 16, 40, b, 1.0, 0.5)
    assert not _same(ra[:4], rb[:4])
    for _ in range(2):
        assert _same(_search(y, lens, 16, 40, a, 1.0, 0.5), ra) and _same(_search(y, lens, 16, 40, b, 1.0, 0.5), rb)
    del a
    c = NGramLM(paths[0], cat_labels(V))
    assert _same(_search(y, lens, 16, 40, c, 1.0, 0.5), ra) and _same(_search(y, lens, 16, 40, b, 1.0, 0.5), rb)
    _compare(ra, beam_lm_ref(y, lens, 16, 40, c, 1.0, 0.5))


# ---------------------------------------------------------------------------------------------------------------------
# 4. the ctcdecode drop-in with CAT's LM arguments (cat/ctc/decode.py)
# ---------------------------------------------------------------------------------------------------------------------
def test_decoder_with_cat_lm_arguments(tmp_path):
    import ctc_crf
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, 3, [4000, 4000], seed=5)
    labels = cat_labels(V)
    dec = ctc_crf.CTCBeamDecoder(labels=labels, model_path=path, alpha=0.25, beta=-0.5, cutoff_top_n=40, beam_width=32,
                                 num_processes=6, log_probs_input=True, is_token_based=True)
    y, lens = _batch(6, 50, V, seed=3)
    lm = NGramLM(path, labels)
    want = [t.cpu() for t in ctc_crf.ctc_beam_search(torch.tensor(y, device="cuda"), torch.tensor(lens), 32, 40, lm=lm,
                                                     alpha=0.25, beta=-0.5)]
    for logits in (torch.tensor(y), torch.tensor(y, device="cuda")):
        results, scores, timesteps, out_lens = dec.decode(logits, torch.tensor(lens))
        assert results.is_cuda
        assert torch.equal(results.cpu(), want[0]) and torch.equal(out_lens.cpu(), want[1])
        assert torch.equal(timesteps.cpu(), want[2]) and torch.equal(scores.cpu(), -want[3])


# ---------------------------------------------------------------------------------------------------------------------
# 5. the headline shape
# ---------------------------------------------------------------------------------------------------------------------
def test_headline_shape(tmp_path):
    from oracle import oracle
    lm = NGramLM(make_random_arpa(str(tmp_path / "hl.arpa"), V, 3, [150000, 150000], seed=1), cat_labels(V))
    N, T = 64, 1500
    lens = np.maximum(200, T - 37 * np.arange(N)).astype(np.int32)
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=21, lens=lens)
    out = _search(y, lens, 16, 40, lm, 0.25, -0.5)
    assert np.all(out[1][:, 0] >= 0)
    sub = [0, 31, 63]                  # the longest, a middle and the shortest utterance
    _compare([o[sub] for o in out], beam_lm_ref(y[sub], lens[sub], 16, 40, lm, 0.25, -0.5), min_frac=0.66)
