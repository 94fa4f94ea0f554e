"""``ctc_crf.fst_decode`` on the GPU: words, alignment and costs against the numpy restatement ``wfst_decode_ref``
(tests/test_wfst_dispatch.py) over beams, max_active, weights, batch sizes and graphs; the invariances (dtypes, raw logits,
padding, poisoned workspace, a side stream, synchronisation, launches, graph lifetimes); and a several-million-arc
``make_tlg`` graph at N = 64, T = 1500."""
import math

import numpy as np
import pytest
import torch

from cat_b200 import _C, _lib, fst
from cat_b200.ngram import make_random_arpa
from cat_b200.wfst import DecodingGraph
from test_wfst_dispatch import GRAPHS, Tables, peaky, random_wfst, tiny_lexicon, wfst_decode_ref, write_graph

pytestmark = pytest.mark.gpu

WEIGHTS = [(1.0, 1.0, 0.0), (0.7, 1.3, -0.4), (1.5, 0.5, 0.8), (0.1, 1.0, 2.0)]
EXACT = ("words", "num_words", "align", "reached_final")
CLOSE = ("ac_logp", "graph_cost", "cost")


def _decode(dg, y, lens, dtype=torch.float32, **kw):
    import ctc_crf
    logits = (y if isinstance(y, torch.Tensor) else torch.as_tensor(np.asarray(y))).to(device="cuda", dtype=dtype)
    out = ctc_crf.fst_decode(logits, torch.as_tensor(np.asarray(lens), dtype=torch.int32), dg, **kw)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out._asdict().items()}


def _compare(got, ref, rows=None):
    rows = range(len(ref["num_words"])) if rows is None else rows
    for n in rows:
        for k in EXACT:
            assert np.array_equal(got[k][n], ref[k][n]), (k, n, got[k][n], ref[k][n])
        for k in CLOSE:
            a, b = float(got[k][n]), float(ref[k][n])
            if math.isinf(b):
                assert a == b, (k, n)
            else:
                assert abs(a - b) <= 1e-6 * max(1.0, abs(b)), (k, n, a, b)


def _same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in a)


@pytest.fixture(scope="module")
def graphs(tmp_path_factory):
    """The random WFSTs of the restatement's tests and a small make_tlg graph (V = 20, 80 words, a 3-gram)."""
    d = tmp_path_factory.mktemp("wfst")
    out = []
    for i, spec in enumerate(GRAPHS):
        dg = DecodingGraph(write_graph(d, f"r{i}.fst", random_wfst(**spec)))
        out.append((dg, Tables(dg), spec["V"] + 1))
    arpa = make_random_arpa(str(d / "w.arpa"), 82, 3, [300, 300], seed=3)
    g, _ = fst.make_tlg(20, tiny_lexicon(20, 80, seed=3), arpa)
    dg = DecodingGraph(write_graph(d, "tlg.fst", g))
    out.append((dg, Tables(dg), 20))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 1. kernel against the restatement
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beam", [4.0, 8.0, 17.0, math.inf])
@pytest.mark.parametrize("K", [1, 16, 1000, 7000])
def test_kernel_equals_restatement(graphs, beam, K):
    for gi, (dg, tb, V) in enumerate(graphs):
        acwt, lmwt, wip = WEIGHTS[(gi + K + int(min(beam, 99))) % len(WEIGHTS)]
        y, lens = peaky(3, 20, V, seed=gi * 7 + K, lens=[20, 11, 1])
        kw = dict(acwt=acwt, lmwt=lmwt, wip=wip, beam=beam, max_active=K)
        _compare(_decode(dg, y, lens, **kw), wfst_decode_ref(tb, y, lens, **kw))


@pytest.mark.parametrize("N", [1, 3, 64, 130])
def test_batch_sizes(graphs, N):
    dg, tb, V = graphs[-1]
    rng = np.random.default_rng(N)
    lens = rng.integers(0, 17, N)
    lens[:3] = [16, 1, 0][:N]
    y, lens = peaky(N, 16, V, seed=N, lens=lens)
    kw = dict(acwt=0.7, lmwt=1.3, wip=-0.4, beam=8.0, max_active=16)
    _compare(_decode(dg, y, lens, **kw), wfst_decode_ref(tb, y, lens, **kw))


def test_length_zero_decodes_the_start_closure_and_dead_utterances(graphs):
    dg, tb, V = graphs[1]
    y, lens = peaky(3, 6, V, seed=4, lens=[0, 6, 6])
    y[2, 3] = -np.inf                               # every candidate of frame 3 costs +inf
    got = _decode(dg, y, lens)
    ref = wfst_decode_ref(tb, y, lens)
    _compare(got, ref)
    assert got["num_words"][2] == -1 and got["cost"][2] == np.inf and (got["align"][2] == -1).all()
    assert (got["align"][0] == -1).all()


# ---------------------------------------------------------------------------------------------------------------------
# 2. invariances
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def mid(graphs):
    dg, tb, V = graphs[-1]
    y, lens = peaky(9, 40, V, seed=7, lens=[40, 37, 29, 20, 11, 5, 2, 1, 0])
    return dg, tb, y, lens


KW = dict(acwt=0.7, lmwt=1.3, wip=-0.4, beam=8.0, max_active=16)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_half_logits_equal_their_upcast(mid, dtype):
    dg, _, y, lens = mid
    yh = torch.tensor(y).to(dtype)
    assert _same(_decode(dg, yh, lens, dtype, **KW), _decode(dg, yh.float(), lens, **KW))


def test_raw_logits_give_the_same_words_and_alignment(mid):
    dg, tb, y, lens = mid
    z = (y + np.random.default_rng(1).standard_normal((y.shape[0], y.shape[1], 1)) * 5).astype(np.float32)
    zl = torch.log_softmax(torch.tensor(z), -1).numpy()
    a, b = _decode(dg, z, lens, **KW), _decode(dg, zl, lens, **KW)
    _compare(a, wfst_decode_ref(tb, z, lens, **KW))
    ra, rb = wfst_decode_ref(tb, z, lens, **KW), wfst_decode_ref(tb, zl, lens, **KW)
    agree = [n for n in range(len(lens)) if all(np.array_equal(ra[k][n], rb[k][n]) for k in ("words", "align"))]
    assert len(agree) >= 0.9 * len(lens)             # the others hold a near-tie that the fp32 shift decides
    for n in agree:
        assert np.array_equal(a["words"][n], b["words"][n]) and np.array_equal(a["align"][n], b["align"][n]), n


def test_padding_is_never_read(mid):
    dg, _, y, lens = mid
    ref = _decode(dg, y, lens, **KW)
    for v in (np.nan, np.inf, -np.inf):
        y2 = y.copy()
        for n, ln in enumerate(lens):
            y2[n, ln:] = v
        assert _same(_decode(dg, y2, lens, **KW), ref), v


def _native(dg, y, lens, fill, K=16, beam=8.0):
    L = _lib.lib()
    N, T, V = y.shape
    yd = torch.tensor(y, device="cuda")
    ld = torch.tensor(lens, dtype=torch.int32, device="cuda")
    ws = torch.full((int(L.ccb_wfst_decode_ws_bytes(dg.handle, N, T, K)),), fill, dtype=torch.uint8, device="cuda")
    Wcap = (T + 1) * (1 + dg.L)
    o = dict(words=torch.full((N, Wcap), 7, dtype=torch.int32, device="cuda"), num_words=torch.full((N,), 7, dtype=torch.int32, device="cuda"),
             align=torch.full((N, T), 7, dtype=torch.int32, device="cuda"), ac_logp=torch.full((N,), 7.0, device="cuda"),
             graph_cost=torch.full((N,), 7.0, device="cuda"), cost=torch.full((N,), 7.0, device="cuda"),
             reached_final=torch.full((N,), 7, dtype=torch.int32, device="cuda"))
    rc = L.ccb_wfst_decode(yd.data_ptr(), 0, N, T, V, ld.data_ptr(), dg.handle, 0.7, 1.3, -0.4, beam, K, ws.data_ptr(),
                           *[o[k].data_ptr() for k in ("words", "num_words", "align", "ac_logp", "graph_cost", "cost",
                                                       "reached_final")], None)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def test_poisoned_workspace_and_outputs(mid):
    dg, _, y, lens = mid
    ref = _decode(dg, y, lens, **KW)
    for fill in (0x00, 0xFF, 0x7F):
        assert _same(_native(dg, y, lens, fill), ref), fill


def test_no_host_synchronisation(mid):
    import ctc_crf
    dg, _, y, lens = mid
    logits, lx = torch.tensor(y, device="cuda"), torch.tensor(lens, dtype=torch.int32)
    ctc_crf.fst_decode(logits, lx, dg)               # the graph's tables are uploaded by its first search on a device
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = ctc_crf.fst_decode(logits, lx, dg, **KW)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(t.is_cuda for t in out)


def test_side_stream(mid):
    import ctc_crf
    dg, _, y, lens = mid
    ref = _decode(dg, y, lens, **KW)
    s = torch.cuda.Stream()
    logits = torch.tensor(y, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out = ctc_crf.fst_decode(logits, torch.tensor(lens, dtype=torch.int32), dg, **KW)
    s.synchronize()
    assert _same({k: v.cpu().numpy() for k, v in out._asdict().items()}, ref)


def test_one_launch_per_call(graphs):
    dg, _, V = graphs[-1]
    counts = []
    for N, T, beam, K in ((1, 5, 4.0, 1), (64, 40, 17.0, 7000), (130, 12, math.inf, 1000), (3, 200, 8.0, 16)):
        y, lens = peaky(N, T, V, seed=N + T)
        k0 = _C.launch_count()
        _decode(dg, y, lens, beam=beam, max_active=K)
        counts.append(_C.launch_count() - k0)
    assert counts == [1, 1, 1, 1], counts


def test_graph_lifetimes(tmp_path, graphs):
    _, tb0, V = graphs[0]
    p0 = write_graph(tmp_path, "a.fst", random_wfst(**GRAPHS[0]))
    p1 = write_graph(tmp_path, "b.fst", random_wfst(**GRAPHS[1]))
    a, b = DecodingGraph(p0), DecodingGraph(p1)
    ta, tb_ = Tables(a), Tables(b)
    y, lens = peaky(4, 12, max(GRAPHS[0]["V"], GRAPHS[1]["V"]) + 1, seed=3)
    for _ in range(2):                               # both alive, used in turn
        _compare(_decode(a, y, lens), wfst_decode_ref(ta, y, lens))
        _compare(_decode(b, y, lens), wfst_decode_ref(tb_, y, lens))
    import ctc_crf
    out = ctc_crf.fst_decode(torch.tensor(y, device="cuda"), torch.tensor(lens, dtype=torch.int32), a)
    del a                                            # destroyed while its search may still run: cudaFree waits for it
    torch.cuda.synchronize()
    _compare({k: v.cpu().numpy() for k, v in out._asdict().items()}, wfst_decode_ref(ta, y, lens))
    _compare(_decode(b, y, lens), wfst_decode_ref(tb_, y, lens))


# ---------------------------------------------------------------------------------------------------------------------
# 3. at size
# ---------------------------------------------------------------------------------------------------------------------
def headline_graph(d, seed=5):
    """V = 72, 3000 words of 2-6 tokens, a 3-gram of 60 000 bigrams and 60 000 trigrams: about 1.46 M states, 3.7 M arcs."""
    arpa = make_random_arpa(str(d / "big.arpa"), 3002, 3, [60000, 60000], seed=seed)
    rng = np.random.default_rng(seed)
    lex = [(str(i), rng.integers(1, 72, size=int(rng.integers(2, 7))).tolist()) for i in range(2, 3002)]
    g, words = fst.make_tlg(72, lex, arpa)
    path = str(d / "big.fst")
    fst.write_fst(path, g)
    return path, lex


def aligned_logits(lex, N, T, V, seed):
    """Peaky logits along the CTC alignment of a random word sequence's pronunciations, blanks between tokens."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((N, T, V)).astype(np.float32)
    for n in range(N):
        al = []
        while len(al) < T:
            for c in lex[int(rng.integers(len(lex)))][1]:
                al += [c] * int(rng.integers(1, 3)) + [0] * int(rng.integers(1, 4))
        z[n, np.arange(T), np.array(al[:T])] += 8.0
    return torch.log_softmax(torch.tensor(z), -1).numpy()


def test_at_size(tmp_path):
    path, lex = headline_graph(tmp_path)
    dg = DecodingGraph(path)
    assert dg.num_arcs > 3_000_000
    N, T = 64, 1500
    y = aligned_logits(lex, N, T, 72, seed=1)
    lens = np.full(N, T, np.int32)
    lens[1], lens[2] = 1, 0
    kw = dict(beam=17.0, max_active=7000)
    got = _decode(dg, y, lens, **kw)
    assert (got["num_words"][3:] > 10).all()
    tb = Tables(dg)
    rows = [0, 1, 2, 37]
    ref = wfst_decode_ref(tb, y[rows], lens[rows], **kw)
    _compare({k: v[rows] for k, v in got.items()}, ref)
