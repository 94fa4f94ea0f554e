"""``ctc_crf.ctc_beam_search`` on the GPU: hypotheses, timesteps and scores against the numpy restatement
(tests/test_beam_dispatch.py) in both modes, exactness at full beam, lower bounds through the losses, the invariances
(dtypes, raw logits, padding, scratch contents, synchronisation, streams, launches), the ``CTCBeamDecoder`` drop-in and the
headline shape."""
import numpy as np
import pytest
import torch

from cat_b200 import _C, fst
from test_beam_dispatch import beam_ref, enum_crf, enum_plain, hyps, plan_out

pytestmark = pytest.mark.gpu


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _search(y, lens, B, cut, crf, dtype=torch.float32):
    import ctc_crf
    logits = (y if isinstance(y, torch.Tensor) else torch.as_tensor(np.asarray(y))).to(device="cuda", dtype=dtype)
    out = ctc_crf.ctc_beam_search(logits, torch.as_tensor(np.asarray(lens), dtype=torch.int32), B, cut, crf)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def _batch(N, T, V, seed, lens=None, scale=2.0):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((N, T, V)) * scale
    y = (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)
    if lens is None:
        lens = rng.integers(0, T + 1, N)
        lens[:3] = [T, 1, 0][:N] if N >= 3 else lens[:3]
    return y, np.asarray(lens, np.int32)


def _compare(out, ref, min_frac=0.95):
    """Tokens, lengths and timesteps exactly, scores within 1e-6 relative, on every utterance without a near-tie."""
    tk, ln, ts, sc = out
    rt, rl, rs, rsc, near = ref
    N = tk.shape[0]
    assert (~near).sum() >= min_frac * N, (near.sum(), N)
    for n in np.nonzero(~near)[0]:
        assert np.array_equal(ln[n], rl[n]), (n, ln[n], rl[n])
        assert np.array_equal(tk[n], rt[n]) and np.array_equal(ts[n], rs[n]), n
        fin = rl[n] >= 0
        np.testing.assert_allclose(sc[n][fin], rsc[n][fin], rtol=1e-6, atol=1e-6)
        assert np.all(np.isneginf(sc[n][~fin]))


@pytest.fixture(scope="module")
def tlm218(tmp_path_factory):
    """A CTC-shaped T o LM graph over V = 218 labels (a deterministic random phone LM composed with the CTC topology)."""
    lm = fst.make_random_lm(H=60, V=218, d=8, seed=3)
    p = str(tmp_path_factory.mktemp("beam") / "tlm218.fst")
    fst.write_fst(p, fst.compose_ctc_lm(lm))
    return p, lm


# ---------------------------------------------------------------------------------------------------------------------
# 1. kernel against the restatement
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("crf", [False, True])
@pytest.mark.parametrize("cut", [40, 218])
@pytest.mark.parametrize("B", [1, 4, 16, 128])
def test_kernel_equals_restatement(tlm218, crf, cut, B):
    path, _ = tlm218
    ctx = _ctx(path)
    G = plan_out(path, _sms(), 16) if crf else None
    y, lens = _batch(3, 24 if B < 128 else 12, 218, seed=B + cut)
    _compare(_search(y, lens, B, cut, crf), beam_ref(y, lens, B, cut, G), min_frac=0.6)
    del ctx


@pytest.mark.parametrize("crf", [False, True])
@pytest.mark.parametrize("N", [1, 64, 130])
def test_batch_sizes(tlm218, crf, N):
    path, _ = tlm218
    ctx = _ctx(path)
    G = plan_out(path, _sms(), 16) if crf else None
    y, lens = _batch(N, 16, 218, seed=N)
    _compare(_search(y, lens, 16, 40, crf), beam_ref(y, lens, 16, 40, G))
    del ctx


@pytest.mark.parametrize("env", ["HUBS", "CTAS"])
def test_hub_rows_and_small_grid(tmp_path, monkeypatch, env):
    lm = fst.make_random_lm(H=30, V=40, d=12, seed=8)
    p = str(tmp_path / "tlm40.fst")
    fst.write_fst(p, fst.compose_ctc_lm(lm))
    if env == "HUBS":
        monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
        monkeypatch.setenv("CCB_PART_ARCS", "7")
        n_ctas = _sms()
        from cat_b200 import plan
        assert plan.load_plan(p, n_ctas, 16).hub_states.size > 0
    else:
        monkeypatch.setenv("CCB_DEN_CTAS", "16")
        n_ctas = 16
    ctx = _ctx(p)
    G = plan_out(p, n_ctas, 16)
    y, lens = _batch(8, 40, 40, seed=2)
    for B, cut in ((16, 10), (64, 40)):
        _compare(_search(y, lens, B, cut, True), beam_ref(y, lens, B, cut, G))
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# 2. exactness at full beam, and lower bounds
# ---------------------------------------------------------------------------------------------------------------------
def test_full_beam_is_exact(tmp_path):
    from oracle import oracle
    lm = fst.make_random_lm(H=3, V=4, d=2, seed=5)
    p = str(tmp_path / "tiny.fst")
    fst.write_fst(p, fst.compose_ctc_lm(lm))
    ctx = _ctx(p)
    G = plan_out(p, _sms(), 16)
    T = 4                              # at most 1 + 3 + 9 + 27 + 81 = 121 prefixes: nothing is pruned at B = 128
    y, _ = _batch(3, T, 4, seed=9)
    lens = np.full(3, T, np.int32)
    for crf in (False, True):
        tk, ln, ts, sc = _search(y, lens, 128, 4, crf)
        for n in range(3):
            want = enum_crf(G, y[n], T) if crf else enum_plain(y[n], T)
            got = hyps(tk, ln, sc, n)
            assert set(got) == set(want), crf
            for k, v in want.items():
                assert abs(got[k] - v) <= 1e-5 * max(1, abs(v)), (crf, k)
                if crf:
                    lp, _ = oracle.ctc(y[n:n + 1], np.asarray(k, np.int32), [len(k)], [T], want_grad=False)
                    assert abs(got[k] - fst.lm_logprob(lm, k) - lp[0]) <= 1e-4 * max(1, abs(v))
    del ctx


def test_scores_are_lower_bounds(tlm218):
    import ctc_crf
    from oracle import oracle
    path, lm = tlm218
    ctx = _ctx(path)
    y, lens = _batch(6, 30, 218, seed=4, lens=[30, 25, 17, 9, 3, 1])
    logits = torch.tensor(y, device="cuda")
    lx = torch.tensor(lens)
    for crf in (False, True):
        tk, ln, ts, sc = ctc_crf.ctc_beam_search(logits, lx, 8, 40, crf)
        labels, ly, utt = ctc_crf.samples_to_labels(tk, ln)
        with torch.no_grad():
            cost = ctc_crf.WARP_CTC_LOSS(size_average=False, reduction="none")(logits, labels, lx, ly, utt=utt).cpu().numpy()
        s = sc.cpu().numpy()[ln.cpu().numpy() >= 0]
        assert len(s) == len(cost)
        bound = -cost
        if crf:
            lab = labels.numpy()
            off = np.concatenate([[0], np.cumsum(ly.numpy())])
            bound = bound + np.array([fst.lm_logprob(lm, lab[off[i]:off[i + 1]]) for i in range(len(cost))])
        assert np.all(s <= bound + 1e-4 * np.abs(bound) + 1e-4), np.max(s - bound)
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# 3. invariances
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def mid(tlm218):
    path, _ = tlm218
    ctx = _ctx(path)
    y, lens = _batch(9, 40, 218, seed=7, lens=[40, 37, 29, 20, 11, 5, 2, 1, 0])
    yield path, y, lens
    del ctx


def _same(a, b):
    return all(np.array_equal(x, z) for x, z in zip(a, b))


@pytest.mark.parametrize("crf", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_half_logits_equal_their_upcast(mid, crf, dtype):
    path, y, lens = mid
    yh = torch.tensor(y).to(dtype)
    assert _same(_search(yh, lens, 16, 40, crf, dtype), _search(yh.float(), lens, 16, 40, crf))


@pytest.mark.parametrize("crf", [False, True])
def test_raw_logits_give_the_same_hypotheses(mid, crf):
    path, y, lens = mid
    G = plan_out(path, _sms(), 16) if crf else None
    z = (y + np.random.default_rng(1).standard_normal((y.shape[0], y.shape[1], 1)) * 5).astype(np.float32)
    zl = torch.log_softmax(torch.tensor(z), -1).numpy()
    a, b = _search(z, lens, 16, 40, crf), _search(zl, lens, 16, 40, crf)
    ra, rb = beam_ref(z, lens, 16, 40, G), beam_ref(zl, lens, 16, 40, G)
    shift = np.array([np.logaddexp.reduce(z[n, :lens[n]].astype(np.float64), -1).sum() for n in range(len(lens))])
    ok = ~(ra[4] | rb[4])
    assert ok.sum() >= 0.9 * len(lens)
    for n in np.nonzero(ok)[0]:
        assert np.array_equal(a[0][n], b[0][n]) and np.array_equal(a[1][n], b[1][n]), n
        fin = a[1][n] >= 0
        np.testing.assert_allclose(a[3][n][fin] - shift[n], b[3][n][fin], rtol=1e-5, atol=1e-3)


@pytest.mark.parametrize("crf", [False, True])
def test_padding_is_never_read(mid, crf):
    path, y, lens = mid
    ref = _search(y, lens, 16, 40, crf)
    for v in (np.nan, np.inf, -np.inf):
        y2 = y.copy()
        for n, l in enumerate(lens):
            y2[n, l:] = v
        assert _same(_search(y2, lens, 16, 40, crf), ref), v


@pytest.mark.parametrize("byte", [0x00, 0xFF, 0x7F])
def test_scratch_contents_change_nothing(mid, monkeypatch, byte):
    from test_scratch_proxy import ScratchProxy
    path, y, lens = mid
    clean = [_search(y, lens, 16, 40, crf) for crf in (False, True)]
    proxy = ScratchProxy(byte)
    monkeypatch.setattr(_C, "torch", proxy)
    for crf, c in zip((False, True), clean):
        assert _same(_search(y, lens, 16, 40, crf), c), (crf, byte)
    L = _C._lib.lib()
    assert any(b == int(L.ccb_ctc_beam_search_ws_bytes(len(lens), y.shape[1], 16)) for b, _, d in proxy.record)


def test_no_host_synchronisation(mid):
    import ctc_crf
    path, y, lens = mid
    logits = torch.tensor(y, device="cuda")
    lx = torch.tensor(lens)
    ctc_crf.ctc_beam_search(logits, lx, 16, 40, True)      # warm-up: the first crf call checks and uploads the graph
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = [ctc_crf.ctc_beam_search(logits, lx, 16, 40, crf) for crf in (False, True)]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(t.is_cuda for o in out for t in o)


def test_side_stream(mid):
    import ctc_crf
    path, y, lens = mid
    ref = [_search(y, lens, 16, 40, crf) for crf in (False, True)]
    s = torch.cuda.Stream()
    logits = torch.tensor(y, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out = [ctc_crf.ctc_beam_search(logits, torch.tensor(lens), 16, 40, crf) for crf in (False, True)]
    s.synchronize()
    for o, r in zip(out, ref):
        assert _same([t.cpu().numpy() for t in o], r)


def test_launch_count_does_not_depend_on_beam(mid):
    path, y, lens = mid
    for crf in (False, True):
        counts = []
        for B in (1, 16, 128):
            k0 = _C.launch_count()
            _search(y, lens, B, 40, crf)
            counts.append(_C.launch_count() - k0)
        assert counts[0] == counts[1] == counts[2] == 1, counts


def test_crf_refuses_a_graph_that_is_not_ctc_shaped(tmp_graphs):
    import ctc_crf
    path, _, V = tmp_graphs["tlm_small"]
    ctx = _ctx(path)
    logits = torch.zeros(1, 5, V, device="cuda")
    for _ in range(2):      # the cached result raises again
        with pytest.raises(RuntimeError, match="not CTC-shaped.*file state"):
            ctc_crf.ctc_beam_search(logits, torch.tensor([5], dtype=torch.int32), 4, V, True)
    ctc_crf.ctc_beam_search(logits, torch.tensor([5], dtype=torch.int32), 4, V, False)      # plain mode needs no graph
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# 4. the ctcdecode drop-in, as cat/ctc/train.py's get_wer uses it
# ---------------------------------------------------------------------------------------------------------------------
def _edit_distance(a, b):
    d = list(range(len(b) + 1))
    for i, x in enumerate(a, 1):
        prev, d[0] = d[0], i
        for j, z in enumerate(b, 1):
            prev, d[j] = d[j], min(d[j] + 1, d[j - 1] + 1, prev + (x != z))
    return d[len(b)]


def test_decoder_drop_in_and_get_wer_pattern(mid):
    import ctc_crf
    path, y, lens = mid
    labels = [str(i) for i in range(y.shape[2])]
    dec = ctc_crf.CTCBeamDecoder(labels, beam_width=16, cutoff_top_n=40, num_processes=6, blank_id=0)
    logits = torch.tensor(y)                        # on the CPU, as get_wer hands it over after .float().cpu()
    probs = logits.exp()
    results, scores, timesteps, out_lens = dec.decode(probs, torch.tensor(lens))
    tk, ln, ts, sc = [t.cpu() for t in ctc_crf.ctc_beam_search(probs.cuda().log(), torch.tensor(lens), 16, 40)]
    assert torch.equal(results.cpu(), tk) and torch.equal(out_lens.cpu(), ln) and torch.equal(timesteps.cpu(), ts)
    assert torch.equal(scores.cpu(), -sc)
    lp = ctc_crf.CTCBeamDecoder(labels, beam_width=16, log_probs_input=True).decode(torch.tensor(y, device="cuda"), lens)
    same = _search(y, lens, 16, 40, False)
    assert np.array_equal(lp[0].cpu().numpy(), same[0])
    # get_wer: the best hypothesis of each utterance against a reference
    refs = [list(range(1, 1 + n % 5)) for n in range(len(lens))]
    err = 0
    for i in range(len(lens)):
        hyp = results[i][0][:out_lens[i][0]].tolist()
        err += _edit_distance(hyp, refs[i])
    assert 0 <= err <= sum(max(len(r), int(out_lens[i][0])) for i, r in enumerate(refs))


# ---------------------------------------------------------------------------------------------------------------------
# 5. the headline shape
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def headline(tmp_path_factory):
    """A CTC-shaped T o LM graph of 1.10 M arcs over V = 218 (1800 LM states, 24 successors each)."""
    lm = fst.make_random_lm(H=1800, V=218, d=24, seed=1)
    p = str(tmp_path_factory.mktemp("hl") / "headline_tlm.fst")
    fst.write_fst(p, fst.compose_ctc_lm(lm))
    return p


@pytest.mark.parametrize("crf", [False, True])
def test_headline_shape(headline, crf):
    from oracle import oracle
    ctx = _ctx(headline)
    N, T = 64, 1500
    lens = np.maximum(200, T - 37 * np.arange(N)).astype(np.int32)
    y, _, lens, _ = oracle.synth_batch(N, T, 218, seed=21, lens=lens)
    out = _search(y, lens, 16, 40, crf)
    assert np.all(out[1][:, 0] >= 0)
    G = plan_out(headline, _sms(), 16) if crf else None
    sub = [0, 1, 31, 63]
    ref = beam_ref(y[sub], lens[sub], 16, 40, G)
    _compare([o[sub] for o in out], ref, min_frac=0.75)
    del ctx
