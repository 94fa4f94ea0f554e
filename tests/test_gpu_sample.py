"""``ctc_crf.crf_sample`` on the GPU: exact paths against the numpy restatement (tests/test_sample_dispatch.py), the sequence
distribution against exhaustive enumeration, per-frame label frequencies against the fp64 den occupancies at size, and the
invariances (checkpointed alpha, slicing, seeds, dtypes, raw logits, padding, scratch contents, synchronisation, launches)."""
import itertools

import numpy as np
import pytest
import torch

from cat_b200 import _C, fst
from test_sample_dispatch import plan_csr, sample_ref

pytestmark = pytest.mark.gpu


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _sample(y, lens, K, seed, dtype=torch.float32):
    import ctc_crf
    logits = torch.as_tensor(y).to(device="cuda", dtype=dtype)
    out = ctc_crf.crf_sample(logits, torch.as_tensor(lens, dtype=torch.int32), K, generator=_gen(seed))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def _call_seed(seed):
    return _C.draw_seed(_gen(seed))


def _valid_rows(P, y, lens, tokens, lengths, align, logp, atol):
    """Every feasible sample is a path of the graph ending in a final state and its collapse is `tokens`.  Yields the fp64
    log-sum of the scores of the graph's state paths with these frame labels: the score of the sampled path where the labels
    determine the states (T o LM graphs), an upper bound of it otherwise."""
    S, off, src, w, lab, fin = P["S"], P["in_off"], P["in_src"], P["in_w"].astype(np.float64), P["state_label"], \
        P["final_lin"].astype(np.float64)
    dst = np.repeat(np.arange(S), np.diff(off))
    order = np.argsort(src, kind="stable")
    o_src, o_dst, o_w = src[order], dst[order], w[order]
    o_off = np.searchsorted(o_src, np.arange(S + 1))
    y = np.asarray(y, np.float64)
    for n in range(align.shape[0]):
        ln = int(lens[n])
        for k in range(align.shape[1]):
            if lengths[n, k] < 0:
                continue
            row = align[n, k]
            assert np.all(row[ln:] == -1)
            toks = [int(l) for j, l in enumerate(row[:ln]) if l != 0 and (j == 0 or row[j - 1] != l)]
            assert lengths[n, k] == len(toks) and list(tokens[n, k, :len(toks)]) == toks
            assert np.all(tokens[n, k, len(toks):] == -1)
            act = {P["start"]: 0.0}      # state -> log weight
            for t in range(ln):
                nxt = {}
                for q, lw in act.items():
                    sl = slice(o_off[q], o_off[q + 1])
                    for d, ww in zip(o_dst[sl], o_w[sl]):
                        if lab[d] == row[t] and ww > 0:
                            v = lw + np.log(ww) + y[n, t, row[t]]
                            nxt[int(d)] = np.logaddexp(nxt.get(int(d), -np.inf), v)
                act = nxt
                assert act, f"utterance {n} sample {k}: no path with these labels at frame {t}"
            ends = [lw + np.log(fin[q]) for q, lw in act.items() if fin[q] > 0]
            assert ends, f"utterance {n} sample {k}: the path ends in no final state"
            yield n, k, np.logaddexp.reduce(ends)


# ---------------------------------------------------------------------------------------------------------------------
# 1. exact paths
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tlm_small", "random_split", "fixture"])
def test_paths_equal_the_restatement(tmp_graphs, fixture_fst, fixture_inputs, name):
    from oracle import oracle
    if name == "fixture":
        path = fixture_fst
        y0 = fixture_inputs["y"]
        y = np.concatenate([y0, y0[:, ::-1], y0 * 1.5 - 0.2], 0).astype(np.float32)
        lens = np.array([5, 4, 3], np.int32)
    else:
        path, _, V = tmp_graphs[name]
        y, _, lens, _ = oracle.synth_batch(6, 24, V, seed=5, lens=np.array([24, 20, 17, 9, 3, 1], np.int32))
    ctx = _ctx(path)
    K, seed = 96, 11
    tokens, lengths, align, logp = _sample(y, lens, K, seed)
    P = plan_csr(path, _sms(), 16)
    rt, rl, ra, rlogp, near = sample_ref(P, y, lens, K, _call_seed(seed))
    draws = int(((lens + 1)[:, None] * np.ones((1, K))).sum())
    assert near.sum() <= 1e-3 * draws, (near.sum(), draws)
    same = np.all(align == ra, axis=2) & (lengths == rl) & np.all(tokens == rt, axis=2)
    assert np.all(same | (near > 0)), np.argwhere(~same & (near == 0))[:5]
    ok = same & (rl >= 0)
    assert ok.sum() > 0.9 * (rl >= 0).sum()
    np.testing.assert_allclose(logp[ok], rlogp[ok], atol=1e-4, rtol=0)
    la, _, _ = oracle.den(fst.read_fst(path), y, lens)
    for n, k, sc in _valid_rows(P, y, lens, tokens, lengths, align, logp, 1e-4):
        assert logp[n, k] <= sc - la[n] + 1e-4
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# 2. the sequence distribution
# ---------------------------------------------------------------------------------------------------------------------
def test_sequence_distribution_is_the_posterior(tmp_path):
    from scipy import stats
    from oracle import oracle
    V, T = 4, 5
    lm = fst.make_random_lm(H=3, V=V, d=2, seed=5)
    g = fst.compose_ctc_lm(lm)
    p = str(tmp_path / "tlm.fst")
    fst.write_fst(p, g)
    rng = np.random.default_rng(2)
    x = rng.standard_normal((1, T, V))
    y = (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)
    la, _, _ = oracle.den(g, y, [T])
    post = {}
    for L in range(0, T + 1):
        for l in itertools.product(range(1, V), repeat=L):
            lp_lm = fst.lm_logprob(lm, l)
            if not np.isfinite(lp_lm):
                continue
            lp, _ = oracle.ctc(y, np.asarray(l, np.int32), [L], [T], want_grad=False)
            if np.isfinite(lp[0]):
                post[l] = np.exp(lp_lm + lp[0] - la[0])
    assert abs(sum(post.values()) - 1.0) < 1e-5
    ctx = _ctx(p)
    K = 1 << 17
    tokens, lengths, _, logp = _sample(y, [T], K, seed=3)
    assert (lengths >= 0).all()
    counts = {}
    for k in range(K):
        key = tuple(tokens[0, k, :lengths[0, k]].tolist())
        counts[key] = counts.get(key, 0) + 1
    assert set(counts) <= set(post), set(counts) - set(post)
    big = [l for l in post if post[l] * K >= 5]
    rest = [l for l in post if post[l] * K < 5]
    obs = [counts.get(l, 0) for l in big] + ([sum(counts.get(l, 0) for l in rest)] if rest else [])
    exp = [post[l] * K for l in big] + ([sum(post[l] for l in rest) * K] if rest else [])
    exp = np.array(exp) * (K / sum(exp))
    assert len(big) >= 5
    pval = stats.chisquare(obs, exp).pvalue
    assert pval > 1e-3, pval
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# 3. at size: label frequencies against the den occupancies
# ---------------------------------------------------------------------------------------------------------------------
def _check_occupancy(g, P, y, lens, K, seed, n_check, atol_score):
    from oracle import oracle
    tokens, lengths, align, logp = _sample(y, lens, K, seed)
    assert (lengths >= 0).all()
    sub = np.arange(min(n_check, len(lens)))
    la, _, gam = oracle.den(g, y[sub], lens[sub], fast=True)
    V = y.shape[2]
    for n in sub:
        ln = int(lens[n])
        freq = np.zeros((ln, V))
        for t in range(ln):
            freq[t] = np.bincount(align[n, :, t], minlength=V)[:V] / K
        p = gam[n, :ln]
        # 6 sigma, and at least 3 samples of slack: over the ~10^5 (frame, label) cells of an utterance, labels of occupancy
        # ~1e-5 are drawn twice in a few cells by chance, which is 2e-3 at K = 1024
        excess = np.abs(freq - p) - (6 * np.sqrt(p * (1 - p) / K) + max(1e-3, 3.0 / K))
        assert np.all(excess <= 0), (np.unravel_index(np.argmax(excess), excess.shape), excess.max())
    # a few rows per utterance through the graph, scored in fp64
    rows = np.zeros_like(lengths) - 1
    rows[sub, :4] = lengths[sub, :4]
    for n, k, sc in _valid_rows(P, y, lens, tokens, rows, align, logp, atol_score):
        assert logp[n, k] <= sc - la[n] + atol_score, (sc - la[n], logp[n, k])


@pytest.fixture(scope="module")
def headline(tmp_path_factory):
    g = fst.make_synthetic_den(20000, 24, 218, seed=7)
    p = str(tmp_path_factory.mktemp("hl") / "headline.fst")
    fst.write_fst(p, g)
    return p, g


@pytest.mark.parametrize("N", [4, 64])
def test_at_size_headline(headline, N):
    from oracle import oracle
    path, g = headline
    ctx = _ctx(path)
    T = 1500
    lens = np.maximum(200, T - 37 * np.arange(N)).astype(np.int32)
    y, _, lens, _ = oracle.synth_batch(N, T, 218, seed=21, lens=lens)
    P = plan_csr(path, _sms(), 16)
    _check_occupancy(g, P, y, lens, 1024, 5, 2, 2e-2)
    del ctx


@pytest.mark.parametrize("env", ["HUBS", "CTAS"])
def test_at_size_hub_rows_and_small_grid(tmp_graphs, monkeypatch, env):
    from oracle import oracle
    if env == "HUBS":
        monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
        monkeypatch.setenv("CCB_PART_ARCS", "7")
        n_ctas = _sms()
    else:
        monkeypatch.setenv("CCB_DEN_CTAS", "16")
        n_ctas = 16
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    P = plan_csr(path, n_ctas, 16)
    if env == "HUBS":
        from cat_b200 import plan
        assert plan.load_plan(path, n_ctas, 16).hub_states.size > 0
    T = 400
    y, _, lens, _ = oracle.synth_batch(8, T, V, seed=9, lens=np.array([400, 390, 300, 250, 200, 120, 50, 7], np.int32))
    _check_occupancy(g, P, y, lens, 1024, 6, 3, 2e-3)
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# 4. invariances
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def mid(tmp_graphs):
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    lens = np.array([60, 55, 41, 33, 20, 9, 2, 60, 47], np.int32)
    y, _, lens, _ = oracle.synth_batch(len(lens), 60, V, seed=4, lens=lens)
    yield path, y, lens
    del ctx


def _same(a, b):
    """The same samples (tokens, lengths, align bit for bit) and the same path_logp but for logZ's run-to-run spread (the den
    forward pass sums its column totals with atomics, so logZ, and with it every path_logp, can move by an ulp)."""
    return (all(np.array_equal(x, z) for x, z in zip(a[:3], b[:3])) and np.array_equal(np.isinf(a[3]), np.isinf(b[3]))
            and np.allclose(a[3], b[3], rtol=0, atol=1e-4))


def test_checkpointed_equals_full_spill(mid, monkeypatch):
    path, y, lens = mid
    full = _sample(y, lens, 32, 1)
    for k in (1, 7, 60):
        monkeypatch.setattr(_C, "_ckpt_k_override", k)
        assert _same(_sample(y, lens, 32, 1), full), k


def test_slicing_and_batch_independence(mid, monkeypatch):
    path, y, lens = mid
    import ctc_crf
    full = _sample(y, lens, 16, 2)
    monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 4)
    assert _same(_sample(y, lens, 16, 2), full)
    monkeypatch.undo()
    # utterance n alone, as row n of a batch (the counter carries the batch index): same samples through n_base
    seed = _call_seed(2)
    logits = torch.tensor(y, device="cuda")
    lx = torch.tensor(lens, dtype=torch.int32)
    L = _C._lib.lib()
    for n in (0, 4, 8):
        tk = torch.empty((1, 16, y.shape[1]), dtype=torch.int32, device="cuda")
        le = torch.empty((1, 16), dtype=torch.int32, device="cuda")
        al = torch.empty_like(tk)
        lp = torch.empty((1, 16), dtype=torch.float32, device="cuda")
        tmax = int(lens[n])
        lx_d = lx[n:n + 1].cuda()
        a_ws = torch.empty(int(L.ccb_den_alpha_floats(1, tmax)), dtype=torch.float32, device="cuda")
        x_ws = torch.empty(int(L.ccb_den_aux_bytes(1, tmax)), dtype=torch.uint8, device="cuda")
        s_ws = torch.empty(int(L.ccb_crf_sample_ws_bytes(1, 16, tmax)), dtype=torch.uint8, device="cuda")
        rc = L.ccb_crf_sample(logits[n:n + 1].data_ptr(), 0, 1, y.shape[1], y.shape[2], tmax, 0, lx_d.data_ptr(), 16, seed, n,
                              a_ws.data_ptr(), x_ws.data_ptr(), s_ws.data_ptr(), tk.data_ptr(), le.data_ptr(), al.data_ptr(),
                              lp.data_ptr(), C_stream())
        assert rc == 0, _C._lib.last_error()
        torch.cuda.synchronize()
        assert np.array_equal(al.cpu().numpy()[0], full[2][n]) and np.array_equal(tk.cpu().numpy()[0], full[0][n])
        np.testing.assert_allclose(lp.cpu().numpy()[0], full[3][n], rtol=0, atol=1e-4)
    # and the same utterances in a batch of their own through the public entry (indices differ: other samples)
    sub = _sample(y[[0, 4, 8]], lens[[0, 4, 8]], 16, 2)
    assert np.array_equal(sub[2][0], full[2][0])


def C_stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def test_generator_reproduces_and_next_call_differs(mid):
    path, y, lens = mid
    import ctc_crf
    logits = torch.tensor(y, device="cuda")
    lx = torch.tensor(lens, dtype=torch.int32)
    g = _gen(5)
    a = [t.cpu().numpy() for t in ctc_crf.crf_sample(logits, lx, 8, generator=g)]
    b = [t.cpu().numpy() for t in ctc_crf.crf_sample(logits, lx, 8, generator=g)]
    g.manual_seed(5)
    c = [t.cpu().numpy() for t in ctc_crf.crf_sample(logits, lx, 8, generator=g)]
    assert _same(a, c)
    assert not np.array_equal(a[2], b[2])
    torch.manual_seed(3)
    d = [t.cpu().numpy() for t in ctc_crf.crf_sample(logits, lx, 8)]
    torch.manual_seed(3)
    e = [t.cpu().numpy() for t in ctc_crf.crf_sample(logits, lx, 8)]
    assert _same(d, e)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_half_logits(mid, dtype):
    path, y, lens = mid
    K = 32
    out = _sample(y, lens, K, 7, dtype=dtype)
    yr = torch.tensor(y).to(dtype).float().numpy()
    P = plan_csr(path, _sms(), 16)
    rt, rl, ra, rlogp, near = sample_ref(P, yr, lens, K, _call_seed(7))
    same = np.all(out[2] == ra, axis=2)
    assert np.all(same | (near > 0))
    np.testing.assert_allclose(out[3][same], rlogp[same], atol=1e-3, rtol=0)


def test_raw_logits_give_the_same_paths(mid):
    path, y, lens = mid
    rng = np.random.default_rng(1)
    z = (y + rng.standard_normal((y.shape[0], y.shape[1], 1)) * 5).astype(np.float32)   # a per-frame shift
    a = _sample(z, lens, 64, 9)
    b = _sample(torch.log_softmax(torch.tensor(z), -1).numpy(), lens, 64, 9)
    same = np.all(a[2] == b[2], axis=2)
    assert same.mean() >= 0.999
    np.testing.assert_allclose(a[3][same], b[3][same], atol=1e-3, rtol=0)


def test_padding_is_never_read(mid):
    path, y, lens = mid
    a = _sample(y, lens, 16, 4)
    y2 = y.copy()
    for n, ln in enumerate(lens):
        y2[n, ln:] = np.nan
    assert _same(_sample(y2, lens, 16, 4), a)


@pytest.mark.parametrize("byte", [0xFF, 0x7F])
def test_scratch_contents_change_nothing(mid, monkeypatch, byte):
    from test_scratch_proxy import ScratchProxy
    path, y, lens = mid
    monkeypatch.setattr(_C, "torch", ScratchProxy(0))
    clean = _sample(y, lens, 16, 8)
    monkeypatch.setattr(_C, "torch", ScratchProxy(byte))
    assert _same(_sample(y, lens, 16, 8), clean)
    monkeypatch.setattr(_C, "_ckpt_k_override", 5)
    ck = _sample(y, lens, 16, 8)
    assert _same(ck, clean), [np.argwhere(a != b)[:4].tolist() for a, b in zip(ck, clean)]


# ---------------------------------------------------------------------------------------------------------------------
# 5. edge cases
# ---------------------------------------------------------------------------------------------------------------------
def test_infeasible_and_empty_utterances(mid):
    path, y, lens = mid
    y2 = y.copy()
    y2[1, 10] = -np.inf             # a frame no path crosses
    lens2 = lens.copy()
    lens2[3] = 0
    tokens, lengths, align, logp = _sample(y2, lens2, 8, 1)
    for n in (1, 3):
        assert np.all(lengths[n] == -1) and np.all(tokens[n] == -1) and np.all(align[n] == -1)
        assert np.all(np.isneginf(logp[n]))
    assert np.all(lengths[[0, 2, 4]] >= 0) and np.all(np.isfinite(logp[[0, 2, 4]]))
    a = _sample(y, lens, 8, 1)
    ok = [0, 2, 4, 5, 6, 7, 8]
    assert np.array_equal(a[2][ok], align[ok])


def test_samples_feed_the_loss(mid):
    path, y, lens = mid
    import ctc_crf
    logits = torch.tensor(y, device="cuda", requires_grad=True)
    lx = torch.tensor(lens, dtype=torch.int32)
    tokens, lengths, _, _ = ctc_crf.crf_sample(logits, lx, 4, generator=_gen(2))
    labels, ly, utt = ctc_crf.samples_to_labels(tokens, lengths)
    assert int(ly.numel()) == 4 * len(lens)
    costs = ctc_crf.CTC_CRF_LOSS(reduction="none")(logits, labels, lx, ly, utt=utt)
    assert torch.isfinite(costs).all()
    costs.sum().backward()
    assert torch.isfinite(logits.grad).all()


def test_no_host_synchronisation(mid):
    path, y, lens = mid
    import ctc_crf
    logits = torch.tensor(y, device="cuda")
    lx = torch.tensor(lens, dtype=torch.int32)
    ctc_crf.crf_sample(logits, lx, 4, generator=_gen(1))     # warm-up: the first call uploads the in-arc table
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = ctc_crf.crf_sample(logits, lx, 4, generator=_gen(1))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert out[0].is_cuda and out[3].is_cuda


def test_launch_count_does_not_depend_on_k(mid):
    path, y, lens = mid
    counts = []
    for K in (1, 16, 200):
        k0 = _C.launch_count()
        _sample(y, lens, K, 3)
        counts.append(_C.launch_count() - k0)
    assert counts[0] == counts[1] == counts[2], counts
