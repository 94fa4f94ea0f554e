"""GPU: the RNN-T beam search with LM fusion and ILM estimation (``cat_b200.rnnt_decode``): the n-gram rows kernel against
the textbook scorer and the walk, the fused step frame by frame through the C ABI against ``beam_ref_fused``, and
``RNNTDecoder`` end to end against the restatement of CAT's decoder (tests/rnnt_fusion_oracle.py)."""
import numpy as np
import pytest
import torch

from cat_b200 import _lib
from cat_b200.ngram import NGramLM, make_random_arpa
from cat_b200.rnnt_decode import RNNTDecoder, rnnt_beam_search
from rnnt_decode_oracle import LSTMPredictor
from rnnt_fusion_oracle import CatNGram, JointNet, LSTMLM, beam_ref_fused, cat_decode_fused, fuse_term
from test_ngram_dispatch import LN10, Textbook, Walk

pytestmark = pytest.mark.gpu

_DT = {"fp32": (torch.float32, 0), "bf16": (torch.bfloat16, 1), "fp16": (torch.float16, 2)}


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


def _rounded(x, dt):
    return torch.tensor(np.asarray(x, dtype=np.float32)).to(dt).float().numpy()


# ---- n-gram rows -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V, order, counts", [(30, 2, 80), (30, 3, [150, 200]), (40, 5, [200, 250, 250, 250]),
                                              (4232, 5, [20000, 20000, 20000, 20000])])
def test_slot_rows_match_textbook_and_walk(tmp_path, V, order, counts):
    path = make_random_arpa(str(tmp_path / "lm.arpa"), V, order, counts, seed=order, pruned_prefixes=0.3)
    labels = _labels(V)
    lm = NGramLM(path, labels)
    t = lm.tables()
    tb, walk = Textbook(path, labels), Walk(lm)
    L = _lib.lib()
    N, B = 3, 5
    dev = torch.device("cuda")
    st = [torch.full((N, B), -7, dtype=torch.int32, device=dev) for _ in range(2)]
    rows = torch.full((N * B, V), float("nan"), device=dev)
    rng = np.random.default_rng(V + order)
    grams = [[int(w) for w in g] for g in tb.g if len(g) == order and all(w.isdigit() for w in g)]
    prefixes = [[()] * B for _ in range(N)]
    states = np.full((N, B), int(t["root_dst"][t["eos"]]))
    ks = np.arange(V) if V <= 100 else np.concatenate([[0, 1], rng.choice(np.arange(2, V), 200, replace=False)])
    for step in range(8):
        if step == 0:
            rc = L.ccb_ngram_slot_rows(lm.handle, N, B, V, None, None, None, st[0].data_ptr(), rows.data_ptr(), None)
        else:
            par = rng.integers(0, B, (N, B))
            tok = np.where(rng.random((N, B)) < 0.3, -1, rng.integers(1, V, (N, B)))
            if grams:   # follow the LM's own n-grams too, so that the long histories are reached
                for n in range(N):
                    g = grams[rng.integers(len(grams))]
                    tok[n, 0] = g[min(step - 1, len(g) - 1)]
            par_d = torch.tensor(par, dtype=torch.int32, device=dev)   # (kept alive until the launch has read them)
            tok_d = torch.tensor(tok, dtype=torch.int32, device=dev)
            rc = L.ccb_ngram_slot_rows(lm.handle, N, B, V, par_d.data_ptr(), tok_d.data_ptr(), st[0].data_ptr(),
                                       st[1].data_ptr(), rows.data_ptr(), None)
            st.reverse()
            new_p, new_s = [], np.empty_like(states)
            for n in range(N):
                new_p.append([prefixes[n][par[n, q]] + ((int(tok[n, q]),) if tok[n, q] >= 0 else ()) for q in range(B)])
                for q in range(B):
                    s = states[n, par[n, q]]
                    new_s[n, q] = walk(s, int(t["tok2word"][tok[n, q]]))[1] if tok[n, q] >= 0 else s
            prefixes, states = new_p, new_s
        assert rc == 0, _lib.last_error()
        S = st[0].cpu().numpy()
        R = rows.cpu().numpy()
        assert (S == states).all()
        for n in range(N):
            for q in range(B):
                r = R[n * B + q]
                assert r[0] == 0.0
                hist = ["</s>"] + [tb.word(labels[c]) for c in prefixes[n][q]]
                h = tuple(hist[max(0, len(hist) - (order - 1)):])
                for k in ks[ks > 0]:
                    acc, _ = walk(int(S[n, q]), int(t["tok2word"][k]))
                    assert r[k] == np.float32(acc * LN10), (n, q, k)
                    ref = tb.log10(h, tb.word(labels[k])) * LN10
                    assert abs(float(r[k]) - ref) <= 1e-6 * (1 + abs(ref))


# ---- the fused step, frame by frame -----------------------------------------------------------------------------------
def _drive_fused(mode, dname, N, T, B, V, lens, seed, use_lm, use_ilm, alpha=0.7, beta=-0.4, w=-0.35, scale=2.0):
    """Runs ccb_rnnt_beam_step_fused frame by frame, each live slot's rows built from the prefix read back from the step
    outputs.  Returns (per utterance {prefix: score + LM part} of the final beam, lp, term) for beam_ref_fused."""
    dt, code = _DT[dname]

    def draw(*key):
        return np.random.default_rng(hash((seed,) + key) & 0xffffffff).standard_normal(V) * scale

    f = np.stack([np.stack([_rounded(draw(-1, n, t), dt) for t in range(T)]) for n in range(N)]) if mode == 2 else None

    def kernel_row(n, t, p):
        z = draw(n, t, *p)
        if mode == 0:
            z = z - np.logaddexp.reduce(z)
        return _rounded(z, dt)

    def lm_row(n, p):   # an LM row of the prefix, -inf at one label
        z = draw(-2, n, *p)
        z = z - np.logaddexp.reduce(z)
        z[(len(p) * 7 + 3) % V] = -np.inf
        return _rounded(z, dt)

    def ilm_row(n, p):
        return _rounded(draw(-3, n, *p), dt)

    def lp(n, t, p):
        z = kernel_row(n, t, p).astype(np.float64)
        if mode == 0:
            return z
        if mode == 2:
            z = (np.float32(f[n, t]) + z.astype(np.float32)).astype(np.float64)
        return z - np.logaddexp.reduce(z)

    def term(n, t, p):
        return fuse_term(lm_row(n, p) if use_lm else None, ilm_row(n, p) if use_ilm else None, alpha, beta, w)

    L = _lib.lib()
    dev = torch.device("cuda")
    par, tok, nod = (torch.empty((N, B), dtype=torch.int32, device=dev) for _ in range(3))
    sc = torch.empty((N, B), dtype=torch.float64, device=dev)
    lmp = torch.zeros((N, B), dtype=torch.float64, device=dev)
    ws = torch.empty(int(L.ccb_rnnt_beam_ws_bytes(N, T, B)), dtype=torch.uint8, device=dev)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    fd = torch.tensor(f, dtype=torch.float32).to(dt).to(dev).contiguous() if mode == 2 else None
    assert L.ccb_rnnt_beam_init(N, T, B, ws.data_ptr(), par.data_ptr(), tok.data_ptr(), nod.data_ptr(), sc.data_ptr(),
                                None) == 0, _lib.last_error()
    prefixes = [[()] + [None] * (B - 1) for _ in range(N)]
    for t in range(T):
        blocks = [np.zeros((N * B, V), dtype=np.float32) for _ in range(3)]
        for n in range(N):
            for q, p in enumerate(prefixes[n]):
                if p is not None:
                    blocks[0][n * B + q] = kernel_row(n, t, p)
                    blocks[1][n * B + q] = lm_row(n, p)
                    blocks[2][n * B + q] = ilm_row(n, p)
        rt, lt, it = (torch.tensor(b).to(dt).to(dev).contiguous() for b in blocks)
        rc = L.ccb_rnnt_beam_step_fused(rt.data_ptr(), fd.data_ptr() if fd is not None else None, code, mode, N, T, B, V,
                                        t, lens_d.data_ptr(), 0, ws.data_ptr(), par.data_ptr(), tok.data_ptr(),
                                        nod.data_ptr(), sc.data_ptr(), lt.data_ptr() if use_lm else None, code, alpha,
                                        beta, it.data_ptr() if use_ilm else None, code, w, lmp.data_ptr(), None)
        assert rc == 0, _lib.last_error()
        P, K, S = (x.cpu().numpy() for x in (par, tok, sc))
        for n in range(N):
            if t >= lens[n]:
                assert (P[n] == np.arange(B)).all() and (K[n] == -1).all()
                continue
            old = prefixes[n]
            prefixes[n] = [None if S[n, q] == -np.inf else old[P[n, q]] + ((int(K[n, q]),) if K[n, q] >= 0 else ())
                           for q in range(B)]
    S, M = sc.cpu().numpy(), lmp.cpu().numpy()
    beams = [{p: (S[n, q], M[n, q]) for q, p in enumerate(prefixes[n]) if p is not None} for n in range(N)]
    return beams, lp, term


@pytest.mark.parametrize("terms", ["lm", "ilm", "both"])
@pytest.mark.parametrize("dname", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N, T, B, V", [(3, 6, 4, 37), (2, 5, 16, 300), (2, 3, 16, 4232), (2, 4, 1, 9), (2, 3, 128, 300)])
def test_fused_step_matches_beam_ref(mode, dname, N, T, B, V, terms):
    lens = [T, max(T - 2, 1)] + [0] * (N - 2)
    use_lm, use_ilm = terms in ("lm", "both"), terms in ("ilm", "both")
    beams, lp, term = _drive_fused(mode, dname, N, T, B, V, lens, V + 7 * mode, use_lm, use_ilm)
    # the ILM normaliser is an fp32 reduction in the kernel, so only the LM alone is exact to fp64 rounding in mode 0
    tol = 1e-12 if mode == 0 and not use_ilm else 1e-5
    for n in range(N):
        ref = beam_ref_fused(lens[n], V, B, lambda t, p: lp(n, t, p), lambda t, p: term(n, t, p))
        assert set(beams[n]) == {p for p, _ in ref}, n
        for p, s in ref:
            a, m = beams[n][p]
            assert abs((a + m) - s) <= tol * (1 + abs(s)), (n, p, a, m, s)


# ---- end to end ---------------------------------------------------------------------------------------------------------
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


def _compare(got, ref, tol=1e-4):
    for (gh, gs), (rh, rs) in zip(got, ref):
        assert gh == rh
        for a, b in zip(gs, rs):
            assert abs(a - b) <= tol * (1 + abs(b)), (a, b)


@pytest.mark.parametrize("lm_kind, mode, alpha, beta, w", [
    ("ngram2", "add", 0.6, 0.5, 0.0), ("ngram5", "add", 0.6, 0.5, 0.0), ("lstm", "add", 0.5, 0.2, 0.0),
    (None, "add", 0.0, 0.0, 0.3), (None, "cat", 0.0, 0.0, 0.3),
    ("ngram3", "add", 0.28125, 0.5, -0.3125), ("lstm", "cat", 0.28125, 0.5, -0.3125),
])
@pytest.mark.parametrize("B", [1, 4, 16])
def test_decoder_matches_cat_restatement(tmp_path, lm_kind, mode, alpha, beta, w, B):
    V = 29
    pred, joiner = _build(V, mode=mode)
    lm = ref_lm = None
    if lm_kind == "lstm":
        lm = ref_lm = _lstm_lm(V)
    elif lm_kind:
        lm, ref_lm = _ngram(tmp_path, V, int(lm_kind[-1]))
    torch.manual_seed(5)
    enc = torch.randn(5, 9, 32, device="cuda")
    lens = torch.tensor([9, 1, 0, 6, 9])
    dec = RNNTDecoder(pred, joiner, beam_size=B, lm_module=lm, alpha=alpha, beta=beta, est_ilm=w != 0, ilm_weight=w)
    got = dec(enc, lens)
    ref = cat_decode_fused(enc, lens, pred, joiner, B, lm=ref_lm, alpha=alpha, beta=beta, ilm_weight=w)
    _compare(got, ref)
    assert got[2] == ([[]], [0.0])


def test_cat_sized(tmp_path):
    V, H = 4232, 512
    torch.manual_seed(0)
    pred = LSTMPredictor(V, H).cuda().eval()
    joiner = JointNet(H, H, V, H).cuda().eval()
    for p in joiner.fc.parameters():
        p.data.mul_(4.0)
    lm, ref_lm = _ngram(tmp_path, V, 3, [8000, 8000])
    enc = torch.randn(2, 8, H, device="cuda")
    lens = torch.tensor([8, 5])
    got = RNNTDecoder(pred, joiner, beam_size=16, lm_module=lm, alpha=0.28125, beta=0.5, est_ilm=True,
                      ilm_weight=-0.3125)(enc, lens)
    _compare(got, cat_decode_fused(enc, lens, pred, joiner, 16, lm=ref_lm, alpha=0.28125, beta=0.5, ilm_weight=-0.3125))


def test_zero_weights_are_the_search_without_fusion(tmp_path):
    V = 23
    pred, joiner = _build(V)
    lm, _ = _ngram(tmp_path, V, 3)
    enc = torch.randn(3, 7, 32, device="cuda")
    lens = torch.tensor([7, 3, 5])
    plain = rnnt_beam_search(enc, lens, pred, joiner, beam_size=4)
    for kw in (dict(lm=lm, alpha=0.0, beta=0.7), dict(lm=_lstm_lm(V), alpha=0.0), dict(ilm_weight=0.0)):
        for x, y in zip(plain, rnnt_beam_search(enc, lens, pred, joiner, beam_size=4, **kw)):
            assert torch.equal(x, y)
    dec = RNNTDecoder(pred, joiner, beam_size=4, lm_module=lm, alpha=0.0, beta=0.7, est_ilm=True, ilm_weight=0.0)
    assert dec(enc, lens) == RNNTDecoder(pred, joiner, beam_size=4)(enc, lens)


# ---- properties ---------------------------------------------------------------------------------------------------------
def _fused(tmp_path, V=19, kind="ngram"):
    pred, joiner = _build(V)
    lm = _ngram(tmp_path, V, 3)[0] if kind == "ngram" else _lstm_lm(V)
    return pred, joiner, dict(lm=lm, alpha=0.5, beta=0.3, ilm_weight=-0.25)


@pytest.mark.parametrize("kind", ["ngram", "lstm"])
def test_fp16_autocast(tmp_path, kind):
    V = 31
    pred, joiner = _build(V)
    lm, ref_lm = _ngram(tmp_path, V, 3) if kind == "ngram" else (_lstm_lm(V),) * 2
    enc = torch.randn(3, 8, 32, device="cuda")
    lens = torch.tensor([8, 5, 2])
    with torch.autocast("cuda", dtype=torch.float16):
        got = RNNTDecoder(pred, joiner, beam_size=4, lm_module=lm, alpha=0.4, beta=0.2, est_ilm=True,
                          ilm_weight=-0.3)(enc, lens)
        ref = cat_decode_fused(enc, lens, pred, joiner, 4, lm=ref_lm, alpha=0.4, beta=0.2, ilm_weight=-0.3)
    _compare(got, ref, 1e-3)


@pytest.mark.parametrize("kind", ["ngram", "lstm"])
def test_device_lengths_nan_past_the_end_and_repeat_bits(tmp_path, kind):
    pred, joiner, kw = _fused(tmp_path, kind=kind)
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


def test_scratch_contents_do_not_matter(tmp_path):
    pred, joiner, kw = _fused(tmp_path)
    enc = torch.randn(2, 6, 32, device="cuda")
    lens = torch.tensor([6, 3])
    a = rnnt_beam_search(enc, lens, pred, joiner, beam_size=8, **kw)
    for fill in (float("nan"), -1.0):   # what the caching allocator hands out next holds garbage
        junk = torch.full((1 << 24,), fill, device="cuda")
        del junk
        b = rnnt_beam_search(enc, lens, pred, joiner, beam_size=8, **kw)
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def test_side_stream(tmp_path):
    pred, joiner, kw = _fused(tmp_path)
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
    pred, joiner, kw = _fused(tmp_path, kind=kind)
    enc = torch.randn(2, 6, 32, device="cuda")
    for lens in (torch.tensor([6, 2]), torch.tensor([6, 2], device="cuda")):
        rnnt_beam_search(enc, lens, pred, joiner, beam_size=4, **kw)   # warm-up (uploads the LM)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            rnnt_beam_search(enc, lens, pred, joiner, beam_size=4, **kw)
        finally:
            torch.cuda.set_sync_debug_mode(0)
