"""GPU: the CTC-T beam search (``cat_b200.ctct_decode``), step by step through the C ABI against ``beam_ref``, against the
CTC-T loss on the GPU, and end to end against the restatement of CAT's decoder (tests/ctct_decode_oracle.py)."""
import numpy as np
import pytest
import torch

import warp_ctct
from cat_b200 import _lib
from cat_b200.ctct_decode import CTCTDecoder, ctct_beam_search
from ctct_decode_oracle import beam_ref, cat_decode
from rnnt_decode_oracle import CatJoiner, EmbeddingPredictor, JointNet, LogAdd, LSTMPredictor

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


def _rounded(x, dt):
    return torch.tensor(np.asarray(x, dtype=np.float32)).to(dt).float().numpy().astype(np.float64)


def _drive(mode, dname, N, T, B, V, lens, seed, blank=0, scale=2.0, row_fn=None):
    """Runs the C ABI frame by frame, each live slot's row built from the prefix read back from the step outputs (row_fn(t,
    prefix) in place of the random rows if given).  Returns (per utterance the final beam [(prefix, fp64 score)] in slot
    order, the finish outputs, the kernel's rows as lp(n, t, prefix), the kernel's input row as kernel_row(n, t, prefix))."""
    dt, code = _DT[dname]

    def draw(*key):
        return np.random.default_rng(hash((seed,) + key) & 0xffffffff).standard_normal(V) * scale

    f = np.stack([np.stack([_rounded(draw(-1, n, t), dt) for t in range(T)]) for n in range(N)]) if mode == 2 else None

    def kernel_row(n, t, p):
        if row_fn is not None:
            return _rounded(row_fn(t, p), dt)
        z = draw(n, t, *p)
        if mode == 0:
            z = z - np.logaddexp.reduce(z)
        return _rounded(z, dt)

    def lp(n, t, p):
        z = kernel_row(n, t, p)
        if mode == 0:
            return z
        if mode == 2:
            z = (np.float32(f[n, t]) + np.float32(z)).astype(np.float64)
        return z - np.logaddexp.reduce(z)

    L = _lib.lib()
    dev = torch.device("cuda")
    par, tok, nod = (torch.empty((N, B), dtype=torch.int32, device=dev) for _ in range(3))
    sc = torch.empty((N, B), dtype=torch.float64, device=dev)
    ws = torch.empty(int(L.ccb_ctct_beam_ws_bytes(N, T, B)), dtype=torch.uint8, device=dev)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    fd = torch.tensor(f, dtype=torch.float32).to(dt).to(dev).contiguous() if mode == 2 else None
    assert L.ccb_ctct_beam_init(N, T, B, ws.data_ptr(), par.data_ptr(), tok.data_ptr(), nod.data_ptr(), sc.data_ptr(),
                                None) == 0, _lib.last_error()
    prefixes = [[()] + [None] * (B - 1) for _ in range(N)]
    node_of = [{(): 0} for _ in range(N)]
    for t in range(T):
        rows = np.full((N * B, V), np.nan, dtype=np.float32)   # dead slots' rows are never read
        for n in range(N):
            for q, p in enumerate(prefixes[n]):
                if p is not None:
                    rows[n * B + q] = kernel_row(n, t, p)
        rt = torch.tensor(rows).to(dt).to(dev).contiguous()
        rc = L.ccb_ctct_beam_step(rt.data_ptr(), fd.data_ptr() if fd is not None else None, code, mode, N, T, B, V, t,
                                  lens_d.data_ptr(), blank, ws.data_ptr(), par.data_ptr(), tok.data_ptr(), nod.data_ptr(),
                                  sc.data_ptr(), None)
        assert rc == 0, _lib.last_error()
        P, K, D, S = (x.cpu().numpy() for x in (par, tok, nod, sc))
        for n in range(N):
            if t >= lens[n]:
                assert (P[n] == np.arange(B)).all() and (K[n] == -1).all()
                continue
            old, new = prefixes[n], []
            for q in range(B):
                if S[n, q] == -np.inf:
                    assert D[n, q] == -1 and P[n, q] == q and K[n, q] == -1
                    new.append(None)
                    continue
                p = old[P[n, q]] + ((int(K[n, q]),) if K[n, q] >= 0 else ())
                assert node_of[n].setdefault(p, int(D[n, q])) == D[n, q], "one trie node per prefix"
                new.append(p)
            live = [p for p in new if p is not None]
            assert len(set(live)) == len(live) and new[:len(live)] == live
            prefixes[n] = new
    S = sc.cpu().numpy()
    beams = [[(p, S[n, q]) for q, p in enumerate(prefixes[n]) if p is not None] for n in range(N)]
    tokens = torch.empty((N, B, T), dtype=torch.int32, device=dev)
    lengths = torch.empty((N, B), dtype=torch.int32, device=dev)
    scores = torch.empty((N, B), dtype=torch.float32, device=dev)
    assert L.ccb_rnnt_beam_finish(N, T, B, B, ws.data_ptr(), nod.data_ptr(), sc.data_ptr(), tokens.data_ptr(),
                                  lengths.data_ptr(), scores.data_ptr(), None) == 0, _lib.last_error()
    return beams, (tokens.cpu().numpy(), lengths.cpu().numpy(), scores.cpu().numpy()), lp, kernel_row


def _check_finish(beam, tokens, lengths, scores, B):
    """the finish of a ranked beam: slot order, the kernel's own fp64 scores rounded"""
    for k in range(B):
        if k < len(beam):
            p, s = beam[k]
            assert lengths[k] == len(p) and tuple(tokens[k, :lengths[k]]) == p
            assert (tokens[k, lengths[k]:] == -1).all()
            assert scores[k] == np.float32(s)
        else:
            assert lengths[k] == -1 and (tokens[k] == -1).all() and scores[k] == -np.inf


@pytest.mark.parametrize("dname", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N, T, B, V, blank", [(3, 6, 4, 37, 0), (2, 5, 16, 300, 0), (2, 3, 16, 4232, 0),
                                               (2, 4, 1, 9, 0), (2, 5, 8, 5, 0), (2, 5, 4, 37, 11), (2, 4, 16, 300, 299),
                                               (1, 2, 128, 4232, 0)])
def test_step_matches_beam_ref(mode, dname, N, T, B, V, blank):
    lens = ([T, max(T - 2, 1)] + [0] * N)[:N]
    beams, (tokens, lengths, scores), lp, _ = _drive(mode, dname, N, T, B, V, lens, seed=V + 7 * mode + blank, blank=blank)
    tol = (lambda s: 1e-12 * (1 + abs(s))) if mode == 0 else (lambda s: 1e-5 * (1 + abs(s)))
    for n in range(N):
        ref = beam_ref(lens[n], V, B, lambda t, p: lp(n, t, p), blank=blank)
        assert [p for p, _ in beams[n]] == [p for p, _ in ref], n   # the beam in rank order
        for (_, g), (p, s) in zip(beams[n], ref):
            assert abs(g - s) <= tol(s), (n, p, g, s)
        _check_finish(beams[n], tokens[n], lengths[n], scores[n], B)


def _fold_rows(t, p):
    # tests/test_ctct_decode_dispatch.py::fold_rows: an extension folded into a later entry's stay, whose target ties
    # another one exactly and ranks first by the extension's key
    if t == 0:
        return np.log([0.6, 0.3, 0.1])
    if p == ():
        return np.log([0.2, 0.4, 0.4])
    return np.array([-np.inf, -np.inf, 0.0])


def _repeat_rows(t, p):
    # (1,) enters frame 2 with b / s = 0.7; there its row ranks the repeat 1 first (0.4), 2 (0.3) second, 3 (0.29) third,
    # but by path score b lp[1] = 0.28 s < s lp[3]
    if t == 0:
        return np.log([0.001, 0.997, 0.001, 0.001])
    if p != (1,):
        return np.log(np.full(4, 0.25))
    return np.log([0.7, 0.2998, 1e-4, 1e-4]) if t == 1 else np.log([0.01, 0.4, 0.3, 0.29])


def _integer_rows(V):
    # integer log-probs: many equal row values (the top-k's ties) and exactly equal sums (the selection's ties)
    return lambda t, p: -1.0 - (np.arange(V) + len(p) + t) % 3


@pytest.mark.parametrize("case, V, T, B", [("fold", 3, 2, 2), ("integer", 6, 3, 1), ("integer", 6, 3, 3),
                                           ("integer", 6, 4, 8), ("integer", 40, 3, 16)])
def test_exact_ties(case, V, T, B):
    fn = _fold_rows if case == "fold" else _integer_rows(V)
    beams, _, lp, _ = _drive(0, "fp32", 1, T, B, V, [T], seed=0, row_fn=fn)
    ref = beam_ref(T, V, B, lambda t, p: lp(0, t, p))
    assert [p for p, _ in beams[0]] == [p for p, _ in ref]
    for (_, g), (_, s) in zip(beams[0], ref):
        assert g == pytest.approx(s, rel=1e-14, abs=1e-14)
    if case == "fold":
        assert [p for p, _ in beams[0]] == [(1, 2), (1,)]


def test_candidates_are_ranked_by_row_value():
    # tests/test_ctct_decode_dispatch.py::repeat_rows: ranked by path score, the repeat of (1,)'s last token would fall out
    # of the top-2 and token 3 take its place
    beams, _, lp, _ = _drive(0, "fp32", 1, 3, 2, 4, [3], seed=0, row_fn=_repeat_rows)
    ref = beam_ref(3, 4, 2, lambda t, p: lp(0, t, p))
    assert [p for p, _ in beams[0]] == [p for p, _ in ref] == [(1, 2), (1, 1)]
    for (_, g), (_, s) in zip(beams[0], ref):
        assert abs(g - s) <= 1e-12 * (1 + abs(s))


@pytest.mark.parametrize("blank", [0, 2])
@pytest.mark.parametrize("T, V", [(3, 4), (4, 3), (2, 6)])
def test_exhaustive_beam_equals_the_ctct_loss(T, V, blank):
    # with B >= V - 1 and B >= the number of prefixes nothing is pruned: each prefix's score is log P of its lattice, which
    # the CTC-T loss computes from the same logits by an independent kernel
    B = 128
    beams, _, _, kernel_row = _drive(1, "fp32", 1, T, B, V, [T], seed=3 + blank, blank=blank)
    beam = beams[0]
    assert len(beam) < B
    Umax = max(len(p) for p, _ in beam)
    x = np.zeros((len(beam), T, Umax + 1, V), dtype=np.float32)
    labels = np.zeros((len(beam), max(Umax, 1)), dtype=np.int32)
    for i, (p, _) in enumerate(beam):
        for t in range(T):
            for u in range(len(p) + 1):
                x[i, t, u] = kernel_row(0, t, p[:u])
        labels[i, :len(p)] = p
    costs = warp_ctct.ctct_loss(torch.tensor(x, device="cuda"), torch.tensor(labels, device="cuda"),
                                torch.full((len(beam),), T, dtype=torch.int32, device="cuda"),
                                torch.tensor([len(p) for p, _ in beam], dtype=torch.int32, device="cuda"),
                                reduction="none", blank=blank, compact=False, from_logits=True).double().cpu().numpy()
    for (p, s), c in zip(beam, costs):
        assert abs(s + c) <= 1e-5 * (1 + abs(c)), (p, s, -c)
    assert abs(np.logaddexp.reduce([s for _, s in beam])) <= 1e-5


# ---- end to end ---------------------------------------------------------------------------------------------------------
def _build(pname, jname, V, H=32, seed=0):
    torch.manual_seed(seed)
    Hp = V if jname == "logadd" else H
    pred = LSTMPredictor(V, Hp) if pname == "lstm" else EmbeddingPredictor(V, H, Hp)
    joiner = {"jointnet": lambda: JointNet(H, Hp, V, H), "logadd": LogAdd, "cat": lambda: CatJoiner(H, Hp, V)}[jname]()
    for m in (pred, joiner):
        for p in m.parameters():
            p.data.mul_(3.0)   # spread the scores so that ranks are well separated
    He = V if jname == "logadd" else H
    return pred.cuda().eval(), joiner.cuda().eval(), He


def _compare(got, ref):
    for (gh, gs), (rh, rs) in zip(got, ref):
        assert gh == rh
        for a, b in zip(gs, rs):
            assert abs(a - b) <= 1e-4 * (1 + abs(b)), (a, b)


@pytest.mark.parametrize("pname", ["lstm", "embedding"])
@pytest.mark.parametrize("jname", ["jointnet", "logadd", "cat"])
@pytest.mark.parametrize("B, nbest", [(1, -1), (4, -1), (4, 2), (16, 5)])
def test_decoder_matches_cat_restatement(pname, jname, B, nbest):
    V = 29
    pred, joiner, He = _build(pname, jname, V)
    torch.manual_seed(5)
    enc = torch.randn(5, 9, He, device="cuda")
    lens = torch.tensor([9, 1, 0, 6, 9])
    got = CTCTDecoder(pred, joiner, beam_size=B, nbest=nbest)(enc, lens)
    ref = cat_decode(enc, lens, pred, joiner, B, B if nbest == -1 else nbest)
    _compare(got, ref)
    assert got[2] == ([[]], [0.0])


def test_blank_not_zero_end_to_end():
    pred, joiner, He = _build("lstm", "jointnet", 23)
    enc = torch.randn(3, 7, He, device="cuda")
    lens = torch.tensor([7, 3, 5])
    _compare(CTCTDecoder(pred, joiner, blank_id=5, bos_id=5, beam_size=4)(enc, lens),
             cat_decode(enc, lens, pred, joiner, 4, blank=5))


def test_device_lengths_and_full_length_default():
    pred, joiner, He = _build("lstm", "jointnet", 23)
    enc = torch.randn(3, 7, He, device="cuda")
    lens = torch.tensor([7, 3, 5])
    dec = CTCTDecoder(pred, joiner, beam_size=4)
    a = dec(enc, lens)
    assert dec(enc, lens.cuda()) == a
    assert dec(enc, lens.to(torch.int32).cuda()) == a
    _compare(dec(enc), cat_decode(enc, torch.tensor([7, 7, 7]), pred, joiner, 4))
    assert dec(enc[:, :0], torch.tensor([0, 0, 0])) == [([[]], [0.0])] * 3


def test_fp16_autocast():
    pred, joiner, He = _build("lstm", "jointnet", 31)
    enc = torch.randn(3, 8, He, device="cuda")
    lens = torch.tensor([8, 5, 2])
    with torch.autocast("cuda", dtype=torch.float16):
        got = CTCTDecoder(pred, joiner, beam_size=4)(enc, lens)
        ref = cat_decode(enc, lens, pred, joiner, 4)
    _compare(got, ref)


def test_cat_sized():
    V, H = 4232, 512
    torch.manual_seed(0)
    pred = LSTMPredictor(V, H).cuda().eval()
    joiner = JointNet(H, H, V, H).cuda().eval()
    for p in joiner.fc.parameters():
        p.data.mul_(4.0)
    enc = torch.randn(2, 12, H, device="cuda")
    lens = torch.tensor([12, 7])
    _compare(CTCTDecoder(pred, joiner, beam_size=16)(enc, lens), cat_decode(enc, lens, pred, joiner, 16))


# ---- properties ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jname", ["jointnet", "logadd", "cat"])
def test_nan_past_the_end_changes_nothing_and_calls_repeat_bits(jname):
    pred, joiner, He = _build("lstm", jname, 19)
    enc = torch.randn(3, 8, He, device="cuda")
    lens = torch.tensor([8, 4, 6])
    a = ctct_beam_search(enc, lens, pred, joiner, beam_size=4)
    enc2 = enc.clone()
    enc2[1, 4:] = float("nan")
    enc2[2, 6:] = float("nan")
    b = ctct_beam_search(enc2, lens, pred, joiner, beam_size=4)
    c = ctct_beam_search(enc, lens, pred, joiner, beam_size=4)
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_side_stream():
    pred, joiner, He = _build("lstm", "logadd", 17)
    enc = torch.randn(2, 6, He, device="cuda")
    lens = torch.tensor([6, 3])
    a = ctct_beam_search(enc, lens, pred, joiner, beam_size=4)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = ctct_beam_search(enc, lens, pred, joiner, beam_size=4)
    torch.cuda.current_stream().wait_stream(s)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("jname", ["jointnet", "logadd"])
def test_no_host_synchronisation(jname):
    pred, joiner, He = _build("lstm", jname, 21)
    enc = torch.randn(2, 6, He, device="cuda")
    for lens in (torch.tensor([6, 2]), torch.tensor([6, 2], device="cuda")):
        ctct_beam_search(enc, lens, pred, joiner, beam_size=4)   # warm-up
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            ctct_beam_search(enc, lens, pred, joiner, beam_size=4)
        finally:
            torch.cuda.set_sync_debug_mode(0)
