"""GPU: the kernels at the shapes that select their less common branches -- vocabularies of 300 to 25 000 classes, label
sequences of 1 023 and 1 100 tokens, batches of 257 to 512 utterances in one call -- against the fp64 oracle.

The rest of the suite runs phone-sized vocabularies (V <= 218), label sequences of at most 400 and at most 200 utterances
per den call.  Each case here names the branch it runs; the den cases first check, through ccb_plan_launch on this device's
SM count and opt-in shared memory, that the launch they make is the one they claim.

Tolerances are the suite's (BASELINE.json north_star): loss 1e-4 relative, gradients 1e-3 absolute (occupancies in [0, 1]).
"""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3
SAME_RTOL = 1e-6      # forward-only against the training path, one slicing against another: den atomics only

FIELDS = ("tier", "lanes", "U", "batch", "w1_smem", "Npad", "tile_rows", "gacc_rows", "arcs_off", "ring_off", "bar_off",
          "w1_off", "abar_off", "aring_off", "total")


@pytest.fixture(scope="module")
def wide_graphs(tmp_path_factory):
    """Den graphs with thousands of labels and few states per label (tests/test_den_launch.py pins their launches at
    132 CTAs): G4k, G20k (T-compose-LM shaped) and an unstructured graph with 2 500 labels."""
    from cat_b200 import fst
    d = tmp_path_factory.mktemp("wide_graphs")
    out = {}
    for name, g, V in (("G4k", fst.make_synthetic_den(3000, 8, 4000, seed=7), 4000),
                       ("G20k", fst.make_synthetic_den(6000, 8, 20000, seed=7), 20000),
                       ("random_2500", fst.make_random_den(3000, 30000, 2500, seed=5), 2500)):
        fst.write_fst(str(d / f"{name}.fst"), g)
        out[name] = (str(d / f"{name}.fst"), g, V)
    return out


def _graph(tmp_graphs, wide_graphs, name):
    return tmp_graphs[name] if name in tmp_graphs else wide_graphs[name]


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _launch(path, N, backward):
    """The den launch a call of N utterances makes on this device (den_launch.h ChooseDenLaunch, no test hooks)."""
    from cat_b200 import _lib
    props = torch.cuda.get_device_properties(0)
    L = _lib.lib()
    h = L.ccb_plan_create(path.encode(), props.multi_processor_count, 16)
    assert h, _lib.last_error()
    try:
        out = (C.c_long * len(FIELDS))()
        assert L.ccb_plan_launch(h, N, int(backward), props.shared_memory_per_block_optin, 0, out) == 0, _lib.last_error()
        return dict(zip(FIELDS, out))
    finally:
        L.ccb_plan_destroy(h)


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32)


def _close(a, b, rtol=LOSS_RTOL):
    assert abs(a - b) <= rtol * max(1.0, abs(b)), (a, b)


def _ragged(N, T, seed, zero=True):
    """Lengths in [2, T] with T first, then 0 (or 2) and 1 at fixed places, N-1 one short of T.  (A length-0 utterance has
    logZ = -inf on these graphs, which makes a batch loss NaN: the fused cases leave it out.)"""
    lens = np.random.default_rng(seed).integers(2, T + 1, size=N).astype(np.int32)
    lens[0], lens[1], lens[N // 2], lens[N - 1] = T, 0 if zero else 2, 1, T - 1
    return lens


def _lane_subset(N):
    """One utterance in every 32-lane group (at a different lane in each), the first two and the last."""
    sub = {32 * k + (7 * k + 3) % min(32, N - 32 * k) for k in range((N + 31) // 32)}
    return np.array(sorted(sub | {0, 1, N // 2, N - 1}))


def _labels_of(labels, ly, sub):
    off = np.concatenate([[0], np.cumsum(ly)])
    return np.concatenate([labels[off[n]:off[n + 1]] for n in sub]).astype(np.int32)


def _rows_past_len_zero(grad, lens):
    """grad (N,T,V) on the device: every row t >= lens[n] is exactly zero."""
    T = grad.shape[1]
    past = torch.arange(T, device=grad.device)[None, :] >= torch.tensor(lens, device=grad.device)[:, None]
    assert not bool(grad[past].any())


def _fused_vs_oracle(g, y, labels, lens, ly, lamb, sub=None):
    """CTC_CRF_LOSS (loss + gradient through autograd) and _C.ctc_crf_loss_fwd's parts against oracle.ctc_crf on the
    utterances `sub` (all by default); the no_grad loss against the training loss.  Returns the training loss."""
    import ctc_crf
    from oracle import oracle
    N = y.shape[0]
    sub = np.arange(N) if sub is None else sub
    x = torch.tensor(y, device="cuda").requires_grad_(True)
    crit = ctc_crf.CTC_CRF_LOSS(lamb=lamb, size_average=False)
    loss = crit(x, _i32(labels), _i32(lens), _i32(ly))
    loss.backward()
    _rows_past_len_zero(x.grad, lens)
    _, _, parts = ctc_crf._C.ctc_crf_loss_fwd(x.detach(), _i32(labels), _i32(lens), _i32(ly), lamb, False, want_parts=True)
    parts = parts.cpu().numpy()
    with torch.no_grad():
        ev = crit(x.detach(), _i32(labels), _i32(lens), _i32(ly))
    _close(float(ev.item()), float(loss.item()), SAME_RTOL)
    oloss, ograd, oparts = oracle.ctc_crf(g, y[sub], _labels_of(labels, ly, sub), lens[sub], ly[sub], lamb,
                                          size_average=False, fast=True)
    if len(sub) == N:
        _close(float(loss.item()), oloss)
    np.testing.assert_allclose(parts[:N][sub], oparts["logz_alpha"], rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(parts[N:][sub], oparts["logp_ctc"], rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(x.grad[torch.tensor(sub, device="cuda")].cpu().numpy() - ograd).max() < GRAD_ATOL
    return float(loss.item())


# ---------------------------------------------------------------------------------------------------------------------
# a. large vocabularies through the fused loss
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,V", [("tlm_mid", 600), ("G4k", 4000), ("G20k", 20000)])
def test_large_vocabulary_fused_loss(tmp_graphs, wide_graphs, name, V):
    """Numerator emission rows read from global memory every frame (ctc_alpha_beta_kernel, `!row_in_regs`): labels of at
    most 10 give Lmax + 1 = 11 -> 64 threads, and V > 4 x 64 = 256.  Occupancy kernel (LaunchCtcGamma) at 8 warps per CTA
    for V = 600 (8 x 600 x 4 B <= 48 KB), 2 for V = 4000, 1 warp with 80 KB of dynamic shared memory for V = 20000.
    On tlm_mid the logits are wider than the graph's 40 labels: columns 40..599 carry the numerator's occupancy only."""
    from oracle import oracle
    path, g, _ = _graph(tmp_graphs, wide_graphs, name)
    N, T = 8, 60
    lens = np.array([60, 60, 55, 41, 33, 20, 9, 3], np.int32)
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=61, lens=lens)
    assert ly.max() == 10 and labels.max() >= 40
    ctx = _ctx(path)
    _fused_vs_oracle(g, y, labels, lens, ly, 0.1)
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# b. a wide label accumulator in the den backward pass
# ---------------------------------------------------------------------------------------------------------------------
def test_wide_label_accumulator(wide_graphs):
    """Den backward with a shared-memory label accumulator of hundreds of rows: on G20k a CTA tile spans 213 labels at
    132 CTAs (273 at 114), and nearly every row end changes label (the `new_label` branch of do_row, the forward `new_label`
    emission refresh).  N = 64 where 64 lanes of those rows fit in 64 KB, else N = 32."""
    from oracle import oracle
    path, g, V = wide_graphs["G20k"]
    N = next(n for n in (64, 32) if _launch(path, n, True)["gacc_rows"] > 0)
    L = _launch(path, N, True)
    assert L["Npad"] == N and L["gacc_rows"] >= 200, L
    T = 30
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=62, lens=_ragged(N, T, seed=62, zero=False))
    ctx = _ctx(path)
    _fused_vs_oracle(g, y, labels, lens, ly, 0.1, sub=np.array([0, 1, N // 2, N - 2, N - 1]))
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# c. global-atomic occupancies and the widest batches through _C.gpu_den
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,N,gacc", [
    ("G20k", 100, False),         # Npad 128: 213 rows x 128 lanes x 4 B > 64 KB -> flush_gsum adds into the gradient
    ("G20k", 200, False),         # Npad 256
    ("G4k", 384, False),          # Npad 384: 3 forward lane groups at U = 4, 6 backward at U = 2
    ("G4k", 512, False),          # Npad 512: 4 / 8 lane groups, the kernels' widest batch
    ("tlm_mid", 384, True),       # the same widths with a 3-row accumulator
    ("tlm_mid", 512, True),
    ("random_2500", 300, True),   # unstructured, states split by in-label, 2 500 labels
])
def test_den_wide_batches(tmp_graphs, wide_graphs, name, N, gacc):
    """_C.gpu_den (reference signature): logZ from alpha and from beta and the occupancies against oracle.den, on every
    utterance or on one per 32-lane group plus the first, the last and those of length 0 and 1."""
    from oracle import oracle
    from cat_b200 import _C
    path, g, V = _graph(tmp_graphs, wide_graphs, name)
    Npad = 128 * ((N + 127) // 128)
    fwd, bwd = _launch(path, N, False), _launch(path, N, True)
    assert (fwd["Npad"], fwd["U"], bwd["Npad"], bwd["U"]) == (Npad, 4, Npad, 2), (fwd, bwd)
    assert (bwd["gacc_rows"] > 0) == gacc, bwd
    T = 16
    lens = _ragged(N, T, seed=N)
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=63, lens=lens)
    ctx = _ctx(path)
    logits = torch.tensor(y, device="cuda")
    grad = torch.zeros_like(logits)
    ca = torch.zeros(N, device="cuda")
    cb = torch.zeros(N, device="cuda")
    _C.gpu_den(logits, grad, _i32(lens).cuda(), ca, cb)
    _rows_past_len_zero(grad, lens)
    sub = np.arange(N) if N * T * V <= 512 * 16 * 40 else _lane_subset(N)
    la, lb, gd = oracle.den(g, y[sub], lens[sub], fast=True)
    np.testing.assert_allclose(ca.cpu().numpy()[sub], la, rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(cb.cpu().numpy()[sub], lb, rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(grad[torch.tensor(sub, device="cuda")].cpu().numpy() - gd).max() < GRAD_ATOL
    del ctx


def test_den_rejects_513_utterances(tmp_graphs):
    """513 utterances are more than one den call takes (16 warps x 32 lanes): a RuntimeError from the host-side check in
    CheckDen, before anything is launched."""
    from cat_b200 import _C
    path, _, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 513, 4
    logits = torch.full((N, T, V), -float(np.log(V)), device="cuda")
    with pytest.raises(RuntimeError, match="512 utterances"):
        _C.gpu_den(logits, torch.zeros_like(logits), torch.full((N,), T, dtype=torch.int32, device="cuda"),
                   torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda"))
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# d. the fused loss with 257..512 utterances in one call
# ---------------------------------------------------------------------------------------------------------------------
def test_fused_300_utterances_in_one_call(tmp_graphs, monkeypatch):
    """CTC_CRF_LOSS with MAX_UTTS_PER_CALL = 512: 300 utterances in one native call (den Npad 384, forward U = 4, backward
    U = 2, label accumulator present) equal the default 64-wide slicing and the oracle."""
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    N, T = 300, 20
    fwd, bwd = _launch(path, N, False), _launch(path, N, True)
    assert (fwd["Npad"], fwd["U"], bwd["U"]) == (384, 4, 2) and bwd["gacc_rows"] > 0, (fwd, bwd)
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=64, lens=_ragged(N, T, seed=64, zero=False))
    ctx = _ctx(path)

    def run():
        x = torch.tensor(y, device="cuda").requires_grad_(True)
        loss = ctc_crf.CTC_CRF_LOSS(lamb=0.1)(x, _i32(labels), _i32(lens), _i32(ly))
        loss.backward()
        return float(loss.item()), x.grad

    ref_loss, ref_grad = run()
    seen = []
    plan_slices = _C._plan_slices
    monkeypatch.setattr(_C, "_plan_slices", lambda *a: seen.append(plan_slices(*a)) or seen[-1])
    monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 512)
    loss, grad = run()
    assert [(s[0], s[1]) for s in seen[-1]] == [(0, N)], seen[-1]
    _close(loss, ref_loss, SAME_RTOL)
    assert float((grad - ref_grad).abs().max()) < 1e-6
    _rows_past_len_zero(grad, lens)
    sub = _lane_subset(N)
    oloss, ograd, _ = oracle.ctc_crf(g, y[sub], _labels_of(labels, ly, sub), lens[sub], ly[sub], 0.1, size_average=False,
                                     fast=True)
    assert np.abs(grad[torch.tensor(sub, device="cuda")].cpu().numpy() * N - ograd).max() < GRAD_ATOL
    _, _, parts = _C.ctc_crf_loss_fwd(torch.tensor(y, device="cuda"), _i32(labels), _i32(lens), _i32(ly), 0.1, True,
                                      want_parts=True)
    la, _, _ = oracle.den(g, y[sub], lens[sub], fast=True)
    np.testing.assert_allclose(parts.cpu().numpy()[:N][sub], la, rtol=LOSS_RTOL, atol=1e-4)
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# e. label sequences of 1 024 tokens and more
# ---------------------------------------------------------------------------------------------------------------------
def _long_labels(V, Lmax, T, blank=0, seed=0):
    """Three utterances of T, T and T - 150 frames: Lmax labels with a few repeats; Lmax labels with exactly T - Lmax
    repeats (L + repeats == T: one path through the lattice); Lmax - 300 labels.  Labels avoid `blank`."""
    rng = np.random.default_rng(seed)
    tokens = np.array([k for k in range(V) if k != blank])

    def seq(L, n_rep):
        rep = set(rng.choice(np.arange(1, L), size=n_rep, replace=False).tolist())
        lab = [int(rng.choice(tokens))]
        for i in range(1, L):                                 # a repeat where chosen, a different token elsewhere
            k = lab[-1]
            while k == lab[-1] and i not in rep:
                k = int(rng.choice(tokens))
            lab.append(k)
        lab = np.array(lab)
        assert int((lab[1:] == lab[:-1]).sum()) == n_rep
        return lab

    lens = np.array([T, T, T - 150], np.int32)
    ly = np.array([Lmax, Lmax, Lmax - 300], np.int32)
    labels = np.concatenate([seq(Lmax, 5), seq(Lmax, T - Lmax), seq(Lmax - 300, 3)]).astype(np.int32)
    return labels, lens, ly


def _torch_ctc_logp(y, labels, lens, ly, blank):
    """log p(l|x) by torch.nn.functional.ctc_loss in fp64 on the CPU."""
    lp = torch.tensor(y, dtype=torch.float64).transpose(0, 1)
    nll = torch.nn.functional.ctc_loss(lp, torch.tensor(labels, dtype=torch.long), torch.tensor(lens, dtype=torch.long),
                                       torch.tensor(ly, dtype=torch.long), blank=blank, reduction="none")
    return -nll.numpy()


@pytest.mark.parametrize("Lmax,V,blank", [
    (1023, 300, 0),      # 1 024 threads, one cell pair each; V <= 4 x 1024: emission row prefetched into registers
    (1100, 300, 0),      # 1 024 threads, threads 0..76 own a second cell pair (cells i >= NT); row in registers
    (1023, 6000, 0),     # V > 4 x 1024: row read from global memory every frame
    (1100, 6000, 0),     # both: cells past the first 1 024 and the row from global memory
    (1100, 300, 299),    # blank = V - 1
])
def test_long_label_sequences_ctc(Lmax, V, blank):
    """Numerator at Lmax >= 1 023: blockDim = min(1024, round32(Lmax + 1)) = 1 024, so Lmax = 1 100 loops over 1 101 cells
    per lattice row (alpha, beta); the emission row sits in registers when V <= 4 x blockDim.  _C.gpu_ctc (reference
    signature, (T,N,V), blank chosen by the caller) and WARP_CTC_LOSS against oracle.ctc and torch's fp64 ctc_loss;
    the no_grad loss against the training loss."""
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C
    N, T = 3, 1300
    labels, lens, ly = _long_labels(V, Lmax, T, blank=blank, seed=Lmax + V)
    y, _, _, _ = oracle.synth_batch(N, T, V, seed=65, lens=lens)
    lp, gc = oracle.ctc(y, labels, ly, lens, blank=blank)
    np.testing.assert_allclose(_torch_ctc_logp(y, labels, lens, ly, blank), lp, rtol=1e-9)   # the two references agree
    act = torch.tensor(y, device="cuda").transpose(0, 1).contiguous()
    grads = torch.zeros_like(act)
    costs = torch.zeros(N)
    _C.gpu_ctc(act, grads, _i32(labels), _i32(ly), _i32(lens), N, costs, blank)
    np.testing.assert_allclose(costs.numpy(), lp, rtol=LOSS_RTOL)
    assert np.abs(grads.transpose(0, 1).cpu().numpy() - gc).max() < GRAD_ATOL
    del act, grads
    if blank != 0:                                  # WARP_CTC_LOSS takes blank 0 (the reference's signature)
        return
    x = torch.tensor(y, device="cuda").requires_grad_(True)
    crit = ctc_crf.WARP_CTC_LOSS(size_average=False)
    loss = crit(x, _i32(labels), _i32(lens), _i32(ly))
    loss.backward()
    _close(float(loss.item()), -lp.sum())
    assert np.abs(x.grad.cpu().numpy() + gc).max() < GRAD_ATOL
    _rows_past_len_zero(x.grad, lens)
    with torch.no_grad():
        ev = crit(x.detach(), _i32(labels), _i32(lens), _i32(ly))
    _close(float(ev.item()), float(loss.item()), SAME_RTOL)


def test_long_label_sequences_fused(wide_graphs):
    """CTC_CRF_LOSS on G4k with label sequences of 1 100 tokens over 1 300 frames: the numerator's looped cells (blockDim
    1 024) and its emission row from global memory (V = 4 000 > 4 x 1 024), next to a den walk of 1 300 frames."""
    from oracle import oracle
    path, g, V = wide_graphs["G4k"]
    T = 1300
    labels, lens, ly = _long_labels(V, 1100, T, seed=66)
    y, _, _, _ = oracle.synth_batch(3, T, V, seed=66, lens=lens)
    ctx = _ctx(path)
    _fused_vs_oracle(g, y, labels, lens, ly, 0.1)
    del ctx


def _viterbi_np(y, lab, blank=0):
    """Best path over the blank-expanded lattice, vectorised over the cells (fp64): tokens per frame and the path score.
    Ties go to the smaller back-pointer (stay < s-1 < s-2), as in the kernel."""
    T = y.shape[0]
    ext = np.full(2 * len(lab) + 1, blank, np.int64)
    ext[1::2] = lab
    S = len(ext)
    skip = np.zeros(S, bool)
    skip[2:] = (ext[2:] != blank) & (ext[2:] != ext[:-2])
    v = np.full(S, -np.inf)
    v[0] = y[0, blank]
    if S > 1:
        v[1] = y[0, ext[1]]
    bp = np.zeros((T, S), np.int64)
    cols = np.arange(S)
    for t in range(1, T):
        c1 = np.concatenate([[-np.inf], v[:-1]])
        c2 = np.where(skip, np.concatenate([[-np.inf, -np.inf], v[:-2]]), -np.inf)
        k = np.argmax(np.stack([v, c1, c2]), axis=0)
        v = np.stack([v, c1, c2])[k, cols] + y[t, ext]
        bp[t] = k
    s = S - 1 if S == 1 or v[S - 1] >= v[S - 2] else S - 2
    score = v[s]
    out = np.zeros(T, np.int64)
    for t in range(T - 1, -1, -1):
        out[t] = ext[s]
        s -= bp[t, s]
    return out, score


def test_long_label_sequences_align():
    """ctc_align (ctc_viterbi_kernel) with 1 100 labels: 1 024 threads, cells i >= 1 024 looped, against a vectorised
    fp64 Viterbi -- the path score, the path's own score where the path differs (ties), and the collapse to the labels."""
    import ctc_crf
    from oracle import oracle
    V, T = 300, 1300
    labels, lens, ly = _long_labels(V, 1100, T, seed=67)
    y, _, _, _ = oracle.synth_batch(3, T, V, seed=67, lens=lens)
    align, score = ctc_crf.ctc_align(torch.tensor(y, device="cuda"), _i32(labels), _i32(lens), _i32(ly))
    align, score = align.cpu().numpy(), score.cpu().numpy()
    off = np.concatenate([[0], np.cumsum(ly)])
    for n in range(3):
        lab = labels[off[n]:off[n + 1]]
        yn = y[n, :lens[n]].astype(np.float64)
        ref, sc = _viterbi_np(yn, lab)
        _close(float(score[n]), sc)
        assert (align[n, lens[n]:] == -1).all()
        got = align[n, :lens[n]]
        if not np.array_equal(got, ref):
            _close(float(yn[np.arange(lens[n]), got].sum()), sc)
        collapsed = [int(k) for i, k in enumerate(got) if k != 0 and (i == 0 or got[i - 1] != k)]
        assert collapsed == [int(k) for k in lab]


# ---------------------------------------------------------------------------------------------------------------------
# f. 16-bit raw logits at V = 20 000
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_raw_16bit_logits_large_vocabulary(wide_graphs, dtype):
    """CTC_CRF_LOSS's raw-logit entry (from_logits=True) on fp16 / bf16 logits at V = 20 000 on G20k: the frame
    log-normaliser over 20 000 16-bit classes, the numerator row from global memory, the one-warp occupancy kernel.
    Against the oracle fed the upcast values; every gradient row sums to ~0 (softmax Jacobian)."""
    import ctc_crf
    from oracle import oracle
    path, g, V = wide_graphs["G20k"]
    N, T = 8, 60
    _, labels, lens, ly = oracle.synth_batch(N, T, V, seed=68, lens=[60, 60, 55, 41, 33, 20, 9, 3])
    z = (4.0 * np.random.default_rng(68).standard_normal((N, T, V)) + 7.0).astype(np.float32)
    zt = torch.tensor(z, device="cuda").to(dtype)
    z64 = zt.double().cpu().numpy()
    y64 = z64 - (z64.max(-1, keepdims=True) + np.log(np.exp(z64 - z64.max(-1, keepdims=True)).sum(-1, keepdims=True)))
    ctx = _ctx(path)
    loss, grad, parts = ctc_crf._C.ctc_crf_loss_fwd(zt, _i32(labels), _i32(lens), _i32(ly), 0.1, True, want_parts=True,
                                                    from_logits=True)
    oloss, og, oparts = oracle.ctc_crf(g, y64.astype(np.float32), labels, lens, ly, 0.1, fast=True)
    odz = og - np.exp(y64) * og.sum(-1, keepdims=True)
    _close(float(loss.item()), oloss)
    parts = parts.cpu().numpy()
    np.testing.assert_allclose(parts[:N], oparts["logz_alpha"], rtol=LOSS_RTOL, atol=1e-3)
    np.testing.assert_allclose(parts[N:], oparts["logp_ctc"], rtol=LOSS_RTOL, atol=1e-3)
    gz = grad.cpu().numpy()
    assert np.abs(gz - odz).max() < GRAD_ATOL
    assert np.abs(gz.sum(-1)).max() < 1e-4
    _rows_past_len_zero(grad, lens)
    with torch.no_grad():
        ev = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=True)(zt, _i32(labels), _i32(lens), _i32(ly))
    _close(float(ev.item()), float(loss.item()), SAME_RTOL)
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# the numerator's vocabulary bound
# ---------------------------------------------------------------------------------------------------------------------
def test_numerator_vocabulary_bound():
    """The numerator stages two emission rows of V floats in at most 200 KB of shared memory: with labels of up to 20,
    V = 25 000 runs (against the oracle) and V = 32 000 raises a RuntimeError that names V and the largest V allowed
    (25 505 = (204 800 - 16 x 41 - 4 x 21 - 16) / 8)."""
    import ctc_crf
    from oracle import oracle
    N, T = 2, 30
    for V in (25000, 32000):
        y, _, lens, _ = oracle.synth_batch(N, T, V, seed=69, lens=[30, 24])
        ly = np.array([20, 12], np.int32)
        labels = np.random.default_rng(69).integers(1, V, size=int(ly.sum())).astype(np.int32)
        x = torch.tensor(y, device="cuda").requires_grad_(True)
        crit = ctc_crf.WARP_CTC_LOSS(size_average=False)
        if V == 32000:
            with pytest.raises(RuntimeError, match=r"V = 32000 .* at most 25505"):
                crit(x, _i32(labels), _i32(lens), _i32(ly))
            continue
        loss = crit(x, _i32(labels), _i32(lens), _i32(ly))
        loss.backward()
        lp, gc = oracle.ctc(y, labels, ly, lens)
        _close(float(loss.item()), -lp.sum())
        assert np.abs(x.grad.cpu().numpy() + gc).max() < GRAD_ATOL
