"""GPU parity tests (run on the H100; reference CUDA = oracle/_ref patched build, see oracle/Makefile): the CUDA path, called through the reference-facing surface
(ctc_crf.CTC_CRF_LOSS / _C.gpu_den / _C.gpu_ctc -> C ABI), against the fp64 oracle, the committed golden
vectors, and the reference's own CUDA code (oracle/_ref) on the same seeded inputs.

Tolerances (BASELINE.json north_star): loss 1e-4 relative, gradients 1e-3 (absolute; occupancies are in [0,1]).
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _run_ours(y, labels, lx, ly, lamb, size_average=True, dtype=torch.float32):
    import ctc_crf
    logits = torch.tensor(y, device="cuda", dtype=dtype).requires_grad_(True)
    crit = ctc_crf.CTC_CRF_LOSS(lamb=lamb, size_average=size_average)
    loss = crit(logits, torch.tensor(labels, dtype=torch.int32), torch.tensor(lx, dtype=torch.int32),
                torch.tensor(ly, dtype=torch.int32))
    loss.backward()
    return float(loss.item()), logits.grad.float().cpu().numpy()


def _close_loss(a, b, rtol=LOSS_RTOL):
    assert abs(a - b) <= rtol * max(1.0, abs(b)), (a, b)


def test_fixture_kat(fixture_fst, fixture_inputs):
    """The reference's own test input (test/main.py) -> survey/oracle known answers."""
    from oracle import oracle
    from cat_b200 import fst
    fi = fixture_inputs
    ctx = _ctx(fixture_fst)
    loss, grad = _run_ours(fi["y"], fi["labels"], fi["lx"], fi["ly"], fi["lamb"])
    _close_loss(loss, -2.47862480)
    oloss, ograd, _ = oracle.ctc_crf(fst.read_fst(fixture_fst), fi["y"], fi["labels"], fi["lx"], fi["ly"], fi["lamb"])
    _close_loss(loss, oloss)
    assert np.abs(grad - ograd).max() < GRAD_ATOL
    np.testing.assert_allclose(grad[0, 0], [0.658503, 0.311666, -0.980169, 0, 0], atol=2e-5)
    del ctx


@pytest.mark.parametrize("name,N,T,lens", [
    ("tlm_small", 3, 20, [20, 13, 7]),
    ("random_split", 3, 20, [20, 13, 7]),          # loader has to split states by in-label
    ("tlm_small", 5, 33, [33, 33, 1, 2, 17]),
    ("tlm_mid", 64, 40, None),                      # two utterances per lane
    ("tlm_mid", 33, 25, None),                      # ragged lane padding
    ("tlm_mid", 130, 12, None),                     # four utterances per lane, padded to 256
    ("tlm_mid", 200, 9, None),                      # ... and two lane groups per warp (Npad = 256)
])
def test_den_vs_oracle(tmp_graphs, name, N, T, lens):
    """_C.gpu_den (reference signature) vs the oracle: logZ from alpha, logZ from beta, occupancies."""
    from oracle import oracle
    from cat_b200 import _C
    path, g, V = tmp_graphs[name]
    ctx = _ctx(path)
    if lens is None:
        lens = np.maximum(1, T - (np.arange(N) * 7) % T).astype(np.int32)
        lens[0] = T
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=5, lens=lens)
    logits = torch.tensor(y, device="cuda")
    grad = torch.zeros_like(logits)
    ca = torch.zeros(N, device="cuda")
    cb = torch.zeros(N, device="cuda")
    _C.gpu_den(logits, grad, torch.tensor(lens, dtype=torch.int32).cuda(), ca, cb)
    la, lb, gd = oracle.den(g, y, lens)
    np.testing.assert_allclose(ca.cpu().numpy(), la, rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(cb.cpu().numpy(), lb, rtol=LOSS_RTOL, atol=1e-4)
    gn = grad.cpu().numpy()
    assert np.abs(gn - gd).max() < GRAD_ATOL
    for n in range(N):   # rows beyond the utterance stay untouched (den_calculate.cu:238)
        assert not gn[n, lens[n]:].any()
    del ctx


@pytest.mark.parametrize("N,T,V,lens,ly", [
    (4, 30, 12, [30, 22, 9, 5], [5, 3, 0, 5]),       # L=0 and T == L (+repeats) edge
    (3, 50, 40, [50, 41, 17], [8, 20, 1]),
    (2, 12, 6, [12, 3], [11, 5]),                     # one nearly-full lattice, one infeasible (L > T)
])
def test_ctc_vs_oracle(N, T, V, lens, ly):
    """_C.gpu_ctc (reference signature, (T,N,V) layout, host labels/costs) vs the oracle."""
    from oracle import oracle
    from cat_b200 import _C
    rng = np.random.default_rng(3)
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=9, lens=lens)
    ly = np.asarray(ly, np.int32)
    labels = rng.integers(1, V, size=int(ly.sum())).astype(np.int32)
    if ly[0] >= 3:
        labels[1] = labels[0]                          # force a repeat
    act = torch.tensor(y, device="cuda").transpose(0, 1).contiguous()
    grads = torch.zeros_like(act)
    costs = torch.zeros(N)
    _C.gpu_ctc(act, grads, torch.tensor(labels), torch.tensor(ly), torch.tensor(lens), N, costs, 0)
    lp, gc = oracle.ctc(y, labels, ly, lens)
    got = costs.numpy()
    for n in range(N):
        if np.isinf(lp[n]):
            assert np.isinf(got[n]) and got[n] < 0
        else:
            assert abs(got[n] - lp[n]) <= LOSS_RTOL * max(1.0, abs(lp[n]))
    assert np.abs(grads.transpose(0, 1).cpu().numpy() - gc).max() < GRAD_ATOL


@pytest.mark.parametrize("env", ["CCB_ARCS_IN_GLOBAL", "CCB_W1_IN_GLOBAL", "CCB_NO_PAIRS", "HUBS", "HUBS+CCB_ARCS_IN_GLOBAL",
                                 "CCB_NO_TMA", "CCB_ARCS_IN_GLOBAL+CCB_NO_TMA", "CCB_NO_MERGE", "CCB_NO_MERGE+CCB_NO_TMA",
                                 "CCB_NO_OWN", "CCB_NO_OWN+CCB_NO_TMA"])
def test_fallback_paths(tmp_graphs, monkeypatch, env):
    """Arc tiles streamed from global memory (graphs too large for shared memory: through per-warp bulk-copy rings next to
    the TMA row gathers, or -- CCB_NO_TMA, hub rows -- with plain loads), the un-paired plan, rows split into parts and the
    forward stream with two segments per pair (CCB_NO_MERGE) or with the first member's arc in a tail slot (CCB_NO_OWN) give
    the same answers.  The default on these graphs is own-row terms (blank arcs / self loops as coefficients on plainly
    loaded rows) and one merged segment per pair, which the other variants therefore run through the register-gather and
    arcs-in-global walkers."""
    from oracle import oracle
    from cat_b200 import _C
    for e in env.split("+"):
        if e == "HUBS":     # long in-arc rows computed in atomically accumulated parts
            monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
            monkeypatch.setenv("CCB_PART_ARCS", "7")
        else:
            monkeypatch.setenv(*(e.split("=") if "=" in e else (e, "1")))
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    T = 30
    # 20: one utterance per lane (second weights prefetched with the gathers); 12 / 5: the small-batch kernels (16-float
    # rows), whose backward pass then streams the second weights with bulk copies next to the TMA row gathers
    # ARCS_IN_GLOBAL: 1 and 2 utterances per lane of the streamed-arc backward kernels (two lane groups at 130), 1, 2 and 4 of
    # the forward kernels reading their arcs from L2 (tests/test_den_launch.py pins these tiers)
    for N in ((40, 20, 12, 5) if "W1" in env else (40, 12, 130) if "ARCS" in env else (40, 64) if "RING" in env else (40, 12, 64) if ("MERGE" in env or "OWN" in env) else (40,)):
        lens = np.maximum(1, T - (np.arange(N) * 5) % T).astype(np.int32)
        y, _, lens, _ = oracle.synth_batch(N, T, V, seed=8, lens=lens)
        logits = torch.tensor(y, device="cuda")
        grad = torch.zeros_like(logits)
        ca = torch.zeros(N, device="cuda"); cb = torch.zeros(N, device="cuda")
        _C.gpu_den(logits, grad, torch.tensor(lens, dtype=torch.int32).cuda(), ca, cb)
        la, lb, gd = oracle.den(g, y, lens)
        np.testing.assert_allclose(ca.cpu().numpy(), la, rtol=LOSS_RTOL, atol=1e-4)
        np.testing.assert_allclose(cb.cpu().numpy(), lb, rtol=LOSS_RTOL, atol=1e-4)
        assert np.abs(grad.cpu().numpy() - gd).max() < GRAD_ATOL
    del ctx


def test_fused_vs_oracle_and_bf16(tmp_graphs):
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 8, 60
    lens = [60, 60, 55, 41, 33, 20, 9, 3]
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=21, lens=lens)
    for sa in (True, False):
        loss, grad = _run_ours(y, labels, lens, ly, 0.1, size_average=sa)
        oloss, ograd, _ = oracle.ctc_crf(g, y, labels, lens, ly, 0.1, size_average=sa)
        _close_loss(loss, oloss)
        assert np.abs(grad - ograd).max() < GRAD_ATOL * (1 if sa else N)
    # bf16 logits: parity is defined against the oracle fed the bf16-rounded values (SURVEY.md 7 item 8)
    yb = torch.tensor(y).bfloat16()
    loss, grad = _run_ours(yb.float().numpy(), labels, lens, ly, 0.1, dtype=torch.bfloat16)
    oloss, ograd, _ = oracle.ctc_crf(g, yb.float().numpy(), labels, lens, ly, 0.1)
    _close_loss(loss, oloss)
    assert np.abs(grad - ograd).max() < GRAD_ATOL
    del ctx


def test_composed_den_graph_is_lm_weighted_ctc_sum(tmp_path):
    """SURVEY 8f-2 on the GPU: a den graph composed natively (fst.compose_ctc_lm, no Kaldi/OpenFst) loaded through
    CRFContext; logZ_den must equal log sum_l p_LM(l) p_CTC(l|x), both factors from this library's own kernels
    (den via _C.gpu_den, every p_CTC via _C.gpu_ctc), enumerated over all label sequences."""
    import itertools
    import ctc_crf
    from cat_b200 import fst
    V, T = 4, 5
    lm = fst.make_random_lm(H=3, V=V, d=2, seed=11)
    path = str(tmp_path / "tlm_native.fst")
    fst.write_fst(path, fst.compose_ctc_lm(lm))
    ctx = _ctx(path)
    y = torch.log_softmax(torch.randn(1, T, V, generator=torch.Generator().manual_seed(3)), -1).cuda()
    grad = torch.zeros_like(y)
    ca, cb = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    ctc_crf._C.gpu_den(y, grad, torch.tensor([T], dtype=torch.int32, device="cuda"), ca, cb)
    seqs = [l for L in range(T + 1) for l in itertools.product(range(1, V), repeat=L) if np.isfinite(fst.lm_logprob(lm, l))]
    seqs = [l for l in seqs if len(l) + sum(a == b for a, b in zip(l, l[1:])) <= T]      # CTC-feasible in T frames
    act = y.transpose(0, 1).repeat(1, len(seqs), 1).contiguous()                           # (T, n_seqs, V)
    costs = torch.zeros(len(seqs))
    labels = torch.tensor([p for l in seqs for p in l], dtype=torch.int32)
    ctc_crf._C.gpu_ctc(act, torch.zeros_like(act), labels, torch.tensor([len(l) for l in seqs], dtype=torch.int32),
                       torch.full((len(seqs),), T, dtype=torch.int32), len(seqs), costs, 0)
    torch.cuda.synchronize()
    total = np.logaddexp.reduce([fst.lm_logprob(lm, l) + float(c) for l, c in zip(seqs, costs)])
    assert len(seqs) > 5
    assert abs(float(ca.item()) - total) < 1e-4 * max(1.0, abs(total))
    assert abs(float(cb.item()) - total) < 1e-4 * max(1.0, abs(total))
    del ctx


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_raw_logit_entry(tmp_graphs, dtype):
    """SURVEY 8f-1: CTC_CRF_LOSS(from_logits=True) on raw encoder outputs == log_softmax + loss + autograd chain, against
    the oracle and against our own two-step path (torch log_softmax -> CTC_CRF_LOSS) on the same inputs."""
    import ctc_crf
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 8, 60
    lens = [60, 60, 55, 41, 33, 20, 9, 3]
    _, labels, lens, ly = oracle.synth_batch(N, T, V, seed=23, lens=lens)
    rng = np.random.default_rng(5)
    z = (4.0 * rng.standard_normal((N, T, V)) + 7.0).astype(np.float32)      # unnormalised, offset on purpose
    zt = torch.tensor(z, device="cuda").to(dtype)
    z_used = zt.float().cpu().numpy()                                           # the values the kernel actually sees
    lab_t, lx_t, ly_t = (torch.tensor(a, dtype=torch.int32) for a in (labels, lens, ly))
    for sa in (True, False):
        oloss, odz, oparts = oracle.ctc_crf_from_logits(g, z_used, labels, lens, ly, 0.1, size_average=sa)
        zin = zt.clone().requires_grad_(True)
        loss = ctc_crf.CTC_CRF_LOSS(lamb=0.1, size_average=sa, from_logits=True)(zin, lab_t, lx_t, ly_t)
        loss.backward()
        assert zin.grad.dtype == dtype
        _close_loss(float(loss.item()), oloss)
        tol = GRAD_ATOL * (1 if sa else N) * (4 if dtype == torch.bfloat16 else 1)   # bf16: the returned grad is rounded
        assert np.abs(zin.grad.float().cpu().numpy() - odz).max() < tol
        # rows past each length stay zero; every valid row of d loss/d z sums to ~0 (softmax Jacobian)
        gz = zin.grad.float().cpu().numpy()
        for n in range(N):
            assert np.all(gz[n, lens[n]:] == 0)
        assert np.abs(gz.sum(-1)).max() < (2e-2 if dtype == torch.bfloat16 else 1e-4) * (1 if sa else N)
        # two-step path through torch autograd (what cat/ctc/train.py does)
        z2 = zt.clone().requires_grad_(True)
        loss2 = ctc_crf.CTC_CRF_LOSS(lamb=0.1, size_average=sa)(z2.float().log_softmax(-1), lab_t, lx_t, ly_t)
        loss2.backward()
        _close_loss(float(loss.item()), float(loss2.item()))
        assert np.abs(gz - z2.grad.float().cpu().numpy()).max() < tol
    # parts are reported normalised
    _, _, parts = ctc_crf._C.ctc_crf_loss_fwd(zt.contiguous(), lab_t, lx_t, ly_t, 0.1, True, want_parts=True, from_logits=True)
    parts = parts.cpu().numpy()
    np.testing.assert_allclose(parts[:N], oparts["logz_alpha"], rtol=1e-4, atol=1e-3)
    np.testing.assert_allclose(parts[N:], oparts["logp_ctc"], rtol=1e-4, atol=1e-3)
    del ctx


@pytest.mark.parametrize("N,T,lens,ly", [
    (1, 1, [1], [0]),                       # single frame, empty label sequence
    (1, 1, [1], [1]),                       # single frame, single label
    (2, 6, [6, 0], [2, 0]),                 # an utterance of length zero rides along
    (3, 9, [9, 9, 9], [9, 4, 0]),           # L == T (no blank can be emitted), and L = 0
    (33, 5, None, None),                    # more utterances than one lane group, tiny T
    (130, 7, None, None),                   # 256 lanes: forward walks 4 utterances per lane, backward 2 (4 lane groups)
])
def test_edge_shapes_vs_oracle(tmp_graphs, N, T, lens, ly):
    """Degenerate shapes through the fused op against the oracle (empty labels, T=1, len=0, L=T, ragged lanes)."""
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_small"]
    ctx = _ctx(path)
    rng = np.random.default_rng(17)
    if lens is None:
        lens = rng.integers(1, T + 1, size=N)
        ly = np.minimum(lens // 2, 2)
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=41, lens=lens)
    ly = np.asarray(ly, np.int32)
    labels = rng.integers(1, V, size=int(ly.sum())).astype(np.int32)
    for i in range(1, len(labels)):          # no repeats, so that L == T stays feasible
        if labels[i] == labels[i - 1]:
            labels[i] = labels[i] % (V - 1) + 1
    loss, grad = _run_ours(y, labels, lens, ly, 0.1)
    oloss, ograd, parts = oracle.ctc_crf(g, y, labels, lens, ly, 0.1)
    if np.isfinite(oloss):
        _close_loss(loss, oloss)
        assert np.abs(grad - ograd).max() < GRAD_ATOL
    else:                                     # an infeasible utterance: +inf loss on both sides
        assert not np.isfinite(loss)
    del ctx


def test_sliced_batches_and_padded_frames(tmp_graphs, monkeypatch):
    """Batches are processed in memory-bounded slices that walk only max(len) frames: same loss/grad as one call,
    and frames beyond every length (T padded past max len) cost nothing and stay zero."""
    from oracle import oracle
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 11, 50
    lens = np.array([37, 37, 30, 28, 25, 19, 12, 9, 7, 3, 1], np.int32)      # T=50 > max len
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=31, lens=lens)
    ref_loss, ref_grad = _run_ours(y, labels, lens, ly, 0.05)
    monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 4)                            # 3 slices
    loss, grad = _run_ours(y, labels, lens, ly, 0.05)
    _close_loss(loss, ref_loss, 1e-6)
    assert np.abs(grad - ref_grad).max() < 1e-6
    oloss, ograd, _ = oracle.ctc_crf(g, y, labels, lens, ly, 0.05)
    _close_loss(loss, oloss)
    assert np.abs(grad - ograd).max() < GRAD_ATOL
    for n in range(N):
        assert not grad[n, lens[n]:].any()
    # memory-bounded slicing: 40 utterances need 64 lanes of scratch; with room for 32 lanes only they go in two halves
    from cat_b200 import _lib
    monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 512)
    N2, T2 = 40, 20
    y2, labels2, lens2, ly2 = oracle.synth_batch(N2, T2, V, seed=32)
    ref_loss, ref_grad = _run_ours(y2, labels2, lens2, ly2, 0.05)
    L = _lib.lib()
    need32 = (int(L.ccb_den_alpha_floats(32, T2)) * 4 + int(L.ccb_den_aux_bytes(32, T2))
              + int(L.ccb_ctc_workspace_bytes(32, T2, int(ly2.max()))))
    calls = []
    monkeypatch.setattr(_C, "_scratch_budget", lambda dev, need=0: (calls.append(need), need32 + 4096)[1])
    loss, grad = _run_ours(y2, labels2, lens2, ly2, 0.05)
    assert calls, "the budget hook was not consulted"
    _close_loss(loss, ref_loss, 1e-6)
    assert np.abs(grad - ref_grad).max() < 1e-6
    del ctx


def test_vs_reference_cuda_golden():
    """The CUDA path against the reference's own CUDA outputs recorded in tests/golden/ref_cuda_golden.npz
    (tests/golden/make_ref_golden.py): needs nothing outside the repository."""
    from conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "ref_cuda_golden.npz"), allow_pickle=False)
    for c in sorted({k.split("/")[0] for k in z.files}):
        ctx = _ctx(os.path.join(GOLDEN, str(z[f"{c}/graph"])))
        loss, grad = _run_ours(z[f"{c}/y"], z[f"{c}/labels"], z[f"{c}/lx"], z[f"{c}/ly"], float(z[f"{c}/lamb"]))
        _close_loss(loss, float(z[f"{c}/ref_loss"]))
        assert np.abs(grad - z[f"{c}/ref_grad"]).max() < GRAD_ATOL, c
        del ctx


def test_vs_reference_cuda(tmp_path):
    """Side by side with the reference's own CUDA code (oracle/_ref) on the AISHELL-shaped config scaled to
    what the fp64 oracle also finishes in seconds: V=218, 100k-arc T-compose-LM graph, N=8, T=120."""
    from oracle import oracle, ref_cuda
    from cat_b200 import fst
    if not ref_cuda.available():
        pytest.skip("oracle/_ref not built")
    V = 218
    g = fst.make_synthetic_den(2000, 24, V, seed=7)
    path = str(tmp_path / "den.fst")
    fst.write_fst(path, g)
    N, T = 8, 120
    lens = [120, 120, 111, 97, 80, 64, 30, 12]
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=1234, lens=lens)
    ctx = _ctx(path)
    loss, grad = _run_ours(y, labels, lens, ly, 0.01)
    rctx = ref_cuda.RefContext(path, 0)
    rl, rg, parts = ref_cuda.ctc_crf_forward(rctx, torch.tensor(y, device="cuda"), torch.tensor(labels),
                                             torch.tensor(lens), torch.tensor(ly), 0.01, True)
    torch.cuda.synchronize()
    rctx.close()
    _close_loss(loss, float(rl.item()))
    assert np.abs(grad - rg.cpu().numpy()).max() < GRAD_ATOL
    oloss, ograd, _ = oracle.ctc_crf(g, y, labels, lens, ly, 0.01)
    _close_loss(float(rl.item()), oloss)          # pins the oracle to the reference's actual output
    assert np.abs(rg.cpu().numpy() - ograd).max() < GRAD_ATOL
    del ctx


def test_full_size_properties(tmp_path):
    """BASELINE config 2 (N=32, T=800, V=218, ~1M-arc graph) against the reference CUDA build, plus the
    size-independent invariants: occupancy rows sum to 1 (den) / gradient rows sum to -lamb/N, logZ(alpha)
    == logZ(beta), idempotence (same result twice)."""
    from oracle import oracle, ref_cuda
    from cat_b200 import fst, _C
    V = 218
    g = fst.make_synthetic_den(20000, 24, V, seed=7)
    path = str(tmp_path / "den1m.fst")
    fst.write_fst(path, g)
    N, T = 32, 800
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=1234)
    ctx = _ctx(path)
    logits = torch.tensor(y, device="cuda")
    gden = torch.zeros_like(logits)
    ca = torch.zeros(N, device="cuda"); cb = torch.zeros(N, device="cuda")
    _C.gpu_den(logits, gden, torch.tensor(lens).cuda(), ca, cb)
    rows = gden.sum(-1).cpu().numpy()
    assert np.abs(rows - 1.0).max() < 1e-4
    np.testing.assert_allclose(ca.cpu().numpy(), cb.cpu().numpy(), rtol=1e-5)
    lamb = 0.01
    loss, grad = _run_ours(y, labels, lens, ly, lamb)
    loss2, grad2 = _run_ours(y, labels, lens, ly, lamb)
    _close_loss(loss, loss2, 1e-6)
    assert np.abs(grad - grad2).max() < 1e-5
    # sum_k (gamma_den - (1+lamb) gamma_ctc) = -lamb; the numerator is fp32 log-domain over 800 frames (measured 8e-4)
    assert np.abs(grad.sum(-1) * N + lamb).max() < 2e-3
    # the fp64 oracle on two of the utterances (it needs ~1 min per utterance at this size)
    sub = [0, N - 1]
    off = np.concatenate([[0], np.cumsum(ly)])
    sub_labels = np.concatenate([labels[off[i]:off[i + 1]] for i in sub])
    oloss, ograd, oparts = oracle.ctc_crf(g, y[sub], sub_labels, lens[sub], ly[sub], lamb, size_average=False, nthreads=2)
    d_or = np.abs(grad[sub] * N - ograd).max()
    print("max |grad - oracle| (unscaled occupancies, N=32 T=800 A=1M):", d_or)
    assert d_or < GRAD_ATOL
    np.testing.assert_allclose(ca.cpu().numpy()[sub], oparts["logz_alpha"], rtol=LOSS_RTOL)
    if ref_cuda.available():
        rctx = ref_cuda.RefContext(path, 0)
        rl, rg, parts = ref_cuda.ctc_crf_forward(rctx, logits, torch.tensor(labels), torch.tensor(lens),
                                                 torch.tensor(ly), lamb, True)
        torch.cuda.synchronize()
        rctx.close()
        _close_loss(loss, float(rl.item()))
        rgn = rg.cpu().numpy()
        d = np.abs(grad - rgn).max() * N
        ref_self = np.abs(rgn.sum(-1) * N + lamb).max()          # the reference's own row-sum inconsistency
        d_ref_or = np.abs(rgn[sub] * N - ograd).max()
        print("max |grad - reference CUDA| (unscaled):", d, "| reference row-sum error:", ref_self,
              "| max |reference - oracle|:", d_ref_or)
        # at T=800 the reference's fp32 log domain (|alpha| ~ 2500) is itself several 1e-2 off the fp64 oracle; the
        # tight comparison against the reference is test_vs_reference_cuda (T=120).  Here: no worse than the reference.
        assert d_or <= d_ref_or + GRAD_ATOL
        assert d < 0.1
    del ctx


def test_error_paths(fixture_fst, tmp_path):
    import ctc_crf
    with pytest.raises(RuntimeError):
        ctc_crf.CRFContext(str(tmp_path / "missing.fst"), gpus=0)
    bad = tmp_path / "bad.fst"
    bad.write_bytes(b"not an fst at all")
    with pytest.raises(RuntimeError):
        ctc_crf.CRFContext(str(bad), gpus=0)
    with pytest.raises(RuntimeError):
        ctc_crf.CRFContext(fixture_fst, gpus=99)
    ctx = ctc_crf.CRFContext(fixture_fst, gpus=0)
    crit = ctc_crf.CTC_CRF_LOSS()
    with pytest.raises(RuntimeError):   # V smaller than the den graph's label set
        crit(torch.zeros(1, 4, 3, device="cuda").log_softmax(-1), torch.tensor([1], dtype=torch.int32),
             torch.tensor([4], dtype=torch.int32), torch.tensor([1], dtype=torch.int32))
    del ctx


def _viterbi_ref(y, lab, blank=0):
    """Textbook best path over the blank-expanded CTC lattice (float64, python loops): token per frame, path score."""
    T = y.shape[0]
    ext = [blank]
    for k in lab:
        ext += [int(k), blank]
    S = len(ext)
    v = np.full((T, S), -np.inf)
    bp = np.zeros((T, S), np.int64)
    v[0, 0] = y[0, blank]
    if S > 1:
        v[0, 1] = y[0, ext[1]]
    for t in range(1, T):
        for s in range(S):
            best, k = v[t - 1, s], 0
            if s >= 1 and v[t - 1, s - 1] > best:
                best, k = v[t - 1, s - 1], 1
            if s >= 2 and ext[s] != blank and ext[s] != ext[s - 2] and v[t - 1, s - 2] > best:
                best, k = v[t - 1, s - 2], 2
            v[t, s] = best + y[t, ext[s]]
            bp[t, s] = k
    s = S - 1
    if S > 1 and v[T - 1, S - 2] > v[T - 1, S - 1]:
        s = S - 2
    score = v[T - 1, s]
    out = np.zeros(T, np.int64)
    for t in range(T - 1, -1, -1):
        out[t] = ext[s]
        s -= bp[t, s]
    return out, score


def test_ctc_align_best_path():
    """SURVEY 8f-4 by-product: ctc_crf.ctc_align == textbook Viterbi over the numerator lattice (tokens per frame and the
    path score), collapses back to the label sequence, and marks padding / infeasible utterances with -1."""
    import ctc_crf
    from oracle import oracle
    N, T, V = 5, 40, 9
    lens = [40, 33, 12, 7, 3]
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=19, lens=lens)
    ly = np.array([9, 6, 0, 3, 5], np.int32)                      # L=0; the last one is infeasible (5 labels in 3 frames)
    rng = np.random.default_rng(2)
    labels = rng.integers(1, V, size=int(ly.sum())).astype(np.int32)
    labels[1] = labels[0]                                          # a repeat: needs a blank in between
    align, score = ctc_crf.ctc_align(torch.tensor(y, device="cuda"), torch.tensor(labels), torch.tensor(lens), torch.tensor(ly))
    align, score = align.cpu().numpy(), score.cpu().numpy()
    off = np.concatenate([[0], np.cumsum(ly)])
    for n in range(N):
        lab = labels[off[n]:off[n + 1]]
        if n == N - 1:
            assert np.isinf(score[n]) and score[n] < 0 and (align[n] == -1).all()
            continue
        ref, sc = _viterbi_ref(y[n, :lens[n]].astype(np.float64), lab)
        assert (align[n, lens[n]:] == -1).all()
        assert abs(score[n] - sc) < 1e-4 * max(1.0, abs(sc))
        got = align[n, :lens[n]]
        if not np.array_equal(got, ref):                           # ties may be broken differently in fp32: same score then
            assert abs(float(sum(y[n, t, got[t]] for t in range(lens[n]))) - sc) < 1e-3
        collapsed = [int(k) for i, k in enumerate(got) if k != 0 and (i == 0 or got[i - 1] != k)]
        assert collapsed == [int(k) for k in lab]


def test_warp_ctc_loss_native_path_matches_gpu_ctc():
    """WARP_CTC_LOSS (one native call on (N,T,V), no transpose / zero fill / host costs) against the reference-signature
    route through _C.gpu_ctc on the transposed copy, and against the oracle; infeasible utterance -> +inf loss."""
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C
    N, T, V = 6, 50, 20
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=29, lens=[50, 50, 44, 31, 18, 6])
    yt = torch.tensor(y, device="cuda")
    for sa in (True, False):
        logits = yt.clone().requires_grad_(True)
        loss = ctc_crf.WARP_CTC_LOSS(size_average=sa)(logits, torch.tensor(labels), torch.tensor(lens), torch.tensor(ly))
        loss.backward()
        act = yt.transpose(0, 1).contiguous()
        grads = torch.zeros_like(act)
        costs = torch.zeros(N)
        _C.gpu_ctc(act, grads, torch.tensor(labels), torch.tensor(ly), torch.tensor(lens), N, costs, 0)
        sc = 1.0 / N if sa else 1.0
        assert abs(float(loss.item()) + float(costs.sum()) * sc) <= 1e-5 * max(1.0, abs(float(costs.sum())))
        assert float((logits.grad + grads.transpose(0, 1) * sc).abs().max()) < 1e-6
        lp, gc = oracle.ctc(y, labels, ly, lens)
        _close_loss(float(loss.item()), -lp.sum() * sc)
        assert np.abs(logits.grad.cpu().numpy() + gc * sc).max() < GRAD_ATOL
        for n in range(N):
            assert not bool(logits.grad[n, lens[n]:].any())
    ly_bad = ly.copy(); ly_bad[-1] = 7                               # 7 labels in 6 frames
    labels_bad = np.concatenate([labels, np.ones(int(ly_bad.sum() - ly.sum()), np.int32)])
    loss = ctc_crf.WARP_CTC_LOSS()(yt, torch.tensor(labels_bad), torch.tensor(lens), torch.tensor(ly_bad))
    assert np.isinf(float(loss.item())) and float(loss.item()) > 0
