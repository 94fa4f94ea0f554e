"""Several label sequences per utterance (`utt=`) on the GPU: CTC_CRF_LOSS, WARP_CTC_LOSS and ctc_align.

Costs against the fp64 oracle per sequence (1e-4 relative), gradients against the oracle's per-sequence gradients summed onto
their logits rows (1e-3 absolute, plus the rounding of a 16-bit result); log p bit for bit and logZ to fp32 rounding against
the calls callers make today on logits[utt]; WARP_CTC_LOSS against torch's fp64 ctc_loss; the den work independent of the
number of sequences.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32)


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _close(a, b, rtol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.all(np.abs(a - b) <= rtol * np.maximum(1.0, np.abs(b))), (a, b)


def _seqs(counts, lens, V, seed, shuffle=True):
    """counts[n] label sequences for utterance n, each feasible for lens[n] frames, in a shuffled order.
    Returns (utt, labels, ly)."""
    rng = np.random.default_rng(seed)
    utt = np.repeat(np.arange(len(counts)), counts).astype(np.int32)
    if shuffle:
        utt = utt[rng.permutation(len(utt))]
    ly = np.array([rng.integers(0, max(1, lens[n] // 4) + 1) for n in utt], np.int32)
    labels = rng.integers(1, V, size=int(ly.sum())).astype(np.int32)
    return utt, labels, ly


def _batch(N, T, V, seed, lens, dtype, from_logits):
    from oracle import oracle
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=seed, lens=lens)
    if from_logits:
        y = y + 3.0 * np.random.default_rng(seed).standard_normal((N, T, 1)).astype(np.float32) + 5.0
    yt = torch.tensor(y, device="cuda").to(dtype).contiguous()
    return yt, yt.float().cpu().numpy(), lens


def _oracle(g, y_used, labels, lens, ly, utt, lamb, from_logits):
    """Per-sequence costs and unscaled gradients of the fp64 oracle, each sequence on its own copy of its row."""
    from oracle import oracle
    f = oracle.ctc_crf_from_logits if from_logits else oracle.ctc_crf
    _, grad, parts = f(g, y_used[utt], labels, lens[utt], ly, lamb, size_average=False)
    return parts["logz_alpha"] - (1.0 + lamb) * parts["logp_ctc"], grad


def _rows(per_seq_grad, utt, w, N):
    out = np.zeros((N,) + per_seq_grad.shape[1:], np.float64)
    np.add.at(out, utt, np.asarray(w, np.float64)[:, None, None] * per_seq_grad)
    return out


def _run(crit, yt, labels, lens, ly, utt, w):
    y = yt.clone().requires_grad_(True)
    out = crit(y, _i32(labels), _i32(lens), _i32(ly), utt=_i32(utt))
    (g,) = torch.autograd.grad(out.mul(w).sum(), y)
    return out.detach(), g


def _grad_ok(grad, ref, dtype):
    tol = GRAD_ATOL + 0.5 * torch.finfo(dtype).eps * np.abs(ref)
    err = np.abs(grad.float().cpu().numpy() - ref)
    assert np.all(err <= tol), err.max()


def _check_vs_oracle(g, yt, y_used, labels, lens, ly, utt, lamb, from_logits, seed=0):
    import ctc_crf
    N, M = yt.shape[0], len(utt)
    ocost, ograd = _oracle(g, y_used, labels, lens, ly, utt, lamb, from_logits)
    # reduction 'none' with a random grad_output
    w = np.random.default_rng(seed).uniform(-2.0, 2.0, M).astype(np.float32)
    crit = ctc_crf.CTC_CRF_LOSS(lamb=lamb, from_logits=from_logits, reduction="none")
    costs, grad = _run(crit, yt, labels, lens, ly, utt, torch.tensor(w, device="cuda"))
    assert costs.shape == (M,) and grad.dtype == yt.dtype
    _close(costs.cpu().numpy(), ocost, LOSS_RTOL)
    _grad_ok(grad, _rows(ograd, utt, w, N), yt.dtype)
    # the scalar (mean over the M sequences) and its gradient
    mean = ctc_crf.CTC_CRF_LOSS(lamb=lamb, from_logits=from_logits)
    loss, gm = _run(mean, yt, labels, lens, ly, utt, torch.ones(1, device="cuda"))
    _close(float(loss.item()), float(ocost.sum()) / M, LOSS_RTOL)
    _grad_ok(gm, _rows(ograd, utt, np.full(M, 1.0 / M), N), yt.dtype)
    # forward only: the same costs
    with torch.no_grad():
        ev = crit(yt, _i32(labels), _i32(lens), _i32(ly), utt=_i32(utt))
    _close(ev.cpu().numpy(), costs.cpu().numpy(), 1e-6)
    for n in range(N):
        assert not grad[n, int(lens[n]):].any()
        if n not in set(utt.tolist()):      # an utterance without a sequence: exactly zero
            assert not grad[n].any() and not gm[n].any()
    return costs


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("from_logits", [False, True])
def test_costs_and_grad_vs_oracle(tmp_graphs, dtype, from_logits):
    """0 to 5 sequences per utterance, in a shuffled order."""
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 8, 32
    yt, y_used, lens = _batch(N, T, V, 21, np.linspace(T, 6, N).astype(np.int32), DTYPES[dtype], from_logits)
    utt, labels, ly = _seqs([3, 0, 5, 1, 2, 4, 0, 1], lens, V, seed=5)
    _check_vs_oracle(g, yt, y_used, labels, lens, ly, utt, 0.1, from_logits)
    del ctx


@pytest.mark.parametrize("path_kind", ["slices", "ckpt"])
def test_sliced_and_checkpointed(tmp_graphs, monkeypatch, path_kind):
    """N > 64 (two native calls, the second with utterances lacking sequences) and slices forced to checkpointed alpha."""
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    if path_kind == "slices":
        N, T = 70, 16
        counts = [(n * 7) % 4 for n in range(N)]
    else:
        monkeypatch.setattr(_C, "_ckpt_k_override", 3)
        monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 4)
        N, T = 10, 30
        counts = [2, 1, 0, 3, 1, 2, 0, 0, 4, 1]
    lens = np.maximum(1, T - (np.arange(N) * 5) % T).astype(np.int32)
    for from_logits in (False, True):
        yt, y_used, lens = _batch(N, T, V, 9 + N, lens, torch.float32, from_logits)
        utt, labels, ly = _seqs(counts, lens, V, seed=N)
        _check_vs_oracle(g, yt, y_used, labels, lens, ly, utt, 0.1, from_logits, seed=N)
    del ctx


@pytest.mark.parametrize("tier", ["small_batch", "hub_parts", "arcs_in_global", "no_tma"])
def test_den_tiers(tmp_graphs, monkeypatch, tier):
    """The den launches of the test graphs' Init-time hooks, with several sequences per utterance."""
    env = {"hub_parts": {"CCB_HUB_IN_ARCS": "10", "CCB_PART_ARCS": "7"}, "arcs_in_global": {"CCB_ARCS_IN_GLOBAL": "1"},
           "no_tma": {"CCB_NO_TMA": "1"}}.get(tier, {})
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = (12, 24) if tier == "small_batch" else (40, 20)
    yt, y_used, lens = _batch(N, T, V, 31, np.maximum(2, T - np.arange(N) % T).astype(np.int32), torch.float32, False)
    utt, labels, ly = _seqs([1 + n % 3 for n in range(N)], lens, V, seed=2)
    _check_vs_oracle(g, yt, y_used, labels, lens, ly, utt, 0.1, False)
    del ctx


def test_equivalence_with_repeated_rows(tmp_graphs):
    """Against what callers do today, one call on logits[utt]: the CTC-CRF costs to fp32 rounding (logZ is summed with
    atomics), duplicate sequences at the same bits, WARP_CTC_LOSS bit for bit, ctc_align identical."""
    import ctc_crf
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 6, 30
    for from_logits in (False, True):
        yt, _, lens = _batch(N, T, V, 41, np.array([30, 27, 20, 30, 12, 25], np.int32), torch.float32, from_logits)
        utt, labels, ly = _seqs([2, 3, 1, 0, 2, 4], lens, V, seed=8)
        # a duplicate of sequence 0, on the same row
        off = np.concatenate([[0], np.cumsum(ly)])
        utt = np.append(utt, utt[0]).astype(np.int32)
        labels = np.concatenate([labels, labels[off[0]:off[1]]]).astype(np.int32)
        ly = np.append(ly, ly[0]).astype(np.int32)
        rep = yt[torch.tensor(utt, dtype=torch.long, device="cuda")].contiguous()
        crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits, reduction="none")
        c_seq = crit(yt.clone().requires_grad_(True), _i32(labels), _i32(lens), _i32(ly), utt=_i32(utt)).detach()
        c_rep = crit(rep.clone().requires_grad_(True), _i32(labels), _i32(lens[utt]), _i32(ly)).detach()
        c_seq, c_rep = c_seq.cpu().numpy(), c_rep.cpu().numpy()
        assert c_seq[0] == c_seq[-1]
        _close(c_seq, c_rep, 1e-6)
    yt, y_used, lens = _batch(N, T, V, 43, np.array([30, 27, 20, 30, 12, 25], np.int32), torch.float32, False)
    utt, labels, ly = _seqs([2, 3, 1, 0, 2, 4], lens, V, seed=9)
    rep = yt[torch.tensor(utt, dtype=torch.long, device="cuda")].contiguous()
    warp = ctc_crf.WARP_CTC_LOSS(reduction="none")
    a = warp(yt.clone().requires_grad_(True), _i32(labels), _i32(lens), _i32(ly), utt=_i32(utt))
    b = warp(rep.clone().requires_grad_(True), _i32(labels), _i32(lens[utt]), _i32(ly))
    assert torch.equal(a.detach(), b.detach())          # log p bit for bit
    al, sc = ctc_crf.ctc_align(yt, _i32(labels), _i32(lens), _i32(ly), utt=_i32(utt))
    al2, sc2 = ctc_crf.ctc_align(rep, _i32(labels), _i32(lens[utt]), _i32(ly))
    assert torch.equal(al, al2) and torch.equal(sc, sc2)
    del ctx


def test_crf_logp_bit_identical(tmp_graphs):
    """The numerator's log p of every sequence is the single-sequence call's, bit for bit (read through the CTC-only loss,
    which runs the same kernel instance on the same rows), and the CTC-CRF costs carry it: cost[m] + (1+lamb) log p[m]
    is the row's logZ, the same for every sequence of a row to fp32 rounding."""
    import ctc_crf
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 5, 28
    yt, _, lens = _batch(N, T, V, 51, np.array([28, 20, 25, 9, 28], np.int32), torch.float32, False)
    utt, labels, ly = _seqs([3, 2, 4, 1, 3], lens, V, seed=4)
    with torch.no_grad():
        logp = -ctc_crf.WARP_CTC_LOSS(reduction="none")(yt, _i32(labels), _i32(lens), _i32(ly), utt=_i32(utt)).cpu().numpy()
        single = np.array([-float(ctc_crf.WARP_CTC_LOSS(reduction="none")(
            yt[int(u):int(u) + 1].contiguous(), _i32(labels[o:o + l]), _i32(lens[u:u + 1]), _i32([l]))[0])
            for u, o, l in zip(utt, np.concatenate([[0], np.cumsum(ly)])[:-1], ly)], np.float32)
        assert np.array_equal(logp, single)
        costs = ctc_crf.CTC_CRF_LOSS(lamb=0.1, reduction="none")(yt, _i32(labels), _i32(lens), _i32(ly),
                                                                 utt=_i32(utt)).cpu().numpy()
    logz = costs.astype(np.float64) + 1.1 * logp.astype(np.float64)
    for n in range(N):
        _close(logz[utt == n], np.full((utt == n).sum(), logz[utt == n][0]), 1e-6)
    del ctx


def _torch_ctc(y, labels, lens, ly, w):
    lp = torch.tensor(y, dtype=torch.float64).transpose(0, 1).contiguous().requires_grad_(True)
    costs = torch.nn.functional.ctc_loss(lp, torch.tensor(labels, dtype=torch.long), torch.tensor(lens, dtype=torch.long),
                                         torch.tensor(ly, dtype=torch.long), blank=0, reduction="none")
    (g,) = torch.autograd.grad((costs * torch.tensor(w, dtype=torch.float64)).sum(), lp)
    g = g.transpose(0, 1).numpy().copy()
    for m in range(len(lens)):      # torch's gradient assumes log-softmax inputs (see test_gpu_per_utt._torch_ctc)
        g[m, :lens[m]] -= np.exp(y[m, :lens[m]].astype(np.float64)) * w[m]
    return costs.detach().numpy(), g


@pytest.mark.parametrize("dtype", sorted(DTYPES))
def test_warp_ctc_vs_torch(dtype):
    import ctc_crf
    from oracle import oracle
    N, T, V = 6, 40, 15
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=17, lens=np.array([40, 33, 25, 18, 40, 10], np.int32))
    yt = torch.tensor(y, device="cuda").to(DTYPES[dtype])
    y_used = yt.float().cpu().numpy()
    utt, labels, ly = _seqs([2, 0, 3, 1, 4, 2], lens, V, seed=3)
    M = len(utt)
    w = np.random.default_rng(1).uniform(-2.0, 2.0, M).astype(np.float32)
    costs, grad = _run(ctc_crf.WARP_CTC_LOSS(reduction="none"), yt, labels, lens, ly, utt, torch.tensor(w, device="cuda"))
    tc, tg = _torch_ctc(y_used[utt], labels, lens[utt], ly, w)
    _close(costs.cpu().numpy(), tc, LOSS_RTOL)
    _grad_ok(grad, _rows(tg, utt, np.ones(M), N), DTYPES[dtype])
    loss, gm = _run(ctc_crf.WARP_CTC_LOSS(), yt, labels, lens, ly, utt, torch.ones(1, device="cuda"))
    _close(float(loss.item()), float(tc.sum()) / M, LOSS_RTOL)
    _, tg1 = _torch_ctc(y_used[utt], labels, lens[utt], ly, np.full(M, 1.0 / M))
    _grad_ok(gm, _rows(tg1, utt, np.ones(M), N), DTYPES[dtype])
    with torch.no_grad():
        ev = ctc_crf.WARP_CTC_LOSS(reduction="none")(yt, _i32(labels), _i32(lens), _i32(ly), utt=_i32(utt))
    assert torch.equal(ev, costs)


@pytest.mark.parametrize("from_logits", [False, True])
def test_zero_infinity_per_sequence(tmp_graphs, from_logits):
    """Infeasible sequences (more labels than frames) and a length-0 utterance: without zero_infinity their costs are inf /
    NaN; with it they cost 0 and drop out of the gradient, and everything else is what the batch without them gives."""
    import ctc_crf
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 5, 24
    yt, _, lens = _batch(N, T, V, 61, np.array([24, 6, 0, 20, 15], np.int32), torch.float32, from_logits)
    utt, labels, ly = _seqs([2, 2, 1, 3, 1], np.maximum(lens, 1), V, seed=7, shuffle=False)
    # sequence 2 (utterance 1, 6 frames) made infeasible: 9 labels
    off = np.concatenate([[0], np.cumsum(ly)])
    labels = np.concatenate([labels[:off[2]], np.arange(1, 10) % (V - 1) + 1, labels[off[3]:]]).astype(np.int32)
    ly[2] = 9
    bad = [2, int(np.flatnonzero(utt == 2)[0])]        # the infeasible sequence and the one on the length-0 utterance
    good = [m for m in range(len(utt)) if m not in bad]
    perm = np.random.default_rng(0).permutation(len(utt))   # hand them over in a shuffled order
    off = np.concatenate([[0], np.cumsum(ly)])
    p_labels = np.concatenate([labels[off[m]:off[m + 1]] for m in perm]).astype(np.int32)
    p_utt, p_ly = utt[perm], ly[perm]
    inv = np.argsort(perm)
    w = torch.tensor(np.random.default_rng(2).uniform(0.5, 2.0, len(utt)).astype(np.float32), device="cuda")
    raw = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits, reduction="none")
    c0, _ = _run(raw, yt, p_labels, lens, p_ly, p_utt, w[perm])
    c0 = c0.cpu().numpy()[inv]
    assert c0[bad[0]] == np.inf and not np.isfinite(c0[bad[1]])
    crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits, reduction="none", zero_infinity=True)
    c1, g1 = _run(crit, yt, p_labels, lens, p_ly, p_utt, w[perm])
    c1, g1 = c1.cpu().numpy()[inv], g1.cpu().numpy()
    assert c1[bad[0]] == 0.0 and c1[bad[1]] == 0.0 and np.isfinite(g1).all()
    assert not g1[2].any()
    sub_labels = np.concatenate([labels[off[m]:off[m + 1]] for m in good]).astype(np.int32)
    rc, rg = _run(raw, yt, sub_labels, lens, ly[good], utt[good], w[good])
    _close(c1[good], rc.cpu().numpy(), 1e-6)
    assert np.abs(g1 - rg.cpu().numpy()).max() <= 1e-6
    with torch.no_grad():
        ev = crit(yt, _i32(p_labels), _i32(lens), _i32(p_ly), utt=_i32(p_utt)).cpu().numpy()[inv]
    assert ev[bad[0]] == 0.0 and ev[bad[1]] == 0.0
    _close(ev[good], c1[good], 1e-6)
    del ctx


def test_den_work_independent_of_k(tmp_graphs):
    """M = 4N sequences make as many launches as M = N, in the training call and in the forward-only one, and the peak
    allocated memory rises by no more than the larger numerator workspace."""
    import ctc_crf
    from cat_b200 import _C, _lib
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    N, T = 16, 40
    yt, _, lens = _batch(N, T, V, 71, np.full(N, T, np.int32), torch.float32, False)
    counts, peaks, maxls = {}, {}, {}
    for k in (1, 4):
        utt, labels, ly = _seqs([k] * N, lens, V, seed=k)
        args = (_i32(labels), _i32(lens), _i32(ly))
        crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1)
        y = yt.clone().requires_grad_(True)
        crit(y, *args, utt=_i32(utt)).backward()      # warm-up
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        k0 = _C.launch_count()
        crit(y, *args, utt=_i32(utt)).backward()
        k1 = _C.launch_count()
        torch.cuda.synchronize()
        peaks[k] = torch.cuda.max_memory_allocated() - base
        with torch.no_grad():
            crit(yt, *args, utt=_i32(utt))
        counts[k] = (k1 - k0, _C.launch_count() - k1)
        maxls[k] = int(ly.max())
    assert counts[1] == counts[4], counts
    L = _lib.lib()
    ws = {k: int(L.ccb_ctc_workspace_bytes(k * N, T, maxls[k])) for k in (1, 4)}
    assert peaks[4] - peaks[1] <= ws[4] - ws[1] + (1 << 16), (peaks, ws)
    del ctx


def test_bad_utt_rejected_on_the_gpu(tmp_graphs):
    import ctc_crf
    path, g, V = tmp_graphs["tlm_small"]
    ctx = _ctx(path)
    yt, _, lens = _batch(3, 10, V, 1, np.full(3, 10, np.int32), torch.float32, False)
    utt, labels, ly = _seqs([1, 1, 1], lens, V, seed=1)
    crit = ctc_crf.CTC_CRF_LOSS()
    with pytest.raises(RuntimeError, match="int32 CPU"):
        crit(yt, _i32(labels), _i32(lens), _i32(ly), utt=_i32(utt).cuda())
    with pytest.raises(RuntimeError, match=r"\[0, N\)"):
        crit(yt, _i32(labels), _i32(lens), _i32(ly), utt=_i32([0, 3, 1]))
    with pytest.raises(RuntimeError, match="one entry per label sequence"):
        crit(yt, _i32(labels), _i32(lens), _i32(ly), utt=_i32([0, 1]))
    del ctx
