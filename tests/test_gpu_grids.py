"""GPU: the den kernels on plans cut for grids other than this device's, through the Init-time hook CCB_DEN_CTAS = n.

Every other GPU test runs the plan for the device's own SM count (132 on an H100 SXM).  Other sm_90a parts have fewer SMs
(H100 PCIe 114, H20 78), and the SM count decides where the CTA tiles are cut, the label range of each tile (the backward
label accumulator's rows), the largest tile and so the tier ChooseDenLaunch picks, and whether the plan keeps its own-row
terms.  Each case sets CCB_DEN_CTAS, builds a fresh CRFContext, checks through ccb_plan_launch that the launch is the one
it claims (tests/test_den_launch.py pins them on the CPU) and compares against the fp64 oracle.

Tolerances are the suite's (BASELINE.json north_star): loss 1e-4 relative, gradients 1e-3 absolute (occupancies in [0, 1]).
"""
import ctypes as C
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-4
GRAD_ATOL = 1e-3
SAME_RTOL = 1e-6      # one path against another on the same plan: den atomics only
CTAS = (114, 78, 16, 4, 1)
TIER_SHARED, TIER_GLOBAL, TIER_STREAMED, TIER_SMALL = 0, 1, 2, 3

FIELDS = ("tier", "lanes", "U", "batch", "w1_smem", "Npad", "tile_rows", "gacc_rows", "arcs_off", "ring_off", "bar_off",
          "w1_off", "abar_off", "aring_off", "total")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ctx(monkeypatch, path, n_ctas):
    """A den context whose plan and grid are cut for n_ctas CTAs."""
    import ctc_crf
    if n_ctas > _sms():
        pytest.skip(f"{n_ctas} CTAs need at least as many SMs")
    monkeypatch.setenv("CCB_DEN_CTAS", str(n_ctas))
    return ctc_crf.CRFContext(path, gpus=0)


class _Plan:
    """The host-side plan for n_ctas CTAs (built with the environment's test hooks, as Init builds it)."""

    def __init__(self, path, n_ctas):
        from cat_b200 import _lib
        self.L, self.err = _lib.lib(), _lib.last_error
        self.h = self.L.ccb_plan_create(path.encode(), n_ctas, 16)
        assert self.h, self.err()

    def launch(self, N, backward):
        """The den launch a call of N utterances makes on this device (den_launch.h ChooseDenLaunch, no test hooks)."""
        out = (C.c_long * len(FIELDS))()
        optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
        assert self.L.ccb_plan_launch(self.h, N, int(backward), optin, 0, out) == 0, self.err()
        return dict(zip(FIELDS, out))

    def info(self):
        out = (C.c_long * 13)()
        assert self.L.ccb_plan_info(self.h, out) == 0
        return [int(x) for x in out]

    def close(self):
        self.L.ccb_plan_destroy(self.h)


def _check_loaded(plan):
    """The context's device plan is this plan: the same padded arc slots in both passes (tile cuts pad them)."""
    from cat_b200 import _C
    info, den = plan.info(), _C.den_info()
    assert (den["fwd_slots"], den["bwd_slots"]) == (info[3], info[4]), (den, info)


def _den_grids(run, tmp_path):
    """Grid sizes of the den recursion kernels that `run` launches, from a torch.profiler trace."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    trace = tmp_path / "den_trace.json"
    prof.export_chrome_trace(str(trace))
    events = json.loads(trace.read_text())["traceEvents"]
    return {tuple(e["args"]["grid"]) for e in events
            if e.get("cat") == "kernel" and ("den_forward_kernel" in e["name"] or "den_backward_kernel" in e["name"])}


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32)


def _close(a, b, rtol=LOSS_RTOL):
    assert abs(a - b) <= rtol * max(1.0, abs(b)), (a, b)


def _ragged(N, T, seed, zero=True):
    """Lengths in [2, T] with T first, then 0 (or 2) and 1 at fixed places, N-1 one short of T."""
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
    T = grad.shape[1]
    past = torch.arange(T, device=grad.device)[None, :] >= torch.tensor(lens, device=grad.device)[:, None]
    assert not bool(grad[past].any())


def _gpu_den(y, lens):
    from cat_b200 import _C
    N = y.shape[0]
    logits = torch.tensor(y, device="cuda")
    grad = torch.zeros_like(logits)
    ca, cb = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    _C.gpu_den(logits, grad, _i32(lens).cuda(), ca, cb)
    return ca.cpu().numpy(), cb.cpu().numpy(), grad


def _den_vs_oracle(g, V, N, T, seed, sub=None):
    """_C.gpu_den: logZ from alpha and from beta and the occupancies against oracle.den on the utterances `sub` (all by
    default); rows past each length exactly zero.  Returns (lens, logZ alpha, logZ beta, occupancies on the device)."""
    from oracle import oracle
    lens = _ragged(N, T, seed)
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=seed, lens=lens)
    ca, cb, grad = _gpu_den(y, lens)
    _rows_past_len_zero(grad, lens)
    sub = np.arange(N) if sub is None else np.asarray(sub)
    la, lb, gd = oracle.den(g, y[sub], lens[sub], fast=True)
    np.testing.assert_allclose(ca[sub], la, rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(cb[sub], lb, rtol=LOSS_RTOL, atol=1e-4)
    d = np.abs(grad[torch.tensor(sub, device="cuda")].cpu().numpy() - gd).max()
    assert d < GRAD_ATOL, d
    return lens, ca, cb, grad


# ---------------------------------------------------------------------------------------------------------------------
# a. the suite's small graphs on every grid, through _C.gpu_den
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_ctas", CTAS)
@pytest.mark.parametrize("name", ["tlm_small", "random_split", "tlm_mid"])
def test_den_on_other_grids(tmp_graphs, monkeypatch, tmp_path, name, n_ctas):
    """N = 5 and 12: small-batch kernels; 40: two utterances per lane; 130: four per lane forwards (two lane groups
    backwards); 300: Npad 384.  Arcs resident, label accumulator present on every grid (tests/test_den_launch.py::
    test_small_graphs_on_other_grids); on one CTA tlm_mid's plan has no own-row terms.  The den kernels run on n_ctas CTAs."""
    path, g, V = tmp_graphs[name]
    plan = _Plan(path, n_ctas)
    ctx = _ctx(monkeypatch, path, n_ctas)
    try:
        _check_loaded(plan)
        for N in (5, 12, 40, 130, 300):
            f, b = plan.launch(N, False), plan.launch(N, True)
            want = (TIER_SMALL, 1, TIER_SMALL, 1) if N <= 16 else (TIER_SHARED, {40: 2}.get(N, 4), TIER_SHARED, 2)
            assert (f["tier"], f["U"], b["tier"], b["U"]) == want and b["gacc_rows"] > 0, (N, f, b)
            _den_vs_oracle(g, V, N, 20, seed=N + n_ctas)
        from oracle import oracle
        y, _, lens, _ = oracle.synth_batch(40, 6, V, seed=1)
        assert _den_grids(lambda: _gpu_den(y, lens), tmp_path) == {(n_ctas, 1, 1)}
    finally:
        plan.close()
        del ctx


# ---------------------------------------------------------------------------------------------------------------------
# b. the fused loss and its variants on tlm_mid at 78 and 1 CTAs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_ctas", [78, 1])
def test_fused_loss_on_other_grids(tmp_graphs, monkeypatch, n_ctas):
    """CTC_CRF_LOSS (autograd backward), forward-only under torch.no_grad, checkpointed alpha (_ckpt_k_override), fp16 raw
    logits (from_logits=True) and reduction='none' against the oracle, at N = 12 (small-batch kernels) and 40.  Each path
    sets its own ckpt_mode / ring offsets on the same den launches; on one CTA tlm_mid's plan has no own-row terms."""
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(monkeypatch, path, n_ctas)
    lamb = 0.1
    for N, T in ((12, 40), (40, 30)):
        y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=70 + N + n_ctas, lens=_ragged(N, T, seed=N, zero=False))
        args = (_i32(labels), _i32(lens), _i32(ly))
        oloss, ograd, oparts = oracle.ctc_crf(g, y, labels, lens, ly, lamb, size_average=False, fast=True)
        # training loss through autograd
        x = torch.tensor(y, device="cuda").requires_grad_(True)
        crit = ctc_crf.CTC_CRF_LOSS(lamb=lamb, size_average=False)
        loss = crit(x, *args)
        loss.backward()
        _close(float(loss.item()), oloss)
        assert np.abs(x.grad.cpu().numpy() - ograd).max() < GRAD_ATOL
        _rows_past_len_zero(x.grad, lens)
        # forward-only (alpha on the frame ring)
        with torch.no_grad():
            ev = crit(x.detach(), *args)
        _close(float(ev.item()), float(loss.item()), SAME_RTOL)
        # checkpointed alpha, every 4 frames
        monkeypatch.setattr(_C, "_ckpt_k_override", 4)
        ck_loss, ck_grad, ck_parts = _C.ctc_crf_loss_fwd(x.detach(), *args, lamb, False, want_parts=True)
        monkeypatch.setattr(_C, "_ckpt_k_override", None)
        _close(float(ck_loss.item()), float(loss.item()), SAME_RTOL)
        assert float((ck_grad - x.grad).abs().max()) < 1e-5
        np.testing.assert_allclose(ck_parts.cpu().numpy()[:N], oparts["logz_alpha"], rtol=LOSS_RTOL, atol=1e-4)
        # per-utterance costs, the gradient of a weighted sum
        w = np.random.default_rng(N).uniform(-2.0, 2.0, N).astype(np.float32)
        xc = torch.tensor(y, device="cuda").requires_grad_(True)
        costs = ctc_crf.CTC_CRF_LOSS(lamb=lamb, reduction="none")(xc, *args)
        (costs * torch.tensor(w, device="cuda")).sum().backward()
        ocost = oparts["logz_alpha"] - (1.0 + lamb) * oparts["logp_ctc"]
        np.testing.assert_allclose(costs.detach().cpu().numpy(), ocost, rtol=LOSS_RTOL, atol=1e-4)
        assert np.abs(xc.grad.cpu().numpy() - w[:, None, None] * ograd).max() < GRAD_ATOL
        # fp16 raw logits (log_softmax inside the call); the oracle is fed the fp16 values
        z = (y + 3.0 * np.random.default_rng(N).standard_normal((N, T, 1)) + 5.0).astype(np.float32)
        zt = torch.tensor(z, device="cuda").half()
        z_used = zt.float().cpu().numpy()
        zl, zg, zp = _C.ctc_crf_loss_fwd(zt, *args, lamb, False, want_parts=True, from_logits=True)
        zloss, zgrad, zparts = oracle.ctc_crf_from_logits(g, z_used, labels, lens, ly, lamb, size_average=False)
        _close(float(zl.item()), zloss)
        assert np.abs(zg.float().cpu().numpy() - zgrad).max() < GRAD_ATOL
        np.testing.assert_allclose(zp.cpu().numpy()[:N], zparts["logz_alpha"], rtol=LOSS_RTOL, atol=1e-3)
        _rows_past_len_zero(zg, lens)
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# c. the benchmark's graph and a wide-label graph
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def big_graphs(tmp_path_factory):
    """The benchmark's 1.02 M-arc den graph (BASELINE.json headline) and G4k (3 000 LM states, 4 000 labels)."""
    from cat_b200 import fst
    d = tmp_path_factory.mktemp("grid_graphs")
    out = {}
    for name, (H, deg, V) in (("headline", (20000, 24, 218)), ("G4k", (3000, 8, 4000))):
        g = fst.make_synthetic_den(H, deg, V, seed=7)
        fst.write_fst(str(d / f"{name}.fst"), g)
        out[name] = (str(d / f"{name}.fst"), g, V)
    return out


SH, GL, ST, SM = TIER_SHARED, TIER_GLOBAL, TIER_STREAMED, TIER_SMALL


@pytest.mark.parametrize("n_ctas,tiers_64,tiers_12", [
    (114, (SH, SH), (SM, SM)),      # H100 PCIe: own-row terms, 5 accumulator rows
    (78, (SH, SH), (SM, SM)),       # H20: the same tiers without own-row terms
    (16, (GL, ST), (GL, ST)),       # arcs from L2 forwards, streamed with TMA row staging backwards; no small-batch tier
    (4, (GL, GL), (GL, ST)),        # arcs from L2 in both passes with register gathers (N = 64), streamed backwards (N = 12)
])
def test_headline_graph_on_other_grids(big_graphs, monkeypatch, n_ctas, tiers_64, tiers_12):
    """The 1.02 M-arc graph at N = 64 and 12, T = 300 (tests/test_den_launch.py::test_headline_graph_on_other_grids):
    the oracle on the first, the length-1 and the last utterance; on every utterance logZ from alpha equals logZ from beta
    and every occupancy row inside the utterance sums to 1."""
    path, g, V = big_graphs["headline"]
    plan = _Plan(path, n_ctas)
    ctx = _ctx(monkeypatch, path, n_ctas)
    try:
        _check_loaded(plan)
        for N, tiers in ((64, tiers_64), (12, tiers_12)):
            f, b = plan.launch(N, False), plan.launch(N, True)
            assert (f["tier"], b["tier"]) == tiers, (N, f, b)
            assert b["gacc_rows"] > 0, b
            lens, ca, cb, grad = _den_vs_oracle(g, V, N, 300, seed=N + n_ctas, sub=[0, N // 2, N - 1])
            np.testing.assert_allclose(ca, cb, rtol=1e-5)
            rows = grad.sum(-1).cpu().numpy()
            inside = np.arange(300)[None, :] < lens[:, None]
            assert np.abs(rows[inside] - 1.0).max() < 1e-4
    finally:
        plan.close()
        del ctx


@pytest.mark.parametrize("N,gacc", [(64, True), (130, False)])
def test_wide_labels_at_78_ctas(big_graphs, monkeypatch, N, gacc):
    """G4k at 78 CTAs: 74 accumulator rows, which fit 64 lanes (N = 64) but not 256 (N = 130: the occupancies go straight
    into the gradient with global atomics).  At 132 CTAs both widths keep the accumulator."""
    path, g, V = big_graphs["G4k"]
    plan = _Plan(path, 78)
    ctx = _ctx(monkeypatch, path, 78)
    try:
        _check_loaded(plan)
        b = plan.launch(N, True)
        assert (b["tier"], b["gacc_rows"] > 0) == (TIER_SHARED, gacc), b
        _den_vs_oracle(g, V, N, 16, seed=N, sub=_lane_subset(N))
    finally:
        plan.close()
        del ctx


# ---------------------------------------------------------------------------------------------------------------------
# d. hub rows on a small grid
# ---------------------------------------------------------------------------------------------------------------------
def test_hub_rows_on_4_ctas(tmp_graphs, monkeypatch):
    """Rows of more than 10 in-arcs computed in atomically accumulated parts of 7 (CCB_HUB_IN_ARCS, CCB_PART_ARCS) on a
    4-CTA grid, where a tile holds hundreds of rows: one, two and four utterances per lane forwards at N = 12, 40 and 130
    (the small-batch kernels have no hub-row variant, so a plan with hubs pads 12 utterances to 32 lanes)."""
    monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
    monkeypatch.setenv("CCB_PART_ARCS", "7")
    path, g, V = tmp_graphs["tlm_mid"]
    plan = _Plan(path, 4)
    ctx = _ctx(monkeypatch, path, 4)
    try:
        assert plan.info()[12] > 0          # hub states
        _check_loaded(plan)
        for N, U, Npad in ((12, 1, 32), (40, 2, 64), (130, 4, 256)):
            f = plan.launch(N, False)
            assert (f["tier"], f["U"], f["Npad"]) == (TIER_SHARED, U, Npad), f
            _den_vs_oracle(g, V, N, 20, seed=N)
    finally:
        plan.close()
        del ctx


# ---------------------------------------------------------------------------------------------------------------------
# e. the hook's bounds
# ---------------------------------------------------------------------------------------------------------------------
def test_den_ctas_out_of_range(tmp_graphs, monkeypatch, tmp_path):
    """CCB_DEN_CTAS outside [1, SM count] makes CRFContext raise, naming the value and the SM count; once it is unset, a new
    context runs on every SM again."""
    import ctc_crf
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_small"]
    sms = _sms()
    for bad in ("0", str(sms + 1), "-3", "8x"):
        monkeypatch.setenv("CCB_DEN_CTAS", bad)
        with pytest.raises(RuntimeError, match=rf"CCB_DEN_CTAS={bad} .*\[1, {sms}\]"):
            ctc_crf.CRFContext(path, gpus=0)
    monkeypatch.delenv("CCB_DEN_CTAS")
    plan = _Plan(path, sms)
    ctx = ctc_crf.CRFContext(path, gpus=0)
    try:
        _check_loaded(plan)
        y, _, lens, _ = oracle.synth_batch(40, 6, V, seed=2)
        assert _den_grids(lambda: _gpu_den(y, lens), tmp_path) == {(sms, 1, 1)}
        _den_vs_oracle(g, V, 40, 20, seed=3)
    finally:
        plan.close()
        del ctx
