"""GPU: no result depends on what the scratch and output buffers held before the call.

Every workspace and output `cat_b200/_C.py` hands the library is a `torch.empty`.  In a test process that is fresh device
memory (zeros) or the block the same call just released (a valid image of what is about to be computed), so a word read
before it is written goes unnoticed; in a training process it is the encoder's activations.  Here `_C.torch` is replaced by
`test_scratch_proxy.ScratchProxy`, which fills the raw bytes of every such buffer: 0x00 for the clean run, then 0xFF (NaN
as fp32 / bf16 / fp16, -1 as int32) and 0x7F (3.39e38 as fp32: finite, overflows on the first add; 2139062143 as int32 --
-1 is the CORRECT value of `align` past each length, and a NaN can be swallowed by a max).  Each entry, in each launch regime
that carves its scratch differently, must give the clean run's outputs (`_same_outputs`: 1e-6 plus 32 fp32 ulps, the spread of
the den's atomics), gradient rows at t >= lx[n] exactly 0.0 and `align` there exactly -1; the clean run is checked
against the fp64 oracle (loss 1e-4 relative, gradients 1e-3), and the proxy must have seen an allocation of every
workspace size the call asks the library for.

The grid-barrier words of the den aux block are zeroed by a memset of the same call on the same stream before every den
launch (DESIGN.md "Who initialises the scratch"), which is why a poisoned aux block is safe to run.
"""
import numpy as np
import pytest
import torch

from test_gpu_grids import TIER_SHARED, TIER_SMALL, TIER_STREAMED, _Plan, _labels_of, _lane_subset
from test_gpu_input_values import (DTYPES, GRAD_ATOL, LAMB, LOSS_RTOL, _align, _crf_autograd, _crf_costs, _crf_native,
                                   _crf_no_grad, _gpu_den, _i32, _np, _padding_rows_zero, _raw, _same, _warp, _weights, SAME_TOL)
from test_scratch_proxy import ScratchProxy

pytestmark = pytest.mark.gpu

PATTERNS = (0xFF, 0x7F)


@pytest.fixture
def scratch(monkeypatch):
    from cat_b200 import _C
    proxy = ScratchProxy(0)
    monkeypatch.setattr(_C, "torch", proxy)
    return proxy


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


def _batch(N, T, V, seed, tmax=None):
    """A ragged batch in (N, T, V) logits with every length below T (whole frames beyond every slice), sorted longest first so
    that slices of a large batch walk different numbers of frames; one utterance of length 1.  Returns
    (y, labels, lens, ly, labels_bad, ly_bad): in the second labelling utterance N-1 has more labels than frames."""
    from oracle import oracle
    tmax = T - 3 if tmax is None else tmax
    rng = np.random.default_rng(seed)
    lens = np.sort(rng.integers(min(2, tmax), tmax + 1, size=N))[::-1].astype(np.int32)
    lens[0] = tmax
    if N > 1:
        lens[N // 2] = 1
    y, labels, lens, ly = oracle.synth_batch(N, T, V, seed=seed, lens=lens)
    ly_bad = ly.copy()
    ly_bad[N - 1] = lens[N - 1] + 2
    labels_bad = np.concatenate([labels[:int(ly[:N - 1].sum())],
                                 rng.integers(1, V, size=int(ly_bad[N - 1]))]).astype(np.int32)
    return y, labels, lens, ly, labels_bad, ly_bad


def _past(lens, T):
    return np.arange(T)[None, :] >= np.asarray(lens)[:, None]


def _rows_clean(out, lens, what):
    """Gradient rows at t >= lx[n] exactly 0.0 (not -0.0 times junk, not NaN), align there exactly -1."""
    _padding_rows_zero(out, lens, what)
    for k, v in out.items():
        if k.startswith("grad"):
            assert np.isfinite(v).all(), (what, k)
        if k == "align":
            assert (v[_past(lens, v.shape[1])] == -1).all(), (what, k)


def _same_outputs(clean, got, what):
    """`_same` on every output; the per-utterance costs relative to the largest cost of the call instead of to themselves.
    cost[n] = logZ[n] - (1+lamb) log p[n] is a difference of two fp32 numbers that each carry the run-to-run spread of
    their own magnitude (the den sums logZ with atomics in no fixed order), so a cost near zero -- a two-frame utterance
    with logZ = -6.4 and log p = -6.5 -- moves by 1.4e-6 when logZ moves by three ulps, which is 2e-6 of itself and 2e-8
    of the batch's largest cost."""
    costs = [k for k in clean if k.startswith("costs")]
    _same({k: v for k, v in clean.items() if k not in costs}, got, what)
    for k in costs:
        a, b = clean[k], got[k]
        fin = np.isfinite(a)
        assert np.array_equal(fin, np.isfinite(b)) and np.array_equal(a[~fin], b[~fin], equal_nan=True), (what, k)
        if fin.any():
            tol = SAME_TOL * max(1.0, float(np.abs(a[fin]).max()))
            assert np.abs(a[fin] - b[fin]).max() <= tol, (what, k, np.abs(a[fin] - b[fin]).max(), tol)


def _contents(scratch, run, lens, dtype, sizes=(), rows=True):
    """`run()` with every buffer zero-filled, then NaN / -1 filled, then 0x7F filled: the same outputs.  `sizes`: byte
    counts the proxy must have seen allocated during the clean run.  Returns the clean outputs."""
    scratch.byte = 0
    del scratch.record[:]
    clean = _np(run(), dtype)
    seen = {nb for nb, _, dev in scratch.record if dev.type == "cuda"}
    assert scratch.record and seen, "no allocation went through the proxy"
    missing = [s for s in sizes if int(s) not in seen]
    assert not missing, (missing, sorted(seen))
    if rows:
        _rows_clean(clean, lens, "clean")
    for byte in PATTERNS:
        scratch.byte = byte
        got = _np(run(), dtype)
        if rows:
            _rows_clean(got, lens, hex(byte))
        _same_outputs(clean, got, hex(byte))
    scratch.byte = 0
    return clean


def _slice_sizes(lens, ly, k=0):
    """Workspace bytes of every slice of the fused loss on this batch, and the slices."""
    from cat_b200 import _C, _lib
    L = _lib.lib()
    N = len(lens)
    slices = _C._plan_slices(L, _i32(lens), _i32(ly), N, 0, torch.device("cuda", 0))
    sizes = []
    for n0, n1, tmax, maxl, kk in slices:
        n = n1 - n0
        assert kk == k, (kk, k)
        alpha = L.ccb_den_ckpt_alpha_floats(n, tmax, k) if k else L.ccb_den_alpha_floats(n, tmax)
        sizes += [4 * int(alpha), int(L.ccb_den_aux_bytes(n, tmax)), int(L.ccb_ctc_workspace_bytes(n, tmax, maxl))]
    return sizes, slices


def _fwd_only_sizes(lens, ly):
    from cat_b200 import _C, _lib
    L = _lib.lib()
    sizes = []
    for n0, n1, tmax, _ in _C._plan_fwd_only_slices(L, _i32(lens), _i32(ly), len(lens), torch.device("cuda", 0)):
        n = n1 - n0
        sizes += [4 * int(L.ccb_den_fwd_alpha_floats(n)), int(L.ccb_den_aux_bytes(n, tmax)), int(L.ccb_num_fwd_only_bytes(n))]
    return sizes


def _crf_oracle(g, clean, y_used, labels, lens, ly, fl, sub):
    """`loss` / `grad` / `parts` of _crf_autograd (the mean over the batch) against the oracle on the utterances `sub`."""
    from oracle import oracle
    N = len(lens)
    sub = np.asarray(sub)
    fn = oracle.ctc_crf_from_logits if fl else oracle.ctc_crf
    _, ograd, op = fn(g, y_used[sub], _labels_of(labels, ly, sub), lens[sub], ly[sub], LAMB, size_average=False)
    assert np.isfinite(op["logz_alpha"]).all() and np.isfinite(op["logp_ctc"]).all()
    np.testing.assert_allclose(clean["parts"][:N][sub], op["logz_alpha"], rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(clean["parts"][N:][sub], op["logp_ctc"], rtol=LOSS_RTOL, atol=1e-4)
    ref = ograd / N
    assert np.all(np.abs(clean["grad"][sub] - ref) <= GRAD_ATOL + 0.5 * clean["_eps"] * np.abs(ref))
    if len(sub) == N:
        oloss = float((op["logz_alpha"] - (1.0 + LAMB) * op["logp_ctc"]).sum()) / N
        assert abs(float(clean["loss"][0]) - oloss) <= LOSS_RTOL * max(1.0, abs(oloss))


def _costs_oracle(g, clean, y_used, labels_bad, lens, ly_bad, fl):
    """`costs` / `grad_costs` of _crf_costs (zero_infinity, weights _weights(N)) on the labelling whose last utterance is
    infeasible: cost 0 and zero gradient rows there, the oracle on the first utterances."""
    from oracle import oracle
    N = len(lens)
    assert clean["costs"][N - 1] == 0.0 and not clean["grad_costs"][N - 1].any()
    assert clean["costs_eval"][N - 1] == 0.0
    sub = np.arange(min(N - 1, 4))
    fn = oracle.ctc_crf_from_logits if fl else oracle.ctc_crf
    _, ograd, op = fn(g, y_used[sub], _labels_of(labels_bad, ly_bad, sub), lens[sub], ly_bad[sub], LAMB, size_average=False)
    ocost = op["logz_alpha"] - (1.0 + LAMB) * op["logp_ctc"]
    np.testing.assert_allclose(clean["costs"][sub], ocost, rtol=LOSS_RTOL, atol=1e-4)
    ref = _weights(N).astype(np.float64)[sub, None, None] * ograd
    assert np.all(np.abs(clean["grad_costs"][sub] - ref) <= GRAD_ATOL + 0.5 * clean["_eps"] * np.abs(ref))


# ---------------------------------------------------------------------------------------------------------------------
# a. the fused entries in every lane layout
# ---------------------------------------------------------------------------------------------------------------------
LAYOUTS = {3: (TIER_SMALL, 16), 12: (TIER_SMALL, 16), 40: (TIER_SHARED, 64), 64: (TIER_SHARED, 64), 130: (TIER_SHARED, 256)}


@pytest.mark.parametrize("N,dtype", [(3, "fp32"), (12, "fp32"), (12, "fp16"), (40, "fp32"), (40, "bf16"), (64, "fp32"),
                                     (130, "fp32"), (130, "fp16")])
def test_fused_entries(tmp_graphs, scratch, N, dtype):
    """CTC_CRF_LOSS (scalar through autograd, under no_grad, reduction='none' with zero_infinity, an infeasible utterance and
    a non-constant grad_output), on log-probs and on raw logits, `_C.ctc_crf_loss_fwd(want_parts=True)`, WARP_CTC_LOSS with
    the same options and ctc_align.  N = 3, 12: 16-float rows; 40: 64 lanes of which 24 are padding nobody writes; 130: three
    slices of 64, 64 and 2 utterances walking different numbers of frames."""
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    dt = DTYPES[dtype]
    T = 33
    y, labels, lens, ly, labels_bad, ly_bad = _batch(N, T, V, seed=100 + N)
    assert lens.max() < T and (lens < lens.max()).any()
    plan = _Plan(path, torch.cuda.get_device_properties(0).multi_processor_count)
    ctx = _ctx(path)
    try:
        L = _C._lib.lib()
        sizes, slices = _slice_sizes(lens, ly)
        if N == 130:
            assert [(s[0], s[1]) for s in slices] == [(0, 64), (64, 128), (128, 130)] and len({s[2] for s in slices}) == 3
        for n0, n1, tmax, _, _ in slices:
            f, b = plan.launch(n1 - n0, False), plan.launch(n1 - n0, True)
            if N != 130:
                assert (f["tier"], f["Npad"], b["Npad"]) == LAYOUTS[N] + (LAYOUTS[N][1],), (f, b)
            assert int(L.ccb_den_alpha_floats(n1 - n0, tmax)) % f["Npad"] == 0
            if N == 40:
                assert f["Npad"] > N
        sizes += _fwd_only_sizes(lens, ly) + [int(L.ccb_ctc_align_workspace_bytes(N, T, int(ly.max())))]
        sizes += [int(L.ccb_ctc_workspace_bytes(N, int(lens.max()), int(ly.max())))]          # WARP_CTC_LOSS
        sub = np.arange(N) if N <= 12 else _lane_subset(N)[:5]
        for fl in (False, True):
            yt = torch.tensor(_raw(y, N) if fl else y, device="cuda").to(dt)
            y_used = yt.float().cpu().numpy()

            def run():
                x = yt.clone()
                out = _crf_autograd(x, labels, lens, ly, fl)
                out.update(_crf_no_grad(x, labels, lens, ly, fl))
                out.update(_crf_costs(x, labels_bad, lens, ly_bad, fl))
                if not fl:
                    out.update(_warp(x, labels, lens, ly))
                    out.update(_align(x, labels, lens, ly))
                return out

            clean = _contents(scratch, run, lens, dt, sizes=() if fl else sizes)
            for k in ("loss", "loss_eval") + (() if fl else ("ctc_loss", "ctc_loss_eval")):
                assert np.isfinite(clean[k]).all(), k
            _crf_oracle(g, clean, y_used, labels, lens, ly, fl, sub)
            _costs_oracle(g, clean, y_used, labels_bad, lens, ly_bad, fl)
    finally:
        plan.close()
        del ctx


# ---------------------------------------------------------------------------------------------------------------------
# b. the reference-signature entries
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,N", [("tlm_mid", 3), ("tlm_mid", 12), ("tlm_mid", 40), ("tlm_mid", 64), ("tlm_mid", 130),
                                    ("tlm_small", 40), ("random_split", 40), ("random_split", 130)])
def test_gpu_den_caller_alpha(tmp_graphs, scratch, name, N):
    """`_C.gpu_den` with the alpha it sizes itself from ccb_den_alpha_floats (poisoned: padding lanes, parked pair rows) and
    the library-owned aux block behind it; 130 utterances are several lane groups in one call."""
    from oracle import oracle
    from cat_b200 import _C
    path, g, V = tmp_graphs[name]
    T = 20
    y, _, lens, _, _, _ = _batch(N, T, V, seed=200 + N)
    plan = _Plan(path, torch.cuda.get_device_properties(0).multi_processor_count)
    ctx = _ctx(path)
    try:
        f = plan.launch(N, False)
        if name == "tlm_mid":
            assert (f["tier"], f["Npad"]) == LAYOUTS[N], f
        L = _C._lib.lib()
        need = int(L.ccb_den_alpha_floats(N, T))
        assert need % f["Npad"] == 0
        per = (T + 1) * N
        yt = torch.tensor(y, device="cuda")
        clean = _contents(scratch, lambda: _gpu_den(yt, lens), lens, torch.float32,
                          sizes=[4 * per * max(-(-need // per), _C.den_num_states())])
        sub = np.arange(N) if N <= 12 else _lane_subset(N)
        la, lb, gd = oracle.den(g, y[sub], lens[sub], fast=True)
        np.testing.assert_allclose(clean["den_logz_alpha"][sub], la, rtol=LOSS_RTOL, atol=1e-4)
        np.testing.assert_allclose(clean["den_logz_beta"][sub], lb, rtol=LOSS_RTOL, atol=1e-4)
        assert np.abs(clean["grad_den"][sub] - gd).max() < GRAD_ATOL
    finally:
        plan.close()
        del ctx


def test_gpu_ctc(scratch):
    """`_C.gpu_ctc` in its (T,N,V) layout: the workspace holds its meta block, the costs and the cells."""
    from oracle import oracle
    from cat_b200 import _C
    N, T, V = 7, 30, 23
    y, labels, lens, ly, _, _ = _batch(N, T, V, seed=41)
    yt = torch.tensor(y, device="cuda").transpose(0, 1).contiguous()

    def run():
        grads = torch.zeros_like(yt)
        costs = torch.zeros(N)
        _C.gpu_ctc(yt, grads, _i32(labels), _i32(ly), _i32(lens), N, costs, 0)
        return dict(logp=costs, grad=grads.transpose(0, 1))

    clean = _contents(scratch, run, lens, torch.float32)
    lp, gc = oracle.ctc(y, labels, ly, lens)
    np.testing.assert_allclose(clean["logp"], lp, rtol=LOSS_RTOL)
    assert np.abs(clean["grad"] - gc).max() < GRAD_ATOL


# ---------------------------------------------------------------------------------------------------------------------
# c. checkpointed alpha and the forward-only ring
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [12, 40])
@pytest.mark.parametrize("K", ["1", "sqrt", "all"])
def test_checkpointed_alpha(tmp_graphs, scratch, monkeypatch, K, N):
    """K = 1 (every frame a checkpoint), ceil(sqrt(T)) with T not a multiple of it, and K >= T (one segment): segment
    positions, checkpoints and the carried log-scales are carved from one poisoned buffer."""
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    T, tmax = 34, 31
    k = {"1": 1, "sqrt": _C.ckpt_interval(tmax), "all": tmax + 5}[K]
    assert K != "sqrt" or (k == 6 and tmax % k)
    monkeypatch.setattr(_C, "_ckpt_k_override", k)
    y, labels, lens, ly, labels_bad, ly_bad = _batch(N, T, V, seed=300 + N)
    ctx = _ctx(path)
    sizes, slices = _slice_sizes(lens, ly, k)
    assert len(slices) == 1 and slices[0][2] == tmax
    for fl in (False, True):
        yt = torch.tensor(_raw(y, 5) if fl else y, device="cuda")

        def run():
            out = _crf_autograd(yt.clone(), labels, lens, ly, fl)
            out.update(_crf_costs(yt.clone(), labels_bad, lens, ly_bad, fl))
            return out

        clean = _contents(scratch, run, lens, torch.float32, sizes=sizes)
        _crf_oracle(g, clean, yt.cpu().numpy(), labels, lens, ly, fl, np.arange(N) if N <= 12 else _lane_subset(N)[:5])
        _costs_oracle(g, clean, yt.cpu().numpy(), labels_bad, lens, ly_bad, fl)
    del ctx


@pytest.mark.parametrize("N", [12, 40])
@pytest.mark.parametrize("tmax", [2, 4, 30])
def test_forward_only_ring(tmp_graphs, scratch, tmax, N):
    """The forward-only loss keeps alpha on a ring of 4 frames (plus two parked positions and one checkpoint): batches
    shorter than, as long as and longer than the ring."""
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_mid"]
    T = 33
    y, labels, lens, ly, _, _ = _batch(N, T, V, seed=400 + N + tmax, tmax=tmax)
    assert lens.max() == tmax
    ctx = _ctx(path)
    sizes = _fwd_only_sizes(lens, ly)
    for fl in (False, True):
        yt = torch.tensor(_raw(y, 6) if fl else y, device="cuda")

        def run():
            out = _crf_no_grad(yt, labels, lens, ly, fl)
            out["costs_eval"] = _crf_costs(yt.clone(), labels, lens, ly, fl)["costs_eval"]
            return out

        clean = _contents(scratch, run, lens, torch.float32, sizes=sizes)
        sub = np.arange(min(N, 6))
        fn = oracle.ctc_crf_from_logits if fl else oracle.ctc_crf
        _, _, op = fn(g, yt.cpu().numpy()[sub], _labels_of(labels, ly, sub), lens[sub], ly[sub], LAMB, size_average=False)
        np.testing.assert_allclose(clean["parts_eval"][:N][sub], op["logz_alpha"], rtol=LOSS_RTOL, atol=1e-4)
        np.testing.assert_allclose(clean["parts_eval"][N:][sub], op["logp_ctc"], rtol=LOSS_RTOL, atol=1e-4)
        np.testing.assert_allclose(clean["costs_eval"][sub], op["logz_alpha"] - (1.0 + LAMB) * op["logp_ctc"],
                                   rtol=LOSS_RTOL, atol=1e-4)
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# d. the den launches behind the Init-time hooks
# ---------------------------------------------------------------------------------------------------------------------
HOOKS = {
    "hubs": {"CCB_HUB_IN_ARCS": "10", "CCB_PART_ARCS": "7"},       # hub rows summed in parts into rows zeroed a frame ahead
    "arcs_in_global": {"CCB_ARCS_IN_GLOBAL": "1"},
    "w1_in_global": {"CCB_W1_IN_GLOBAL": "1"},
    "no_tma": {"CCB_NO_TMA": "1"},
    "own_in_l2": {"CCB_OWN_IN_L2": "1"},
    "no_pairs": {"CCB_NO_PAIRS": "1"},
}


@pytest.mark.parametrize("hook", sorted(HOOKS))
def test_den_hooks(tmp_graphs, scratch, monkeypatch, hook):
    """`_C.gpu_den` and the fused loss at N = 12 and 40 on the plans and launches the test hooks select."""
    from oracle import oracle
    for k, v in HOOKS[hook].items():
        monkeypatch.setenv(k, v)
    path, g, V = tmp_graphs["tlm_mid"]
    plan = _Plan(path, torch.cuda.get_device_properties(0).multi_processor_count)
    ctx = _ctx(path)
    try:
        if hook == "hubs":
            assert plan.info()[12] > 0
        for N in (12, 40):
            y, labels, lens, ly, _, _ = _batch(N, 24, V, seed=500 + N)
            yt = torch.tensor(y, device="cuda")

            def run():
                out = _gpu_den(yt, lens)
                out.update(_crf_native(yt, labels, lens, ly, False))
                return out

            clean = _contents(scratch, run, lens, torch.float32)
            sub = _lane_subset(N)[:5]
            la, lb, gd = oracle.den(g, y[sub], lens[sub], fast=True)
            np.testing.assert_allclose(clean["den_logz_alpha"][sub], la, rtol=LOSS_RTOL, atol=1e-4)
            np.testing.assert_allclose(clean["den_logz_beta"][sub], lb, rtol=LOSS_RTOL, atol=1e-4)
            assert np.abs(clean["grad_den"][sub] - gd).max() < GRAD_ATOL
            _crf_oracle(g, clean, y, labels, lens, ly, False, sub)
    finally:
        plan.close()
        del ctx


def test_streamed_backward_on_4_ctas(scratch, monkeypatch, tmp_path):
    """The 1.02 M-arc benchmark graph on a 4-CTA plan at N = 12: the backward pass streams its arcs through per-warp rings
    with TMA row staging."""
    from oracle import oracle
    from cat_b200 import fst
    g = fst.make_synthetic_den(20000, 24, 218, seed=7)
    path = str(tmp_path / "headline.fst")
    fst.write_fst(path, g)
    plan = _Plan(path, 4)
    try:
        assert plan.launch(12, True)["tier"] == TIER_STREAMED
    finally:
        plan.close()
    monkeypatch.setenv("CCB_DEN_CTAS", "4")
    ctx = _ctx(path)
    N, T = 12, 16
    y, _, lens, _, _, _ = _batch(N, T, 218, seed=61)
    yt = torch.tensor(y, device="cuda")
    clean = _contents(scratch, lambda: _gpu_den(yt, lens), lens, torch.float32)
    sub = np.array([0, N // 2, N - 1])
    la, lb, gd = oracle.den(g, y[sub], lens[sub], fast=True)
    np.testing.assert_allclose(clean["den_logz_alpha"][sub], la, rtol=LOSS_RTOL, atol=1e-4)
    np.testing.assert_allclose(clean["den_logz_beta"][sub], lb, rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(clean["grad_den"][sub] - gd).max() < GRAD_ATOL
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# e. several label sequences per utterance
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_multi_seq_entries(tmp_graphs, scratch, dtype):
    """CTC_CRF_LOSS, WARP_CTC_LOSS and ctc_align with `utt=`, the scalar and reduction='none' (whose backward runs on the
    numerator cells and den occupancies the forward call kept), with utterances that have no sequence: their gradient rows
    are exactly zero."""
    import ctc_crf
    from test_gpu_multi_seq import _oracle, _rows, _seqs
    path, g, V = tmp_graphs["tlm_mid"]
    dt = DTYPES[dtype]
    N, T = 8, 33
    y, _, lens, _, _, _ = _batch(N, T, V, seed=71)
    counts = [3, 0, 5, 1, 2, 4, 0, 1]
    utt, labels, ly = _seqs(counts, lens, V, seed=5)
    M = len(utt)
    w = np.random.default_rng(3).uniform(-1.0, 1.0, M).astype(np.float32)
    a = (_i32(labels), _i32(lens), _i32(ly))
    u = _i32(utt)
    ctx = _ctx(path)
    for fl in (False, True):
        yt = torch.tensor(_raw(y, 7) if fl else y, device="cuda").to(dt)
        wt = torch.tensor(w, device="cuda")

        def run():
            out = {}
            for tag, crit_none, crit_mean in (
                    ("crf", ctc_crf.CTC_CRF_LOSS(lamb=LAMB, from_logits=fl, reduction="none", zero_infinity=True),
                     ctc_crf.CTC_CRF_LOSS(lamb=LAMB, from_logits=fl)),
                    ("ctc", ctc_crf.WARP_CTC_LOSS(reduction="none", zero_infinity=True), ctc_crf.WARP_CTC_LOSS())):
                if fl and tag == "ctc":
                    continue
                x = yt.clone().requires_grad_(True)
                costs = crit_none(x, *a, utt=u)
                (gn,) = torch.autograd.grad((costs * wt).sum(), x)
                loss = crit_mean(x, *a, utt=u)
                (gm,) = torch.autograd.grad(loss, x)
                with torch.no_grad():
                    ev = crit_none(x.detach(), *a, utt=u)
                out.update({f"costs_{tag}": costs, f"grad_none_{tag}": gn, f"loss_{tag}": loss.reshape(1),
                            f"grad_mean_{tag}": gm, f"costs_eval_{tag}": ev})
            if not fl:
                out["align"], out["score"] = ctc_crf.ctc_align(yt, *a, utt=u)
            return out

        clean = _contents(scratch, run, lens, dt, rows=False)
        for k, v in clean.items():
            if k.startswith("grad"):
                assert np.isfinite(v).all() and not v[_past(lens, T)].any(), k
                assert not v[[n for n in range(N) if counts[n] == 0]].any(), k
        assert (clean["align"][_past(lens[utt], T)] == -1).all() if not fl else True
        ocost, ograd = _oracle(g, yt.float().cpu().numpy(), labels, lens, ly, utt, LAMB, fl)
        np.testing.assert_allclose(clean["costs_crf"], ocost, rtol=LOSS_RTOL, atol=1e-4)
        ref = _rows(ograd, utt, w, N)
        assert np.all(np.abs(clean["grad_none_crf"] - ref) <= GRAD_ATOL + 0.5 * clean["_eps"] * np.abs(ref))
        ref = _rows(ograd, utt, np.full(M, 1.0 / M), N)
        assert np.all(np.abs(clean["grad_mean_crf"] - ref) <= GRAD_ATOL + 0.5 * clean["_eps"] * np.abs(ref))
    del ctx
