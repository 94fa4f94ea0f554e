"""GPU: a call lives on the caller's CUDA stream and does not stop the host.

include/ctc_crf_b200.h promises that everything is enqueued on `stream`, `_C.py` passes `torch.cuda.current_stream`, and
the fused entries promise never to synchronise the host.  On the legacy default stream -- where every other test runs --
a launch without its stream argument, a `cudaMemset` that should be `cudaMemsetAsync(..., stream)` or a staging copy
recorded on the wrong stream is ordered correctly by implicit synchronisation.  Here all work is done inside
`torch.cuda.stream(s)` for a side stream `s` that does not synchronise with the legacy stream, which stays idle:

* in: the logits hold NaN until a copy that sits on `s` behind a delay of tens of milliseconds fills them in; anything of
  ours that is not on `s` runs against NaN logits (or an accumulator not yet zeroed) and the result is wrong every time;
* out: the outputs are consumed on `s`, then, behind a second delay, the logits are overwritten with NaN on `s`; the host
  synchronises `s` once at the end.  Results against the same calls on the default stream and against the fp64 oracle;
* the host: behind a 100 ms delay on `s`, an entry that promises not to synchronise returns while `s` is still busy, for
  the first four calls on a fresh staging ring; the fifth reuses the first one's pinned buffer and waits for its copy.

Two of the library's calls in flight at once on two streams is not tested: the scratch of the reference-signature route
is per device, and CAT never does it.
"""
import math

import numpy as np
import pytest
import torch

from test_gpu_input_values import GRAD_ATOL, LAMB, LOSS_RTOL, _i32, _np
from test_gpu_scratch_contents import _same_outputs

pytestmark = pytest.mark.gpu

CYCLES_PER_MS = 1_500_000       # of torch.cuda._sleep; an H100 runs at 1.7 to 2.0 GHz, so a "millisecond" here is 0.75 to 0.9 ms


def _delay(ms):
    torch.cuda._sleep(int(ms * CYCLES_PER_MS))


def _ctx(path, gpu=0):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=gpu)


def _case(N, T, V, seed):
    from oracle import oracle
    lens = np.random.default_rng(seed).integers(1, T - 2, size=N).astype(np.int32)
    lens[0] = T - 3
    return oracle.synth_batch(N, T, V, seed=seed, lens=lens)


def _seq_case(N, lens, V, seed):
    from test_gpu_multi_seq import _seqs
    return _seqs([(3 * n + 1) % 4 for n in range(N)], lens, V, seed=seed)


def _entries(x, labels, lens, ly, utt, ulabels, uly, w, wu, delay_ms):
    """The loss entries on the current stream, backward passes included; `w` / `wu` (host arrays) become the grad_output
    of the reduction='none' calls on the current stream behind a delay.  Every output is cloned on the current stream."""
    import ctc_crf
    a = (_i32(labels), _i32(lens), _i32(ly))
    au = (_i32(ulabels), _i32(lens), _i32(uly))
    out = {}

    def leaf():
        return x.detach().clone().requires_grad_(True)

    xs = leaf()                                                       # the scalar: backward = grads * grad_output
    loss = ctc_crf.CTC_CRF_LOSS(lamb=LAMB)(xs, *a)
    loss.backward()
    out.update(loss=loss.detach().reshape(1), grad=xs.grad)
    xn = leaf()                                                       # 'none': backward = grad_rows_scale
    costs = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, reduction="none")(xn, *a)
    _delay(delay_ms)
    wt = torch.from_numpy(w).pin_memory().to(x.device, non_blocking=True)
    costs.backward(wt)
    out.update(costs=costs.detach(), grad_costs=xn.grad)
    xu = leaf()                                                       # utt= with 'none': backward = seqs_backward
    cu = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, reduction="none")(xu, *au, utt=_i32(utt))
    _delay(delay_ms)
    wut = torch.from_numpy(wu).pin_memory().to(x.device, non_blocking=True)
    cu.backward(wut)
    out.update(costs_seqs=cu.detach(), grad_seqs=xu.grad)
    xw = leaf()
    wl = ctc_crf.WARP_CTC_LOSS()(xw, *a)
    wl.backward()
    out.update(ctc_loss=wl.detach().reshape(1), grad_ctc=xw.grad)
    with torch.no_grad():
        out["loss_eval"] = ctc_crf.CTC_CRF_LOSS(lamb=LAMB)(x, *a).reshape(1)
    out["align"], out["score"] = ctc_crf.ctc_align(x, *a)
    return {k: v.clone() for k, v in out.items()}


def _ordered_run(dev, src, args, delay_ms=40):
    """The in / out ordering described at the top of this file, on a fresh side stream of `dev`.  Returns the outputs."""
    s = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(s):
        x = torch.full(tuple(src.shape), math.nan, device=dev)
        _delay(delay_ms)
        x.copy_(src, non_blocking=True)
        out = _entries(x, *args, delay_ms=delay_ms)
        sums = {k: v.float().sum() for k, v in out.items()}          # consumed on s
        _delay(delay_ms)
        x.fill_(math.nan)
    s.synchronize()
    assert torch.cuda.default_stream(dev).query()
    for k, v in sums.items():
        assert math.isfinite(float(v)), k
    return out


def _ordering_case(g, V, dev):
    from oracle import oracle
    from test_gpu_multi_seq import _oracle, _rows
    N, T = 12, 33
    y, labels, lens, ly = _case(N, T, V, seed=7)
    utt, ulabels, uly = _seq_case(N, lens, V, seed=8)
    w = np.linspace(-1.0, 0.9, N).astype(np.float32)
    wu = np.random.default_rng(9).uniform(-1.0, 1.0, len(utt)).astype(np.float32)
    args = (labels, lens, ly, utt, ulabels, uly, w, wu)
    src = torch.tensor(y).pin_memory()
    got = _np(_ordered_run(dev, src, args), torch.float32)
    with torch.cuda.device(dev):
        ref = _np(_entries(torch.tensor(y, device=dev), *args, delay_ms=0), torch.float32)
        torch.cuda.synchronize()
    _same_outputs(ref, got, "side stream against default stream")
    oloss, ograd, op = oracle.ctc_crf(g, y, labels, lens, ly, LAMB, size_average=True)
    assert abs(float(got["loss"][0]) - oloss) <= LOSS_RTOL * max(1.0, abs(oloss))
    assert abs(float(got["loss_eval"][0]) - oloss) <= LOSS_RTOL * max(1.0, abs(oloss))
    assert np.abs(got["grad"] - ograd).max() < GRAD_ATOL
    ocost = op["logz_alpha"] - (1.0 + LAMB) * op["logp_ctc"]
    np.testing.assert_allclose(got["costs"], ocost, rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(got["grad_costs"] - (w * N)[:, None, None] * ograd).max() < GRAD_ATOL
    ucost, ugrad = _oracle(g, y, ulabels, lens, uly, utt, LAMB, False)
    np.testing.assert_allclose(got["costs_seqs"], ucost, rtol=LOSS_RTOL, atol=1e-4)
    assert np.abs(got["grad_seqs"] - _rows(ugrad, utt, wu, N)).max() < GRAD_ATOL
    lp, gc = oracle.ctc(y, labels, ly, lens)
    assert abs(float(got["ctc_loss"][0]) + lp.sum() / N) <= LOSS_RTOL * max(1.0, abs(lp.sum() / N))
    assert np.abs(got["grad_ctc"] + gc / N).max() < GRAD_ATOL


def test_ordering_on_a_side_stream(tmp_graphs):
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    _ordering_case(g, V, torch.device("cuda", 0))
    del ctx


def test_ordering_on_a_second_device(tmp_graphs):
    """The same with the stream, the tensors and the den graph on device 1 while device 0 is the current device."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path, gpu=1)
    assert torch.cuda.current_device() == 0
    _ordering_case(g, V, torch.device("cuda", 1))
    assert torch.cuda.current_device() == 0
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# the host is not stopped
# ---------------------------------------------------------------------------------------------------------------------
def _no_sync_entries(x, labels, lens, ly):
    """The entries of `_C` whose docstrings say that they never synchronise the host."""
    from cat_b200 import _C
    a = (_i32(labels), _i32(lens), _i32(ly))
    return {
        "ctc_crf_loss_fwd": lambda: _C.ctc_crf_loss_fwd(x, *a, LAMB, True),
        "ctc_crf_loss_fwd_only": lambda: _C.ctc_crf_loss_fwd_only(x, *a, LAMB, True),
        "ctc_loss_fwd": lambda: _C.ctc_loss_fwd(x, *a, True),
        "ctc_loss_fwd_only": lambda: _C.ctc_loss_fwd_only(x, *a, True),
    }


def test_docstrings_promise_no_host_synchronisation():
    from cat_b200 import _C
    for name in _no_sync_entries(None, [0], [0], [0]):
        doc = " ".join(getattr(_C, name).__doc__.lower().split())
        assert "never synchronises the host" in doc or "no host synchronisation" in doc, name
    assert "cpu" in _C.gpu_ctc.__doc__.lower()          # costs come back in host memory: that entry has to wait


@pytest.mark.parametrize("entry", ["ctc_crf_loss_fwd", "ctc_crf_loss_fwd_only", "ctc_loss_fwd", "ctc_loss_fwd_only"])
def test_call_returns_while_the_stream_is_busy(tmp_graphs, entry):
    """Behind a delay of about 100 ms on `s` the call returns with `s` still busy: it waited for nothing on the device.
    Four calls per fresh staging ring do; the fifth reuses the first one's pinned buffer and so waits for that copy."""
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    y, labels, lens, ly = _case(12, 33, V, seed=11)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.tensor(y, device="cuda")
        call = _no_sync_entries(x, labels, lens, ly)[entry]
        first = call()                                   # warm up: module load, allocator blocks of `s`, memory figure
        s.synchronize()
        _C._rings.clear()
        _delay(100)
        busy, kept = [], []
        for i in range(4):
            kept.append(call())
            busy.append(not s.query())
        ring = _C._rings[0]
        first_copy = ring.events[0]
        assert not first_copy.query()
        kept.append(call())                              # the fifth: waits for the first call's staging copy, no more
        assert first_copy.query() and ring.events[0] is not first_copy
    s.synchronize()
    assert busy == [True] * 4, busy
    for out in kept:                                     # and every call computed what the warm-up call computed
        for a, b in zip(first, out):
            if a is not None:
                assert torch.allclose(a, b, rtol=1e-5, atol=1e-6, equal_nan=True)
    del ctx


# ---------------------------------------------------------------------------------------------------------------------
# the reference-signature route across streams
# ---------------------------------------------------------------------------------------------------------------------
def test_gpu_den_moves_between_streams(tmp_graphs):
    """`_C.gpu_den` on stream A, then B, then A, at growing and shrinking (N, T), without a host synchronisation in between:
    the library-owned scratch is drained on the stream that used it last before it is regrown on another."""
    from oracle import oracle
    from cat_b200 import _C
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    runs = []
    for i, (s, N, T) in enumerate(((A, 12, 10), (B, 40, 24), (A, 3, 7), (B, 64, 30), (A, 12, 10))):
        lens = np.random.default_rng(20 + i).integers(1, T + 1, size=N).astype(np.int32)
        lens[0] = T
        y, _, lens, _ = oracle.synth_batch(N, T, V, seed=30 + i, lens=lens)
        src = torch.tensor(y).pin_memory()
        with torch.cuda.stream(s):
            x = torch.full((N, T, V), math.nan, device="cuda")
            lens_d = torch.zeros(N, dtype=torch.int32, device="cuda")
            _delay(20)
            x.copy_(src, non_blocking=True)
            lens_d.copy_(_i32(lens).pin_memory(), non_blocking=True)
            grad = torch.zeros_like(x)
            ca, cb = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
            _C.gpu_den(x, grad, lens_d, ca, cb)
            runs.append((y, lens, ca.clone(), cb.clone(), grad.clone(), x, lens_d, src))
    torch.cuda.synchronize()
    for y, lens, ca, cb, grad, *_ in runs:
        la, lb, gd = oracle.den(g, y, lens, fast=True)
        np.testing.assert_allclose(ca.cpu().numpy(), la, rtol=LOSS_RTOL, atol=1e-4)
        np.testing.assert_allclose(cb.cpu().numpy(), lb, rtol=LOSS_RTOL, atol=1e-4)
        assert np.abs(grad.cpu().numpy() - gd).max() < GRAD_ATOL
    del ctx
