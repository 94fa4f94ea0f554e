"""GPU: a call's result does not depend on the calls made before it.

Every other GPU test turns its result into numpy straight after the call, which synchronises the host.  A training loop
does not: calls of different shapes and kinds follow each other with work still in flight.  What then carries over from
one call to the next is the 4-slot pinned staging ring (`_C._PinnedRing`: a slot overwritten before its copy ran shows as
another call's labels), the library-owned scratch of `_C.gpu_den` (kept between calls, regrown, never cleared), the
caching allocator's blocks (a workspace is the previous call's workspace, still being read on the stream), the cached
memory figure behind the slice plan, and the state a reduction='none' call with `utt=` keeps for its backward.

One context, one scripted sequence of calls, each enqueued behind a short device-side delay so that the host runs ahead of
the device as it does in training, with no host synchronisation between them except where an entry's contract
has one (`_C.gpu_ctc` returns its costs on the CPU), results left on the device; then one synchronise, then every result
against the same call made alone after a synchronise (`_same_outputs`), and the first and the last against the fp64 oracle.
"""
import numpy as np
import pytest
import torch

from test_gpu_input_values import GRAD_ATOL, LAMB, LOSS_RTOL, _i32, _np
from test_gpu_scratch_contents import _same_outputs

pytestmark = pytest.mark.gpu


def _ctx(path):
    import ctc_crf
    return ctc_crf.CRFContext(path, gpus=0)


class _Case:
    """Seeded inputs of one call, different in every call: logits on the device (made before the script starts, so that
    no upload synchronises it), labels and lengths on the host."""

    def __init__(self, i, N, T, V, dtype=torch.float32, raw=False, seqs=False):
        from oracle import oracle
        from test_gpu_multi_seq import _seqs
        rng = np.random.default_rng(1000 + i)
        lens = rng.integers(1, T + 1, size=N).astype(np.int32)
        lens[rng.integers(0, N)] = T
        self.N, self.T, self.dtype = N, T, dtype
        self.y, self.labels, self.lens, self.ly = oracle.synth_batch(N, T, V, seed=1000 + i, lens=lens)
        if raw:
            self.y = (self.y + 3.0 * rng.standard_normal((N, T, 1)) + 5.0).astype(np.float32)
        self.x = torch.tensor(self.y, device="cuda").to(dtype)
        self.a = (_i32(self.labels), _i32(self.lens), _i32(self.ly))
        if seqs:
            self.utt, self.ulabels, self.uly = _seqs([(i + 3 * n) % 4 for n in range(N)], self.lens, V, seed=i)
            self.au = (_i32(self.ulabels), _i32(self.lens), _i32(self.uly))
            self.w = torch.tensor(rng.uniform(-1.0, 1.0, (2, len(self.utt))).astype(np.float32), device="cuda")
        else:
            self.w = torch.tensor(rng.uniform(-1.0, 1.0, (2, N)).astype(np.float32), device="cuda")
        self.lens_d = _i32(self.lens).cuda()

    def leaf(self):
        return self.x.detach().clone().requires_grad_(True)


def _autograd(crit, c, **kw):
    x = c.leaf()
    loss = crit(x, *(c.au if kw else c.a), **kw)
    (g,) = torch.autograd.grad(loss, x)
    return dict(loss=loss.detach().reshape(1), grad=g)


def _fused(c, fl=False):
    from cat_b200 import _C
    loss, grad, parts = _C.ctc_crf_loss_fwd(c.x, *c.a, LAMB, True, want_parts=True, from_logits=fl)
    return dict(loss=loss, grad=grad, parts=parts)


def _with(monkeypatch, name, value, fn):
    from cat_b200 import _C
    with monkeypatch.context() as m:
        m.setattr(_C, name, value)
        return fn()


def _den(c):
    from cat_b200 import _C
    grad = torch.zeros_like(c.x)
    ca, cb = torch.zeros(c.N, device="cuda"), torch.zeros(c.N, device="cuda")
    _C.gpu_den(c.x, grad, c.lens_d, ca, cb)
    return dict(den_logz_alpha=ca, den_logz_beta=cb, grad_den=grad)


def _ctc(c):
    from cat_b200 import _C
    xt = c.x.transpose(0, 1).contiguous()
    grads = torch.zeros_like(xt)
    costs = torch.zeros(c.N)
    _C.gpu_ctc(xt, grads, c.a[0], c.a[2], c.a[1], c.N, costs, 0)
    return dict(logp=costs, grad=grads.transpose(0, 1))


def _costs(c):
    import ctc_crf
    x = c.leaf()
    costs = ctc_crf.CTC_CRF_LOSS(lamb=LAMB, reduction="none", zero_infinity=True)(x, *c.a)
    (g,) = torch.autograd.grad(costs, x, c.w[0])
    return dict(costs=costs.detach(), grad_costs=g)


def _eval(c):
    import ctc_crf
    with torch.no_grad():
        return dict(loss_eval=ctc_crf.CTC_CRF_LOSS(lamb=LAMB)(c.x, *c.a).reshape(1),
                    costs_eval=ctc_crf.CTC_CRF_LOSS(lamb=LAMB, reduction="none")(c.x, *c.a))


def _align(c):
    import ctc_crf
    align, score = ctc_crf.ctc_align(c.x, *c.a)
    return dict(align=align, score=score)


def _deferred_fwd(c, kind):
    """The forward call of a reduction='none' loss whose backward runs later: (leaf, costs)."""
    import ctc_crf
    x = c.leaf()
    if kind == "crf_seqs":
        return x, ctc_crf.CTC_CRF_LOSS(lamb=LAMB, reduction="none")(x, *c.au, utt=_i32(c.utt))
    return x, ctc_crf.WARP_CTC_LOSS(reduction="none")(x, *c.a)


def _deferred_bwd(state, c, twice):
    x, costs = state
    out = dict(costs=costs.detach())
    (out["grad_0"],) = torch.autograd.grad(costs, x, c.w[0], retain_graph=twice)
    if twice:
        (out["grad_1"],) = torch.autograd.grad(costs, x, c.w[1])
    return out


def test_results_do_not_depend_on_earlier_calls(tmp_graphs, monkeypatch):
    import ctc_crf
    from oracle import oracle
    from cat_b200 import _C, _lib
    from test_gpu_multi_seq import _oracle, _rows
    path, g, V = tmp_graphs["tlm_mid"]
    ctx = _ctx(path)
    L = _lib.lib()
    shapes = [(3, 20), (8, 20), (12, 33), (130, 64), (1, 7), (64, 33), (12, 20), (40, 33), (3, 64), (12, 7), (40, 33),
              (40, 20), (40, 20), (64, 20), (3, 33), (40, 7), (130, 20), (130, 20), (12, 20)]
    cases = [_Case(i, N, T, V, dtype=torch.float16 if i == 5 else torch.float32, raw=i == 5, seqs=i in (1, 14))
             for i, (N, T) in enumerate(shapes)]
    c12 = cases[12]
    need32 = (int(L.ccb_den_alpha_floats(32, c12.T)) * 4 + int(L.ccb_den_aux_bytes(32, c12.T))
              + int(L.ccb_ctc_workspace_bytes(32, c12.T, int(c12.ly.max()))))
    budget_calls = []

    def small_budget(dev, need=0):
        budget_calls.append(need)
        return need32 + 4096

    script = [
        ("fused scalar through autograd", lambda c: _autograd(ctc_crf.CTC_CRF_LOSS(lamb=LAMB), c)),
        None,                                                          # 1: deferred CTC_CRF_LOSS('none', utt=) forward
        None,                                                          # 2: deferred WARP_CTC_LOSS('none') forward
        ("fused, three slices", _fused),
        ("gpu_den", _den),
        ("from_logits fp16", lambda c: _fused(c, fl=True)),
        ("forward only", _eval),
        ("checkpointed K=3", lambda c: _with(monkeypatch, "_ckpt_k_override", 3, lambda: _fused(c))),
        ("checkpointed K=5", lambda c: _with(monkeypatch, "_ckpt_k_override", 5, lambda: _fused(c))),
        ("per-utterance costs", _costs),
        ("gpu_den", _den),
        ("fused, one slice", _fused),
        ("fused, halved under a small memory figure",
         lambda c: _with(monkeypatch, "_scratch_budget", small_budget, lambda: _fused(c))),
        ("fused, one slice", _fused),
        ("utt= scalar", lambda c: _autograd(ctc_crf.CTC_CRF_LOSS(lamb=LAMB), c, utt=_i32(c.utt))),
        ("WARP_CTC_LOSS", lambda c: _autograd(ctc_crf.WARP_CTC_LOSS(), c)),
        ("ctc_align", _align),
        ("gpu_den", _den),
        ("gpu_ctc", _ctc),
    ]
    assert len(script) == len(cases)
    staged = []
    stage = _C._PinnedRing.stage
    monkeypatch.setattr(_C._PinnedRing, "stage", lambda self, parts, device: (staged.append(1), stage(self, parts, device))[1])
    torch.cuda.synchronize()
    _C._rings.clear()

    # ---- the script: no host synchronisation of ours between the calls
    results = [None] * len(script)
    for i, step in enumerate(script):
        torch.cuda._sleep(30_000_000)     # ~15 ms: the device stays behind the host, so staging copies are still pending
        if step is None:
            results[i] = _deferred_fwd(cases[i], "crf_seqs" if i == 1 else "ctc")
        else:
            results[i] = step[1](cases[i])
    results[2] = _deferred_bwd(results[2], cases[2], twice=False)      # after every other call took and gave back its scratch
    results[1] = _deferred_bwd(results[1], cases[1], twice=True)
    torch.cuda.synchronize()
    assert budget_calls, "the memory figure hook was not consulted"
    assert len(staged) >= 3 * len(_C._rings[0].bufs) + 1, len(staged)      # the staging ring wrapped at least three times
    n_script = len(staged)

    # ---- every call alone
    for i, step in enumerate(script):
        c = cases[i]
        torch.cuda.synchronize()
        if step is None:
            alone = _deferred_bwd(_deferred_fwd(c, "crf_seqs" if i == 1 else "ctc"), c, twice=i == 1)
            what = "deferred backward"
        else:
            alone = step[1](c)
            what = step[0]
        torch.cuda.synchronize()
        _same_outputs(_np(alone, c.dtype), _np(results[i], c.dtype), (i, what))

    assert len(staged) == 2 * n_script        # alone, every call staged what it staged in the script

    # ---- the first and the last against the oracle
    c = cases[0]
    oloss, ograd, _ = oracle.ctc_crf(g, c.y, c.labels, c.lens, c.ly, LAMB, size_average=True)
    got = _np(results[0], c.dtype)
    assert abs(float(got["loss"][0]) - oloss) <= LOSS_RTOL * max(1.0, abs(oloss))
    assert np.abs(got["grad"] - ograd).max() < GRAD_ATOL
    c = cases[1]
    got = _np(results[1], c.dtype)
    ocost, G = _oracle(g, c.y, c.ulabels, c.lens, c.uly, c.utt, LAMB, False)
    np.testing.assert_allclose(got["costs"], ocost, rtol=LOSS_RTOL, atol=1e-4)
    for j in (0, 1):                      # each backward of the retained graph: grad_output * G
        assert np.abs(got[f"grad_{j}"] - _rows(G, c.utt, c.w[j].cpu().numpy(), c.N)).max() < GRAD_ATOL
    c = cases[2]
    got = _np(results[2], c.dtype)
    lp, gc = oracle.ctc(c.y, c.labels, c.ly, c.lens)
    np.testing.assert_allclose(got["costs"], -lp, rtol=LOSS_RTOL)
    assert np.abs(got["grad_0"] + c.w[0].cpu().numpy()[:, None, None] * gc).max() < GRAD_ATOL
    del ctx


def test_context_replaced_while_alive(tmp_graphs):
    """`ctx2 = CRFContext(other_graph)` with the first context still referenced: calls use the new graph; when the first
    context is then released the new device graph survives (the library counts Init against Release per device)."""
    import ctc_crf
    from oracle import oracle
    path, g, V = tmp_graphs["tlm_mid"]
    path2, g2, V2 = tmp_graphs["random_split"]
    crit = ctc_crf.CTC_CRF_LOSS(lamb=LAMB)

    def check(graph, c):
        out = _np(_autograd(crit, c), c.dtype)
        oloss, ograd, _ = oracle.ctc_crf(graph, c.y, c.labels, c.lens, c.ly, LAMB, size_average=True)
        assert abs(float(out["loss"][0]) - oloss) <= LOSS_RTOL * max(1.0, abs(oloss))
        assert np.abs(out["grad"] - ograd).max() < GRAD_ATOL

    ctx = _ctx(path)
    check(g, _Case(50, 12, 20, V))
    ctx2 = _ctx(path2)
    check(g2, _Case(51, 12, 20, V2))
    del ctx
    check(g2, _Case(52, 40, 20, V2))
    check(g2, _Case(53, 3, 33, V2))
    del ctx2
