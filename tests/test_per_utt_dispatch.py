"""CPU: how CTC_CRF_LOSS and WARP_CTC_LOSS pass `reduction` and `zero_infinity` to the native layer.  Non-default values
reach the `_C` loss function of the grad mode in use (loss plus gradient, or forward only); unknown reductions raise
ValueError at construction; the defaults call exactly what they called before the two options existed, with the same
arguments.  The `_C` functions are replaced by fakes, so no GPU runs."""
import pytest
import torch


@pytest.fixture
def fake_core(monkeypatch):
    from cat_b200 import loss as loss_mod
    calls = []

    def out(logits, opts):
        n = logits.shape[0]
        return torch.arange(1.0, n + 1) if opts.get("reduction") == "none" else torch.full((1,), 1.0)

    def crf_fwd(logits, labels, lx, ly, lamb, size_average, want_parts=False, from_logits=False, **opts):
        calls.append(("ctc_crf_loss_fwd", lamb, size_average, dict(from_logits=from_logits, **opts)))
        return out(logits, opts), torch.ones(logits.shape), None

    def crf_fwd_only(logits, labels, lx, ly, lamb, size_average, want_parts=False, from_logits=False, **opts):
        calls.append(("ctc_crf_loss_fwd_only", lamb, size_average, dict(from_logits=from_logits, **opts)))
        return out(logits, opts), None

    def ctc_fwd(logits, labels, lx, ly, size_average, blank=0, **opts):
        calls.append(("ctc_loss_fwd", None, size_average, opts))
        return out(logits, opts), torch.ones(logits.shape), torch.zeros(logits.shape[0])

    def ctc_fwd_only(logits, labels, lx, ly, size_average, blank=0, **opts):
        calls.append(("ctc_loss_fwd_only", None, size_average, opts))
        return out(logits, opts), torch.zeros(logits.shape[0])

    def rows_scale(grad, w, lx, dtype):
        calls.append(("grad_rows_scale", None, None, dict(dtype=dtype)))
        return (grad * w.reshape(-1, 1, 1)).to(dtype)

    monkeypatch.setattr(loss_mod.core, "ctc_crf_loss_fwd", crf_fwd)
    monkeypatch.setattr(loss_mod.core, "ctc_crf_loss_fwd_only", crf_fwd_only)
    monkeypatch.setattr(loss_mod.core, "ctc_loss_fwd", ctc_fwd)
    monkeypatch.setattr(loss_mod.core, "ctc_loss_fwd_only", ctc_fwd_only)
    monkeypatch.setattr(loss_mod.core, "grad_rows_scale", rows_scale)
    return calls


def _args(dtype=torch.float32):
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)
    return torch.zeros(2, 5, 4, dtype=dtype), i32([1, 2, 3]), i32([5, 4]), i32([2, 1])


OPTIONS = [("none", False), ("none", True), (None, True)]


@pytest.mark.parametrize("reduction,zero_infinity", OPTIONS)
@pytest.mark.parametrize("from_logits", [False, True])
def test_crf_options_reach_the_training_call(fake_core, reduction, zero_infinity, from_logits):
    import ctc_crf
    y, lab, lx, ly = _args()
    y.requires_grad_(True)
    crit = ctc_crf.CTC_CRF_LOSS(lamb=0.2, size_average=False, from_logits=from_logits, reduction=reduction,
                                zero_infinity=zero_infinity)
    out = crit(y, lab, lx, ly)
    assert fake_core == [("ctc_crf_loss_fwd", 0.2, False,
                          dict(from_logits=from_logits, reduction=reduction, zero_infinity=zero_infinity))]
    assert out.shape == ((2,) if reduction == "none" else (1,))


@pytest.mark.parametrize("reduction,zero_infinity", OPTIONS)
@pytest.mark.parametrize("from_logits", [False, True])
@pytest.mark.parametrize("mode", ["no_grad", "inference_mode"])
def test_crf_options_reach_the_forward_only_call(fake_core, reduction, zero_infinity, from_logits, mode):
    import ctc_crf
    y, lab, lx, ly = _args()
    crit = ctc_crf.CTC_CRF_LOSS(lamb=0.2, from_logits=from_logits, reduction=reduction, zero_infinity=zero_infinity)
    with getattr(torch, mode)():
        out = crit(y, lab, lx, ly)
    assert fake_core == [("ctc_crf_loss_fwd_only", 0.2, True,
                          dict(from_logits=from_logits, reduction=reduction, zero_infinity=zero_infinity))]
    assert out.shape == ((2,) if reduction == "none" else (1,))


@pytest.mark.parametrize("reduction,zero_infinity", OPTIONS)
def test_ctc_options_reach_both_calls(fake_core, reduction, zero_infinity):
    import ctc_crf
    y, lab, lx, ly = _args()
    crit = ctc_crf.WARP_CTC_LOSS(size_average=False, reduction=reduction, zero_infinity=zero_infinity)
    crit(y.clone().requires_grad_(True), lab, lx, ly)
    with torch.no_grad():
        crit(y, lab, lx, ly)
    opts = dict(reduction=reduction, zero_infinity=zero_infinity)
    assert fake_core == [("ctc_loss_fwd", None, False, opts), ("ctc_loss_fwd_only", None, False, opts)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("crf", [True, False])
def test_per_utterance_backward_weights_rows_in_the_logits_dtype(fake_core, dtype, crf):
    """reduction='none': the backward is grad_rows_scale(G, grad_output, lx, logits dtype)."""
    import ctc_crf
    y, lab, lx, ly = _args(dtype)
    y.requires_grad_(True)
    crit = ctc_crf.CTC_CRF_LOSS(reduction="none") if crf else ctc_crf.WARP_CTC_LOSS(reduction="none")
    costs = crit(y, lab, lx, ly)
    w = torch.tensor([0.5, -2.0])
    (g,) = torch.autograd.grad(costs.mul(w).sum(), y)
    assert fake_core[-1] == ("grad_rows_scale", None, None, dict(dtype=dtype))
    assert g.dtype == dtype
    assert torch.equal(g.float(), torch.ones(y.shape) * w.reshape(-1, 1, 1))


@pytest.mark.parametrize("reduction", ["mean", "sum", "None", "", 0])
def test_unknown_reduction_raises(reduction):
    import ctc_crf
    for make in (lambda: ctc_crf.CTC_CRF_LOSS(reduction=reduction), lambda: ctc_crf.WARP_CTC_LOSS(reduction=reduction)):
        with pytest.raises(ValueError, match="size_average"):
            make()


def test_unknown_reduction_raises_in_C():
    from cat_b200 import _C
    y, lab, lx, ly = _args()
    for fn in (_C.ctc_crf_loss_fwd, _C.ctc_crf_loss_fwd_only):
        with pytest.raises(ValueError, match="size_average"):
            fn(y, lab, lx, ly, 0.1, True, reduction="mean")
    for fn in (_C.ctc_loss_fwd, _C.ctc_loss_fwd_only):
        with pytest.raises(ValueError, match="size_average"):
            fn(y, lab, lx, ly, True, reduction="mean")


@pytest.mark.parametrize("from_logits", [False, True])
def test_defaults_call_what_they_called_before(fake_core, from_logits):
    """Default reduction and zero_infinity: the same `_C` functions with the same arguments as without the options
    (no extra keyword reaches them), and the reference's backward (grads * grad_output)."""
    import ctc_crf
    y, lab, lx, ly = _args()
    y.requires_grad_(True)
    for crit in (ctc_crf.CTC_CRF_LOSS(lamb=0.3, from_logits=from_logits),
                 ctc_crf.CTC_CRF_LOSS(lamb=0.3, from_logits=from_logits, reduction=None, zero_infinity=False)):
        crit(y, lab, lx, ly).backward()
        with torch.no_grad():
            crit(y, lab, lx, ly)
    for crit in (ctc_crf.WARP_CTC_LOSS(), ctc_crf.WARP_CTC_LOSS(size_average=True, reduction=None, zero_infinity=False)):
        crit(y, lab, lx, ly).backward()
        with torch.no_grad():
            crit(y, lab, lx, ly)
    crf = [("ctc_crf_loss_fwd", 0.3, True, dict(from_logits=from_logits)),
           ("ctc_crf_loss_fwd_only", 0.3, True, dict(from_logits=from_logits))]
    ctc = [("ctc_loss_fwd", None, True, {}), ("ctc_loss_fwd_only", None, True, {})]
    assert fake_core == crf + crf + ctc + ctc


def test_options_reassigned_after_construction(fake_core):
    """`reduction` and `zero_infinity` are read at every call: setting them on a built module takes effect in both grad
    modes, and setting them back restores the default call."""
    import ctc_crf
    y, lab, lx, ly = _args()
    y.requires_grad_(True)
    crit = ctc_crf.CTC_CRF_LOSS(lamb=0.2)
    warp = ctc_crf.WARP_CTC_LOSS()
    for m in (crit, warp):
        m.reduction, m.zero_infinity = "none", True
    assert crit(y, lab, lx, ly).shape == (2,) and warp(y, lab, lx, ly).shape == (2,)
    with torch.no_grad():
        assert crit(y, lab, lx, ly).shape == (2,) and warp(y, lab, lx, ly).shape == (2,)
    opts = dict(reduction="none", zero_infinity=True)
    assert fake_core == [("ctc_crf_loss_fwd", 0.2, True, dict(from_logits=False, **opts)), ("ctc_loss_fwd", None, True, opts),
                         ("ctc_crf_loss_fwd_only", 0.2, True, dict(from_logits=False, **opts)),
                         ("ctc_loss_fwd_only", None, True, opts)]
    del fake_core[:]
    crit.reduction, crit.zero_infinity = None, False
    assert crit(y, lab, lx, ly).shape == (1,)
    assert fake_core == [("ctc_crf_loss_fwd", 0.2, True, dict(from_logits=False))]
    crit.reduction = "mean"
    with pytest.raises(ValueError, match="size_average"):
        crit(y, lab, lx, ly)


def test_new_symbols_declared():
    """The entries that carry the costs and the mask are part of the C ABI the library declares and the loader binds."""
    from cat_b200 import _lib
    for s in ("ccb_ctc_crf_loss_costs", "ccb_ctc_crf_loss_costs_fwd_only", "ccb_ctc_loss_costs", "ccb_grad_rows_scale"):
        assert s in _lib.SYMBOLS
        assert hasattr(_lib.lib(), s)
