"""CPU: which native entry CTC_CRF_LOSS and WARP_CTC_LOSS call.  With grad mode off (torch.no_grad, torch.inference_mode)
they take the forward-only entries; with grad mode on they take the loss-plus-gradient entries, also when the logits do
not require grad (a training step may time the loss that way).  The `_C` functions are replaced by fakes, so no GPU runs."""
import pytest
import torch


@pytest.fixture
def fake_core(monkeypatch):
    from cat_b200 import loss as loss_mod
    calls = []

    def crf_fwd(logits, labels, lx, ly, lamb, size_average, want_parts=False, from_logits=False):
        calls.append(("ctc_crf_loss_fwd", from_logits, lamb, size_average))
        return torch.full((1,), 1.0), torch.zeros(logits.shape), None

    def crf_fwd_only(logits, labels, lx, ly, lamb, size_average, want_parts=False, from_logits=False):
        calls.append(("ctc_crf_loss_fwd_only", from_logits, lamb, size_average))
        return torch.full((1,), 2.0), None

    def ctc_fwd(logits, labels, lx, ly, size_average, blank=0):
        calls.append(("ctc_loss_fwd", size_average))
        return torch.full((1,), 3.0), torch.zeros(logits.shape), torch.zeros(logits.shape[0])

    def ctc_fwd_only(logits, labels, lx, ly, size_average, blank=0):
        calls.append(("ctc_loss_fwd_only", size_average))
        return torch.full((1,), 4.0), torch.zeros(logits.shape[0])

    monkeypatch.setattr(loss_mod.core, "ctc_crf_loss_fwd", crf_fwd)
    monkeypatch.setattr(loss_mod.core, "ctc_crf_loss_fwd_only", crf_fwd_only)
    monkeypatch.setattr(loss_mod.core, "ctc_loss_fwd", ctc_fwd)
    monkeypatch.setattr(loss_mod.core, "ctc_loss_fwd_only", ctc_fwd_only)
    return calls


def _args():
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)
    return torch.zeros(2, 5, 4), i32([1, 2, 3]), i32([5, 4]), i32([2, 1])


MODES = {"no_grad": torch.no_grad, "inference_mode": torch.inference_mode}


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("from_logits", [False, True])
def test_crf_loss_without_grad_mode_is_forward_only(fake_core, mode, from_logits):
    import ctc_crf
    crit = ctc_crf.CTC_CRF_LOSS(lamb=0.25, size_average=False, from_logits=from_logits)
    y, lab, lx, ly = _args()
    with MODES[mode]():
        out = crit(y, lab, lx, ly)
    assert fake_core == [("ctc_crf_loss_fwd_only", from_logits, 0.25, False)]
    assert out.shape == (1,) and float(out) == 2.0


@pytest.mark.parametrize("mode", sorted(MODES))
def test_ctc_loss_without_grad_mode_is_forward_only(fake_core, mode):
    import ctc_crf
    y, lab, lx, ly = _args()
    with MODES[mode]():
        out = ctc_crf.WARP_CTC_LOSS(size_average=True)(y, lab, lx, ly)
    assert fake_core == [("ctc_loss_fwd_only", True)]
    assert out.shape == (1,) and float(out) == 4.0


@pytest.mark.parametrize("requires_grad", [False, True])
@pytest.mark.parametrize("from_logits", [False, True])
def test_crf_loss_with_grad_mode_keeps_the_gradient(fake_core, requires_grad, from_logits):
    import ctc_crf
    y, lab, lx, ly = _args()
    y.requires_grad_(requires_grad)
    assert torch.is_grad_enabled()
    ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits)(y, lab, lx, ly)
    assert fake_core == [("ctc_crf_loss_fwd", from_logits, 0.1, True)]


@pytest.mark.parametrize("requires_grad", [False, True])
def test_ctc_loss_with_grad_mode_keeps_the_gradient(fake_core, requires_grad):
    import ctc_crf
    y, lab, lx, ly = _args()
    y.requires_grad_(requires_grad)
    ctc_crf.WARP_CTC_LOSS()(y, lab, lx, ly)
    assert fake_core == [("ctc_loss_fwd", True)]


def test_grad_mode_switched_back_on_inside_no_grad(fake_core):
    """torch.enable_grad() inside no_grad turns the gradient back on: the training entry again."""
    import ctc_crf
    y, lab, lx, ly = _args()
    with torch.no_grad(), torch.enable_grad():
        ctc_crf.CTC_CRF_LOSS()(y, lab, lx, ly)
    assert [c[0] for c in fake_core] == ["ctc_crf_loss_fwd"]


def test_forward_only_symbols_declared():
    """The new entries are part of the C ABI the library declares and the loader binds."""
    from cat_b200 import _lib
    for s in ("ccb_den_fwd_alpha_floats", "ccb_num_fwd_only_bytes", "ccb_ctc_crf_loss_fwd_only", "ccb_ctc_loss_fwd_only"):
        assert s in _lib.SYMBOLS
        assert hasattr(_lib.lib(), s)
