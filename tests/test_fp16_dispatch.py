"""CPU: fp16 logits reach the native entries as they are.  CTC_CRF_LOSS and WARP_CTC_LOSS pass a torch.float16 tensor to
`_C.ctc_crf_loss_fwd` / `_C.ctc_crf_loss_fwd_only` / `_C.ctc_loss_fwd` / `_C.ctc_loss_fwd_only` without a cast, in both grad
modes, and the gradient comes back in fp16.  The `_C` functions are replaced by fakes, so no GPU runs."""
import os
import re

import pytest
import torch

from conftest import ROOT


@pytest.fixture
def fake_core(monkeypatch):
    from cat_b200 import loss as loss_mod
    calls = []

    def crf_fwd(logits, labels, lx, ly, lamb, size_average, want_parts=False, from_logits=False):
        calls.append(("ctc_crf_loss_fwd", logits.dtype, from_logits))
        return torch.full((1,), 1.0), torch.full(logits.shape, 0.5), None

    def crf_fwd_only(logits, labels, lx, ly, lamb, size_average, want_parts=False, from_logits=False):
        calls.append(("ctc_crf_loss_fwd_only", logits.dtype, from_logits))
        return torch.full((1,), 2.0), None

    def ctc_fwd(logits, labels, lx, ly, size_average, blank=0):
        calls.append(("ctc_loss_fwd", logits.dtype))
        return torch.full((1,), 3.0), torch.full(logits.shape, 0.25), torch.zeros(logits.shape[0])

    def ctc_fwd_only(logits, labels, lx, ly, size_average, blank=0):
        calls.append(("ctc_loss_fwd_only", logits.dtype))
        return torch.full((1,), 4.0), torch.zeros(logits.shape[0])

    monkeypatch.setattr(loss_mod.core, "ctc_crf_loss_fwd", crf_fwd)
    monkeypatch.setattr(loss_mod.core, "ctc_crf_loss_fwd_only", crf_fwd_only)
    monkeypatch.setattr(loss_mod.core, "ctc_loss_fwd", ctc_fwd)
    monkeypatch.setattr(loss_mod.core, "ctc_loss_fwd_only", ctc_fwd_only)
    return calls


def _args(dtype=torch.float16):
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)
    return torch.zeros(2, 5, 4, dtype=dtype), i32([1, 2, 3]), i32([5, 4]), i32([2, 1])


@pytest.mark.parametrize("from_logits", [False, True])
def test_crf_loss_passes_fp16_unconverted(fake_core, from_logits):
    import ctc_crf
    crit = ctc_crf.CTC_CRF_LOSS(lamb=0.1, from_logits=from_logits)
    y, lab, lx, ly = _args()
    y.requires_grad_(True)
    loss = crit(y, lab, lx, ly)
    (loss * 2.0).backward()
    with torch.no_grad():
        crit(y, lab, lx, ly)
    assert fake_core == [("ctc_crf_loss_fwd", torch.float16, from_logits),
                         ("ctc_crf_loss_fwd_only", torch.float16, from_logits)]
    # the fp32 gradient of the native entry comes back in the input's dtype: cast by _CTC_CRF_LOGITS.backward on the raw
    # entry, by autograd on the log-prob entry
    assert y.grad.dtype == torch.float16
    assert torch.equal(y.grad, torch.full(y.shape, 1.0, dtype=torch.float16))


def test_ctc_loss_passes_fp16_unconverted(fake_core):
    import ctc_crf
    y, lab, lx, ly = _args()
    y.requires_grad_(True)
    warp = ctc_crf.WARP_CTC_LOSS()
    warp(y, lab, lx, ly).backward()
    with torch.inference_mode():
        warp(y, lab, lx, ly)
    assert fake_core == [("ctc_loss_fwd", torch.float16), ("ctc_loss_fwd_only", torch.float16)]
    assert y.grad.dtype == torch.float16


def test_crf_loss_still_refuses_float64(fake_core):
    import ctc_crf
    y, lab, lx, ly = _args(torch.float64)
    for from_logits in (False, True):
        with pytest.raises(AssertionError, match="torch.float16"):
            ctc_crf.CTC_CRF_LOSS(from_logits=from_logits)(y, lab, lx, ly)
    assert fake_core == []


def test_dtype_codes_match_the_header():
    """_C._DTYPES maps each accepted torch dtype to the CCB_DTYPE_* code the C header defines for it."""
    from cat_b200 import _C
    header = open(os.path.join(ROOT, "include", "ctc_crf_b200.h")).read()
    codes = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define CCB_DTYPE_(\w+) (\d+)", header)}
    assert codes == {"F32": 0, "BF16": 1, "F16": 2}
    assert _C._DTYPES == {torch.float32: codes["F32"], torch.bfloat16: codes["BF16"], torch.float16: codes["F16"]}


def test_native_batch_check_accepts_fp16_and_refuses_float64():
    from cat_b200 import _C
    """The native wrappers' own dtype check (on a CPU tensor that reports itself as a CUDA one)."""
    y, lab, lx, ly = _args()

    class Cuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True

    assert _C._check_batch_args(y.as_subclass(Cuda), lab, lx, ly) == (2, 5, 4)
    with pytest.raises(RuntimeError, match="unsupported logits dtype"):
        _C._check_batch_args(y.double().as_subclass(Cuda), lab, lx, ly)
