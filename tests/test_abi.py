"""CPU: the C-ABI library loads and exports every symbol include/*.h declares; the Python surface mirrors the
reference's names and error behaviour.  No compute calls (no GPU here)."""
import ctypes as C
import os
import re

import pytest
import torch

from conftest import ROOT


def _declared_symbols():
    txt = open(os.path.join(ROOT, "include", "ctc_crf_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    funcs = set(re.findall(r"\b([A-Za-z_][A-Za-z0-9_]*)\s*\([^;{]*\)\s*;", txt))
    funcs -= {"defined"}
    globs = set(re.findall(r"extern\s+int\s+([A-Za-z_][A-Za-z0-9_]*)\s*;", txt))
    return funcs, globs


def test_exports_match_header():
    from cat_b200 import _lib
    funcs, globs = _declared_symbols()
    assert {"Init", "Release", "compute_alpha", "compute_beta_and_grad", "compute_ctc_loss", "get_workspace_size",
            "ccb_ctc_crf_loss_fwd"} <= funcs
    assert globs == {"DEN_NUM_ARCS", "DEN_NUM_STATES"}
    L = _lib.lib()
    for s in sorted(funcs | globs):
        assert hasattr(L, s), f"{s} declared in include/ctc_crf_b200.h but not exported"
    assert set(_lib.SYMBOLS) == funcs and set(_lib.GLOBALS) == globs


def test_status_strings_and_workspace_query():
    from cat_b200 import _lib
    L = _lib.lib()
    assert L.ctcGetStatusString(0) == b"no error"
    assert b"invalid" in L.ctcGetStatusString(2)
    ll = (C.c_int * 2)(3, 5)
    il = (C.c_int * 2)(10, 20)
    n = C.c_size_t(0)
    assert L.get_workspace_size(ll, il, 7, 2, _lib.ctcOptions(None, 0), C.byref(n)) == 0
    assert n.value >= 2 * 20 * 11 * 4
    assert L.get_workspace_size(None, il, 7, 2, _lib.ctcOptions(None, 0), C.byref(n)) == 2   # INVALID_VALUE
    assert L.ccb_launch_count() == 0


def test_ctc_workspace_holds_cells_and_loglikelihoods():
    """ccb_ctc_workspace_bytes: per utterance the alpha and beta cells [T][2L+1] in double + the fp64 log-likelihood, then
    32 doubles of slack, then N floats -- where the fused loss keeps log p(l|x) (api.cu LossFwdImpl places them at double
    offset N * per_utt + 32: the numerator's output lives in the numerator's workspace, not in the den aux block)."""
    from cat_b200 import _lib
    L = _lib.lib()
    L.ccb_ctc_workspace_bytes.restype = C.c_size_t
    for N, T, maxl in [(1, 1, 0), (3, 7, 2), (64, 1500, 250), (17, 33, 5)]:
        per_utt = 2 * T * (2 * maxl + 1) + 1
        logp_off = (N * per_utt + 32) * 8
        assert int(L.ccb_ctc_workspace_bytes(N, T, maxl)) >= logp_off + 4 * N


def test_python_surface_mirrors_reference(tmp_path):
    import ctc_crf
    for name in ("CTC_CRF_LOSS", "WARP_CTC_LOSS", "CRFContext", "__version__", "_C"):
        assert hasattr(ctc_crf, name)
    for fn in ("gpu_den", "gpu_ctc", "init_env", "release_env", "ctc_crf_loss_fwd"):
        assert hasattr(ctc_crf._C, fn)
    crit = ctc_crf.CTC_CRF_LOSS()
    assert crit.lamb == 0.1 and crit.size_average is True
    with pytest.raises(RuntimeError, match="Denominator LM model location is invalid"):
        ctc_crf.CRFContext(str(tmp_path / "nope.fst"), gpus=0)
    f = tmp_path / "x.fst"
    f.write_bytes(b"")
    with pytest.raises(RuntimeError, match="invalid GPU ids"):      # no GPU in this container
        ctc_crf.CRFContext(str(f), gpus=[0] if torch.cuda.device_count() == 0 else [torch.cuda.device_count()])
    # dtype contract of CTC_CRF_LOSS.forward (ctc_crf/__init__.py:115-124)
    lab = torch.tensor([1], dtype=torch.int32)
    with pytest.raises(AssertionError):
        crit(torch.zeros(1, 2, 3, dtype=torch.float64), lab, lab, lab)
    with pytest.raises(AssertionError):
        crit(torch.zeros(1, 2, 3), lab.long(), lab, lab)
    with pytest.raises(AssertionError):
        crit(torch.zeros(1, 2, 3), lab.reshape(1, 1), lab, lab)


def test_no_cpu_fallback():
    """The product path must fail loudly without a GPU / without the extension, never route to a CPU path."""
    import ctc_crf
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lab = torch.tensor([1], dtype=torch.int32)
    with pytest.raises((AssertionError, RuntimeError)):
        ctc_crf.CTC_CRF_LOSS()(torch.zeros(1, 2, 3).log_softmax(-1), lab, torch.tensor([2], dtype=torch.int32), lab)
    src = open(os.path.join(ROOT, "cat_b200", "loss.py")).read() + open(os.path.join(ROOT, "cat_b200", "_C.py")).read()
    assert "oracle" not in src


def test_scratch_budget_is_cached_and_refreshed(monkeypatch):
    """Host logic of the batch slicer: the device-memory query is reused for a few calls, refreshed when a request does
    not fit the cached figure, and counts what the caching allocator holds but is not using."""
    import torch
    from cat_b200 import _C
    calls = []
    state = {"free": 100 << 20, "reserved": 30 << 20, "allocated": 10 << 20}
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev=None: (calls.append(1), (state["free"], 1 << 40))[1])
    monkeypatch.setattr(torch.cuda, "memory_reserved", lambda dev=None: state["reserved"])
    monkeypatch.setattr(torch.cuda, "memory_allocated", lambda dev=None: state["allocated"])
    _C._budget_cache.clear()
    dev = torch.device("cuda", 0)
    b0 = _C._scratch_budget(dev)
    assert b0 == int((120 << 20) * _C._WS_FRACTION) and len(calls) == 1
    for _ in range(5):
        assert _C._scratch_budget(dev) == b0
    assert len(calls) == 1                                   # served from the cache
    state["free"] = 500 << 20
    assert _C._scratch_budget(dev, need=b0 + 1) > b0         # a request that does not fit forces a fresh query
    assert len(calls) == 2
    for _ in range(40):
        _C._scratch_budget(dev)
    assert len(calls) >= 4                                   # and it expires on its own after a few calls
    _C._budget_cache.clear()
