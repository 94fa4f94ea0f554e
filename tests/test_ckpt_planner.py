"""The slice planner's choice between the full alpha spill, halving and the checkpointed denominator (CPU only: a fake
library object whose size functions follow the library's formulas, and a fake memory budget)."""
import math

import pytest
import torch

from cat_b200 import _C


class FakeLib:
    """Size functions of a den graph with S states: full spill (T+3) frames, checkpointed (ceil(T/K) + max(K+1, 4) + 2)
    frames, of S x PadLanes(N) floats each.  small_ok = False: every batch is padded to at least 32 lanes."""

    def __init__(self, S, small_ok=False):
        self.S, self.small_ok = S, small_ok

    def pad(self, n):
        if self.small_ok and n <= 16:
            return 16
        g = (n + 31) // 32
        return (g + 3) // 4 * 4 * 32 if g >= 3 else g * 32

    def ccb_den_alpha_floats(self, n, t):
        return (t + 3) * self.S * self.pad(n)

    def ccb_den_ckpt_alpha_floats(self, n, t, k):
        k = min(k, t)
        return (-(-t // k) + max(k + 1, 4) + 2) * self.S * self.pad(n) + 2 * self.pad(n)

    def ccb_den_aux_bytes(self, n, t):
        return 3 * (t + 2) * self.pad(n) * 4

    def ccb_ctc_workspace_bytes(self, n, t, maxl):
        return n * (2 * t * (2 * maxl + 1) + 1) * 8


def _plan(monkeypatch, L, lens, budget):
    monkeypatch.setattr(_C, "_scratch_budget", lambda dev, need=0: budget)
    lx = torch.tensor(lens, dtype=torch.int32)
    ly = torch.clamp(lx // 6, max=400)
    return _C._plan_slices(L, lx, ly, len(lens), 218, None)


def _need(L, n, t, maxl, k=0):
    alpha = L.ccb_den_ckpt_alpha_floats(n, t, k) if k else L.ccb_den_alpha_floats(n, t)
    return alpha * 4 + L.ccb_den_aux_bytes(n, t) + L.ccb_ctc_workspace_bytes(n, t, maxl)


def test_full_spill_when_it_fits(monkeypatch):
    L = FakeLib(40000)
    slices = _plan(monkeypatch, L, [1500] * 64, 1 << 50)
    assert slices == [(0, 64, 1500, 250, 0)]


def test_halving_above_ckpt_width(monkeypatch):
    """64 utterances (64 lanes) with room for the full spill of 32 lanes: two full-spill halves, not one checkpointed call."""
    monkeypatch.setattr(_C, "CKPT_WIDTH", 32)
    L = FakeLib(40000)
    budget = _need(L, 32, 1500, 250) + 4096
    slices = _plan(monkeypatch, L, [1500] * 64, budget)
    assert slices == [(0, 32, 1500, 250, 0), (32, 64, 1500, 250, 0)]


def test_checkpoint_at_or_below_ckpt_width(monkeypatch):
    """A slice of CKPT_WIDTH utterances whose full spill does not fit runs checkpointed with K = ceil(sqrt(tmax))."""
    monkeypatch.setattr(_C, "CKPT_WIDTH", 32)
    L = FakeLib(40000)
    k = math.ceil(math.sqrt(1500))
    assert _C.ckpt_interval(1500) == k
    budget = _need(L, 32, 1500, 250, k) + 4096
    assert budget < _need(L, 32, 1500, 250)
    slices = _plan(monkeypatch, L, [1500] * 32, budget)
    assert slices == [(0, 32, 1500, 250, k)]


def test_checkpoint_at_once_when_halving_keeps_the_padding(monkeypatch):
    """Config 4's graph (no small-batch rows): 32 utterances and 16 both take 32 lanes, so halving saves no alpha memory --
    the slice runs checkpointed at once, even with CKPT_WIDTH below its width."""
    monkeypatch.setattr(_C, "CKPT_WIDTH", 8)
    L = FakeLib(199999)
    k = _C.ckpt_interval(2000)
    budget = _need(L, 32, 2000, 333, k) + 4096
    slices = _plan(monkeypatch, L, [2000] * 32, budget)
    assert slices == [(0, 32, 2000, 333, k)]


def test_checkpoint_then_halving_until_it_fits(monkeypatch):
    """Checkpointed but still too large: halved further, each half checkpointed."""
    monkeypatch.setattr(_C, "CKPT_WIDTH", 32)
    L = FakeLib(199999)
    k = _C.ckpt_interval(3000)
    budget = _need(L, 8, 3000, 400, k) + 4096
    slices = _plan(monkeypatch, L, [3000] * 16, budget)
    assert [(s[0], s[1], s[4]) for s in slices] == [(0, 8, k), (8, 16, k)]


def test_raise_only_when_one_checkpointed_utterance_does_not_fit(monkeypatch):
    L = FakeLib(199999)
    k = _C.ckpt_interval(3000)
    fits = _need(L, 1, 3000, 400, k)
    assert _plan(monkeypatch, L, [3000], fits) == [(0, 1, 3000, 400, k)]
    with pytest.raises(RuntimeError) as e:
        _plan(monkeypatch, L, [3000], fits - 1)
    msg = str(e.value)
    assert f"{_need(L, 1, 3000, 400) >> 20} MiB" in msg and f"{fits >> 20} MiB" in msg


def test_ckpt_alpha_is_bounded():
    """The checkpointed alpha of config 4's graph at one utterance of 3000 frames is a few GB, not 77."""
    L = FakeLib(199999)
    full = L.ccb_den_alpha_floats(1, 3000) * 4
    ck = L.ccb_den_ckpt_alpha_floats(1, 3000, _C.ckpt_interval(3000)) * 4
    assert full > 76e9 and ck < 3e9
