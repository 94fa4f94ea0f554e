"""The allocation proxy of the scratch-contents tests, and the two host-side facts those tests rest on.

`ScratchProxy` stands in for the module global `torch` of `cat_b200/_C.py`: every buffer that module hands to the library
comes from `torch.empty`, and the proxy fills the raw bytes of each with a chosen pattern, so a word the library reads
before it writes it holds junk (NaN, 3.39e38, -1, 2139062143) instead of the zeros of fresh device memory.  Checked here, on
the CPU:

a. the proxy fills every byte, for every dtype and shape `_C.py` asks for, and is `torch` otherwise;
b. `_C.py` creates its device buffers through `torch.empty` on the module global and in no other spelling, so that none
   escapes the proxy (tests/test_gpu_scratch_contents.py then checks the sizes the proxy saw against the library's);
c. the pinned staging ring waits for slot i exactly when it reuses it, never earlier, and keeps one buffer per slot.
"""
import ast
import os

import pytest
import torch

from conftest import ROOT


class ScratchProxy:
    """`torch`, except that `empty` fills the raw bytes of its result with `byte` (on the current stream for a CUDA tensor)
    and notes (bytes, dtype, device) in `record`."""

    def __init__(self, byte=0):
        self.byte = byte
        self.record = []

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *args, **kwargs):
        t = torch.empty(*args, **kwargs)
        if t.numel():
            t.reshape(-1).view(torch.uint8).fill_(self.byte)
        self.record.append((t.numel() * t.element_size(), t.dtype, t.device))
        return t


# ---------------------------------------------------------------------------------------------------------------------
# a. the proxy
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("byte", [0x00, 0x7F, 0xFF])
@pytest.mark.parametrize("shape", [(), (0,), (7,), (3, 5, 2), (2, 0, 4)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.int32, torch.uint8])
def test_empty_fills_every_byte(dtype, shape, byte):
    proxy = ScratchProxy(byte)
    t = proxy.empty(shape, dtype=dtype)
    assert t.dtype == dtype and tuple(t.shape) == shape and t.is_contiguous()
    raw = t.reshape(-1).view(torch.uint8)
    assert raw.numel() == t.numel() * t.element_size() and bool((raw == byte).all())
    assert proxy.record == [(raw.numel(), dtype, torch.device("cpu"))]


def test_patterns_are_the_values_the_tests_rely_on():
    """0xFF: NaN in the three float types, -1 as int32.  0x7F: finite and huge as fp32 (an add overflows), a large int32."""
    ff, sf = ScratchProxy(0xFF), ScratchProxy(0x7F)
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        assert bool(torch.isnan(ff.empty(4, dtype=dt)).all())
    assert ff.empty(4, dtype=torch.int32).tolist() == [-1] * 4
    v = sf.empty(2, dtype=torch.float32)
    assert bool(torch.isfinite(v).all()) and float(v[0]) > 3.3e38 and bool(torch.isinf(v + v).all())
    assert sf.empty(1, dtype=torch.int32).item() == 2139062143


def test_everything_else_is_torch():
    proxy = ScratchProxy(0xFF)
    for name in ("cat", "zeros", "cumsum", "float32", "int32", "cuda", "Tensor", "device", "sort", "arange"):
        assert getattr(proxy, name) is getattr(torch, name)
    assert proxy.zeros(3).tolist() == [0.0] * 3 and proxy.record == []
    with pytest.raises(AttributeError):
        proxy.no_such_function


# ---------------------------------------------------------------------------------------------------------------------
# b. every device buffer of _C.py is a torch.empty on the module global
# ---------------------------------------------------------------------------------------------------------------------
C_PY = os.path.join(ROOT, "cat_b200", "_C.py")
FACTORIES = {"zeros", "ones", "full", "rand", "randn", "tensor", "empty_strided"}      # fine on the host, not as device scratch
LIKE = {"empty_like", "zeros_like", "ones_like", "full_like", "rand_like", "randn_like"}
NEW = {"new_empty", "new_zeros", "new_ones", "new_full", "new_tensor", "new_empty_strided"}


def _kw(call):
    return {k.arg for k in call.keywords}


def test_c_py_allocates_through_torch_empty_only():
    with open(C_PY) as f:
        tree = ast.parse(f.read(), C_PY)
    bad, empties = [], []
    for node in ast.walk(tree):
        if isinstance(node, ast.ImportFrom) and node.module and node.module.split(".")[0] == "torch":
            bad.append(f"{C_PY}:{node.lineno}: `from torch import ...` hides allocations from the proxy")
        if isinstance(node, ast.Import):
            for a in node.names:
                if a.name.split(".")[0] == "torch" and (a.asname or a.name) != "torch":
                    bad.append(f"{C_PY}:{node.lineno}: torch imported under another name")
        if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute)):
            continue
        attr, on_torch = node.func.attr, isinstance(node.func.value, ast.Name) and node.func.value.id == "torch"
        where = f"{C_PY}:{node.lineno}"
        if attr == "empty":
            if on_torch:
                empties.append(node)
            else:
                bad.append(f"{where}: .empty() not called on the module global `torch`")
        elif attr in LIKE or attr in NEW:
            bad.append(f"{where}: {attr}() allocates behind the proxy's back; use torch.empty(...)")
        elif on_torch and attr in FACTORIES and _kw(node) & {"device", "pin_memory"}:
            bad.append(f"{where}: torch.{attr}(..., device=/pin_memory=) as a library buffer; use torch.empty(...) and let "
                       f"the library initialise what it reads")
    assert not bad, "\n".join(bad)
    on_device = [n for n in empties if "device" in _kw(n)]
    assert len(on_device) >= 40, len(on_device)          # the workspaces and outputs of every entry
    assert any("pin_memory" in _kw(n) for n in empties)  # the staging ring


def test_loss_and_dist_allocate_nothing():
    """`loss.py` and `dist.py` hand the library no buffer of their own: no tensor factory is called in them."""
    for name in ("loss.py", "dist.py"):
        path = os.path.join(ROOT, "cat_b200", name)
        with open(path) as f:
            tree = ast.parse(f.read(), path)
        for node in ast.walk(tree):
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute):
                assert node.func.attr not in ({"empty"} | LIKE | NEW), f"{path}:{node.lineno}: {node.func.attr}()"


# ---------------------------------------------------------------------------------------------------------------------
# c. the staging ring's bookkeeping, CUDA stubbed out
# ---------------------------------------------------------------------------------------------------------------------
class _FakeEvent:
    def __init__(self, log, number):
        self.log, self.number = log, number

    def record(self, stream):
        self.log.append(("record", self.number))

    def synchronize(self):
        self.log.append(("sync", self.number))


class _FakeCuda:
    def __init__(self, log):
        self.log, self.events = log, 0

    def Event(self):
        self.events += 1
        return _FakeEvent(self.log, self.events)

    def current_stream(self, device=None):
        return None


class _HostTorch:
    """`torch` with events that only keep a log and staging buffers in ordinary host memory."""

    def __init__(self):
        self.log = []
        self.cuda = _FakeCuda(self.log)

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *args, pin_memory=False, **kwargs):
        return torch.empty(*args, **kwargs)


@pytest.mark.parametrize("calls", range(1, 10))
def test_ring_waits_for_a_slot_exactly_when_it_reuses_it(monkeypatch, calls):
    from cat_b200 import _C
    host = _HostTorch()
    monkeypatch.setattr(_C, "torch", host)
    ring = _C._PinnedRing()
    slots = len(ring.bufs)
    assert slots == 4
    recorded = []                       # the event of each stage call, in order
    for k in range(calls):
        before = len(host.log)
        part = torch.arange(k, k + 5 + k, dtype=torch.int32)
        out = ring.stage([part, part[:2]], "cpu")
        assert out.tolist() == part.tolist() + part[:2].tolist()
        new = host.log[before:]
        recorded.append(new[-1][1])
        assert new[-1][0] == "record"
        # the only wait is for the copy that used this slot `slots` calls ago; the first `slots` calls wait for nothing
        assert new[:-1] == ([("sync", recorded[k - slots])] if k >= slots else []), (k, new)
    assert len(set(recorded)) == calls


def test_ring_buffers_grow_and_are_not_shared(monkeypatch):
    from cat_b200 import _C
    host = _HostTorch()
    monkeypatch.setattr(_C, "torch", host)
    ring = _C._PinnedRing()
    small = torch.arange(10, dtype=torch.int32)
    for _ in range(4):
        ring.stage([small], "cpu")
    first = [b.data_ptr() for b in ring.bufs]
    assert len(set(first)) == 4 and all(b.numel() >= 10 for b in ring.bufs)
    big = torch.arange(5000, dtype=torch.int32)
    out = ring.stage([big], "cpu")                      # slot 0 again: too small, replaced by a larger buffer
    assert out.tolist() == big.tolist() and ring.bufs[0].numel() >= 5000
    assert [b.data_ptr() for b in ring.bufs[1:]] == first[1:] and all(b.numel() < 5000 for b in ring.bufs[1:])
    assert len({b.data_ptr() for b in ring.bufs}) == 4
    out = ring.stage([small], "cpu")                    # slot 1: a smaller request keeps its buffer
    assert out.tolist() == small.tolist() and ring.bufs[1].data_ptr() == first[1]
