"""CPU: the RNN-T workspace layout that tests/test_gpu_rnnt_precision.py reads the kernels' stage outputs from, and the
allocation fact its poisoned-allocator tests rest on.

a. `rnnt_layout` restates `MakeRnntLayout` (cat_b200/csrc/rnnt_kernels.cu): blocks meta (one 40-byte `RnntMeta` per
   utterance), tail (the first compact row behind the last utterance, int64), logp (log P from alpha for n < N, from beta
   at N + n, fp64), alpha and beta (fp64 per row), lpb, lpl and lse (fp32 per row), each aligned to 256 bytes.  Its total
   must be what the library asks for.
b. `cat_b200/rnnt.py` creates its device buffers through `torch.empty` on the module global and in no other spelling, so
   that `ScratchProxy` sees every one of them.
"""
import ast
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT
from test_scratch_proxy import FACTORIES, LIKE, NEW, _kw

# struct RnntMeta: roff, loff, span (int64), then T, U, ts, bad (int32)
META_DTYPE = np.dtype([("roff", "<i8"), ("loff", "<i8"), ("span", "<i8"), ("T", "<i4"), ("U", "<i4"), ("ts", "<i4"),
                       ("bad", "<i4")])
BLOCKS = (("meta", None), ("tail", None), ("logp", np.float64), ("alpha", np.float64), ("beta", np.float64),
          ("lpb", np.float32), ("lpl", np.float32), ("lse", np.float32))


def _align256(b):
    return (b + 255) // 256 * 256


def rnnt_layout(N, rows):
    """{block: (byte offset, element count, numpy dtype)} of the workspace of an N-utterance, rows-row call, and its total
    byte count."""
    sizes = {"meta": (N, META_DTYPE), "tail": (1, np.dtype("<i8")), "logp": (2 * N, np.dtype(np.float64))}
    for name, dt in BLOCKS[3:]:
        sizes[name] = (rows, np.dtype(dt))
    out, o = {}, 0
    for name, _ in BLOCKS:
        count, dt = sizes[name]
        out[name] = (o, count, dt)
        o += 256 if name == "tail" else _align256(count * dt.itemsize)
    return out, o


def read_workspace(raw, N, rows):
    """The blocks of a workspace given as a uint8 numpy array (copied from the device): {block: numpy array}."""
    lay, total = rnnt_layout(N, rows)
    assert raw.dtype == np.uint8 and raw.size == total, (raw.size, total)
    return {name: raw[o:o + count * dt.itemsize].view(dt) for name, (o, count, dt) in lay.items()}


def _ws_bytes(N, rows):
    from cat_b200 import _lib
    L = _lib.lib()
    return int(L.ccb_rnnt_workspace_bytes(N, rows))


def test_meta_is_40_bytes():
    assert META_DTYPE.itemsize == 40


@pytest.mark.parametrize("N", [1, 2, 5, 6, 7, 31, 32, 255, 256, 257, 300, 512, 4097])
def test_layout_total_matches_library(N):
    for rows in (0, 1, 2, 7, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1000, 12345, 600_000, 3_000_000_017):
        lay, total = rnnt_layout(N, rows)
        assert total == _ws_bytes(N, rows), (N, rows)
        offs = [lay[name][0] for name, _ in BLOCKS]
        assert offs == sorted(offs) and all(o % 256 == 0 for o in offs)
        # 28 bytes per row plus the per-utterance blocks and at most 255 bytes of padding per block
        assert 28 * rows + 40 * N + 8 + 16 * N <= total <= 28 * rows + 56 * N + 256 + 8 * 255


def test_library_size_query_edges():
    from cat_b200 import _lib
    L = _lib.lib()
    assert L.ccb_rnnt_workspace_bytes.restype is C.c_size_t
    assert _ws_bytes(0, 10) == 0 and _ws_bytes(-1, 10) == 0 and _ws_bytes(3, -1) == 0


def test_read_workspace_views():
    N, rows = 3, 17
    _, total = rnnt_layout(N, rows)
    ws = read_workspace(np.zeros(total, np.uint8), N, rows)
    assert ws["meta"].shape == (N,) and ws["logp"].shape == (2 * N,) and ws["tail"].shape == (1,)
    for name in ("alpha", "beta", "lpb", "lpl", "lse"):
        assert ws[name].shape == (rows,)
    with pytest.raises(AssertionError):
        read_workspace(np.zeros(total - 1, np.uint8), N, rows)


RNNT_PY = os.path.join(ROOT, "cat_b200", "rnnt.py")


def test_rnnt_py_allocates_through_torch_empty_only():
    """The same check tests/test_scratch_proxy.py makes for _C.py: every `.empty` is `torch.empty` on the module global, no
    `*_like` / `new_*` allocation, no tensor factory with a device."""
    with open(RNNT_PY) as f:
        tree = ast.parse(f.read(), RNNT_PY)
    bad, empties = [], []
    for node in ast.walk(tree):
        if isinstance(node, ast.ImportFrom) and node.module and node.module.split(".")[0] == "torch" \
                and any(a.name not in ("Function",) for a in node.names):
            bad.append(f"{RNNT_PY}:{node.lineno}: `from torch import ...` hides allocations from the proxy")
        if isinstance(node, ast.Import):
            for a in node.names:
                if a.name.split(".")[0] == "torch" and (a.asname or a.name) != "torch":
                    bad.append(f"{RNNT_PY}:{node.lineno}: torch imported under another name")
        if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute)):
            continue
        attr, on_torch = node.func.attr, isinstance(node.func.value, ast.Name) and node.func.value.id == "torch"
        where = f"{RNNT_PY}:{node.lineno}"
        if attr == "empty":
            if on_torch:
                empties.append(node)
            else:
                bad.append(f"{where}: .empty() not called on the module global `torch`")
        elif attr in LIKE or attr in NEW:
            bad.append(f"{where}: {attr}() allocates behind the proxy's back; use torch.empty(...)")
        elif on_torch and attr in FACTORIES and _kw(node) & {"device", "pin_memory"}:
            bad.append(f"{where}: torch.{attr}(..., device=/pin_memory=) as a library buffer; use torch.empty(...)")
    assert not bad, "\n".join(bad)
    # the loss's workspace, costs, beta costs and gradient; gather.sum's output, its two workspaces and two gradients
    assert len([n for n in empties if "device" in _kw(n)]) == 9
