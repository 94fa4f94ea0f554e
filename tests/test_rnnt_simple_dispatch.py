"""CPU: the fp64 restatement of the LogAdd joiner's RNN-T loss (tests/rnnt_simple_oracle.py) against the RNN-T lattice on
an explicitly materialised joint and against torchaudio; the argument checks of ``warp_rnnt.rnnt_loss_simple``, which
fail before anything reaches a device; and the workspace size the library asks for."""
import numpy as np
import pytest
import torch

from oracle import rnnt as R
from rnnt_simple_oracle import batch, simple
from test_rnnt_workspace import rnnt_layout


def _case(rng, N, Tm, Um, V, scale=2.0):
    lx = rng.integers(1, Tm + 1, N).astype(np.int32)
    ly = rng.integers(0, Um + 1, N).astype(np.int32)
    lx[0], ly[-1] = Tm, Um
    f = (rng.standard_normal((N, Tm, V)) * scale).astype(np.float32)
    g = (rng.standard_normal((N, Um + 1, V)) * scale).astype(np.float32)
    y = rng.integers(1, V, (N, Um)).astype(np.int32)
    return f, g, y, lx, ly


CASES = [(1, 1, 0, 3), (2, 1, 3, 4), (3, 5, 0, 5), (4, 6, 4, 7), (3, 7, 5, 2), (5, 4, 3, 9), (2, 12, 6, 16)]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_simple_matches_materialised_joint(case):
    """The restatement equals oracle.rnnt.rnnt_loss on the fp64 joint f[t] + g[u] taken as raw logits, with the joint's
    gradient summed over u (for f) and over t (for g): the chain rule through the broadcast sum."""
    rng = np.random.default_rng(300 + case)
    f, g, y, lx, ly = _case(rng, *CASES[case])
    f64, g64 = f.astype(np.float64), g.astype(np.float64)
    joint = f64[:, :, None, :] + g64[:, None, :, :]
    jc, jg = R.rnnt_loss(joint, y, lx, ly, from_logits=True)
    c, gf, gg = batch(f, g, y, lx, ly)
    assert np.allclose(c, jc, rtol=1e-12, atol=0)
    assert np.allclose(gf, jg.sum(2), rtol=0, atol=1e-12)
    assert np.allclose(gg, jg.sum(1), rtol=0, atol=1e-12)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_simple_matches_torchaudio(case):
    """torchaudio's rnnt_loss on the fp32 joint, backpropagated through the broadcast sum by autograd.  torchaudio runs in
    fp32 only: its posteriors carry up to ~1e-5 of rounding (tests/test_rnnt_dispatch.py bounds its joint gradient by 3e-5),
    and the gradient on f or g sums up to max(T, U+1) = 12 such entries, so it is held to 3e-5 * 12."""
    F = pytest.importorskip("torchaudio").functional
    rng = np.random.default_rng(400 + case)
    f, g, y, lx, ly = _case(rng, *CASES[case])
    ft, gt = torch.tensor(f, requires_grad=True), torch.tensor(g, requires_grad=True)
    c = F.rnnt_loss(ft[:, :, None] + gt[:, None], torch.tensor(y), torch.tensor(lx), torch.tensor(ly), blank=0,
                    reduction="none", fused_log_softmax=True)
    c.sum().backward()
    oc, ogf, ogg = batch(f, g, y, lx, ly)
    assert np.all(np.abs(oc - c.detach().numpy().astype(np.float64)) <= 1e-6 * np.abs(oc))
    assert np.abs(ogf - ft.grad.numpy()).max() < 3.6e-4
    assert np.abs(ogg - gt.grad.numpy()).max() < 3.6e-4


def test_simple_blank_relabelling_and_minus_inf():
    """Another blank id is a relabelling of the vocabulary; -inf entries at tokens that are neither blank nor a label leave
    the cost finite and get zero gradient."""
    rng = np.random.default_rng(9)
    f, g, y, lx, ly = _case(rng, 3, 6, 4, 7)
    perm = np.roll(np.arange(7), -3)
    c0, gf0, gg0 = batch(f, g, y, lx, ly, blank=0)
    c4, gf4, gg4 = batch(f[..., perm], g[..., perm], np.argsort(perm)[y], lx, ly, blank=4)
    assert np.allclose(c0, c4, rtol=1e-12)
    assert np.allclose(gf0[..., perm], gf4, atol=1e-12) and np.allclose(gg0[..., perm], gg4, atol=1e-12)
    y[:] = 1
    f[:, :, 5] = -np.inf
    g[:, :, 6] = -np.inf
    c, gf, gg = batch(f, g, y, lx, ly)
    assert np.all(np.isfinite(c)) and np.all(gf[..., 5] == 0) and np.all(gg[..., 6] == 0)
    lp, df, dg = simple(f[0, :lx[0]], g[0, :ly[0] + 1], y[0, :ly[0]])
    assert np.isfinite(lp) and np.all(np.isfinite(df)) and np.all(np.isfinite(dg))


# ---------------------------------------------------------------------------------------------------
# argument checks (no device needed: every one fails before a launch)
# ---------------------------------------------------------------------------------------------------
def _args(V=5, dtype=torch.float32, idt=torch.int32):
    f = torch.zeros(2, 3, V, dtype=dtype)
    g = torch.zeros(2, 3, V, dtype=dtype)
    y = torch.tensor([[1, 2], [3, 0]], dtype=idt)
    lx = torch.tensor([3, 2], dtype=idt)
    ly = torch.tensor([2, 1], dtype=idt)
    return f, g, y, lx, ly


def test_simple_dtype_asserts():
    from warp_rnnt import rnnt_loss_simple
    f, g, y, lx, ly = _args()
    with pytest.raises(AssertionError):
        rnnt_loss_simple(f.double(), g.double(), y, lx, ly)
    with pytest.raises(AssertionError):
        rnnt_loss_simple(f, g.half(), y, lx, ly)
    with pytest.raises(AssertionError):
        rnnt_loss_simple(f.bfloat16(), g.half(), y, lx, ly)
    for i in range(3):
        ints = [y, lx, ly]
        ints[i] = ints[i].to(torch.int16)
        with pytest.raises(AssertionError):
            rnnt_loss_simple(f, g, *ints)
        ints[i] = ints[i].float()
        with pytest.raises(AssertionError):
            rnnt_loss_simple(f, g, *ints)


def test_simple_option_and_shape_checks():
    from warp_rnnt import rnnt_loss_simple
    f, g, y, lx, ly = _args()
    for red in ("avg", None, "batchmean"):
        with pytest.raises(ValueError, match="reduction"):
            rnnt_loss_simple(f, g, y, lx, ly, reduction=red)
    for blank in (-1, 5, 1.0, True):
        with pytest.raises(ValueError, match="blank"):
            rnnt_loss_simple(f, g, y, lx, ly, blank=blank)
    with pytest.raises(ValueError, match=r"\(N, Tmax, V\)"):
        rnnt_loss_simple(f[0], g, y, lx, ly)
    with pytest.raises(ValueError, match="share N"):
        rnnt_loss_simple(f, g[:1], y, lx, ly)
    with pytest.raises(ValueError, match="share N"):
        rnnt_loss_simple(f, g[..., :4], y, lx, ly)
    with pytest.raises(ValueError, match=r"\(N, Umax\)"):
        rnnt_loss_simple(f, g[:, :2], y, lx, ly)            # g_pred.shape[1] must be labels.shape[1] + 1
    with pytest.raises(ValueError, match=r"\(N,\)"):
        rnnt_loss_simple(f, g, y, lx, ly[:1])
    with pytest.raises(TypeError):
        rnnt_loss_simple(f, g, y, lx, ly, fastemit_lambda=0.0)


@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
def test_simple_host_length_and_label_checks(idt):
    from warp_rnnt import rnnt_loss_simple
    f, g, y, lx, ly = _args(idt=idt)
    with pytest.raises(ValueError, match="overrun"):
        rnnt_loss_simple(f, g, y, torch.tensor([4, 2], dtype=idt), ly)        # T_n > Tmax
    with pytest.raises(ValueError, match="overrun"):
        rnnt_loss_simple(f, g, y, lx, torch.tensor([3, 0], dtype=idt))        # U_n > Umax
    with pytest.raises(ValueError, match=">= 1"):
        rnnt_loss_simple(f, g, y, torch.tensor([3, 0], dtype=idt), ly)
    with pytest.raises(ValueError, match=">= 1"):
        rnnt_loss_simple(f, g, y, lx, torch.tensor([2, -1], dtype=idt))
    with pytest.raises(ValueError, match="differ from blank"):
        rnnt_loss_simple(f, g, torch.tensor([[1, 0], [3, 0]], dtype=idt), lx, ly)
    with pytest.raises(ValueError, match="differ from blank"):
        rnnt_loss_simple(f, g, torch.tensor([[1, 5], [3, 0]], dtype=idt), lx, ly)
    with pytest.raises(ValueError, match="differ from blank"):
        rnnt_loss_simple(f, g, torch.tensor([[1, 2], [-3, 0]], dtype=idt), lx, ly)
    with pytest.raises(ValueError, match="differ from blank"):
        rnnt_loss_simple(f, g, y, lx, ly, blank=2)
    if idt == torch.int64:
        with pytest.raises(ValueError, match="int32"):
            rnnt_loss_simple(f, g, y, torch.tensor([2 ** 32 + 3, 2]), ly)
        with pytest.raises(ValueError, match="int32"):
            rnnt_loss_simple(f, g, y, lx, torch.tensor([2 ** 31, 1]))
        with pytest.raises(ValueError, match="differ from blank"):     # would wrap to label 1 in int32
            rnnt_loss_simple(f, g, torch.tensor([[2 ** 32 + 1, 2], [3, 0]]), lx, ly)
    # padding labels past U_n are not checked; valid arguments on the CPU stop at the device check
    y[1, 1] = 0
    with pytest.raises(ValueError, match="CUDA"):
        rnnt_loss_simple(f, g, y, lx, ly)
    with pytest.raises(ValueError, match="CUDA"):
        rnnt_loss_simple(f.half(), g.half(), y.long(), lx.long(), ly.long(), reduction="none", blank=4)


def test_simple_checks_need_no_device(monkeypatch):
    """No argument check reaches the native library: with the loader broken, every bad call still raises its own error."""
    from cat_b200 import _lib
    from warp_rnnt import rnnt_loss_simple

    def no_lib():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "lib", no_lib)
    f, g, y, lx, ly = _args()
    with pytest.raises(ValueError, match="overrun"):
        rnnt_loss_simple(f, g, y, torch.tensor([4, 2], dtype=torch.int32), ly)
    with pytest.raises(ValueError, match="CUDA"):
        rnnt_loss_simple(f, g, y, lx, ly)


# ---------------------------------------------------------------------------------------------------
# workspace: the RNN-T loss's blocks over the N Tmax (Umax+1) padded cells, then row maxima and row flags of f and g
# (fp32 / int32) and the per-cell S, W, pb and pl (fp32), each aligned to 256 bytes
# ---------------------------------------------------------------------------------------------------
def _align256(b):
    return (b + 255) // 256 * 256


def simple_layout(N, Tmax, Umax):
    """{block: (byte offset, element count, numpy dtype)} of the workspace of rnnt_loss_simple, and its total."""
    cells = N * Tmax * (Umax + 1)
    out, o = rnnt_layout(N, cells)
    nf, ng = N * Tmax, N * (Umax + 1)
    for name, count, dt in (("mf", nf, np.float32), ("mg", ng, np.float32), ("ff", nf, np.int32), ("fg", ng, np.int32),
                            ("S", cells, np.float32), ("W", cells, np.float32), ("PB", cells, np.float32),
                            ("PL", cells, np.float32)):
        dt = np.dtype(dt)
        out[name] = (o, count, dt)
        o += _align256(count * dt.itemsize)
    return out, o


@pytest.mark.parametrize("N,Tmax,Umax", [(1, 1, 0), (1, 7, 3), (3, 5, 0), (5, 33, 17), (64, 150, 20), (32, 400, 120),
                                         (257, 61, 9)])
def test_simple_workspace_bytes(N, Tmax, Umax):
    from cat_b200 import _lib
    L = _lib.lib()
    lay, total = simple_layout(N, Tmax, Umax)
    assert int(L.ccb_rnnt_simple_workspace_bytes(N, Tmax, Umax)) == total
    offs = sorted(o for o, _, _ in lay.values())
    assert all(o % 256 == 0 for o in offs)
    cells = N * Tmax * (Umax + 1)
    # 44 bytes per cell, 8 per row of f and of g, 56 per utterance, and at most 255 bytes of padding per block
    base = 44 * cells + 8 * (N * Tmax + N * (Umax + 1)) + 56 * N
    assert base <= total <= base + 256 + 16 * 255


def test_simple_workspace_bytes_edges():
    import ctypes as C
    from cat_b200 import _lib
    L = _lib.lib()
    assert L.ccb_rnnt_simple_workspace_bytes.restype is C.c_size_t
    for args in ((0, 3, 2), (-1, 3, 2), (2, 0, 2), (2, 3, -1)):
        assert int(L.ccb_rnnt_simple_workspace_bytes(*args)) == 0
