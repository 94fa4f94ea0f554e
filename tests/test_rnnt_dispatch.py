"""CPU: the fp64 RNN-T restatement (oracle/rnnt.py) against torchaudio's rnnt_loss in both input modes, and the argument
checks of rnnt_loss / gather.sum, which fail before anything reaches a device."""
import numpy as np
import pytest
import torch

from oracle import rnnt as R


def _case(rng, N, Tm, Um, V, full=True):
    lx = rng.integers(1, Tm + 1, N).astype(np.int32)
    ly = rng.integers(0, Um + 1, N).astype(np.int32)
    if full:                    # T and U at the padded extent
        lx[0], ly[-1] = Tm, Um
    x = (rng.standard_normal((N, Tm, Um + 1, V)) * 2).astype(np.float32)
    y = rng.integers(1, V, (N, Um)).astype(np.int32)
    return x, y, lx, ly


CASES = [(1, 1, 0, 3), (2, 1, 3, 4), (3, 5, 0, 5), (4, 6, 4, 7), (3, 7, 5, 2), (5, 4, 3, 9), (2, 12, 6, 16)]


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_oracle_matches_torchaudio(fused, case):
    F = pytest.importorskip("torchaudio").functional
    rng = np.random.default_rng(100 + case)
    x, y, lx, ly = _case(rng, *CASES[case])
    inp = torch.tensor(x) if fused else torch.tensor(x).log_softmax(-1)
    inp = inp.detach().requires_grad_()
    c = F.rnnt_loss(inp, torch.tensor(y), torch.tensor(lx), torch.tensor(ly), blank=0, reduction="none",
                    fused_log_softmax=fused)
    c.sum().backward()
    oc, og = R.rnnt_loss(inp.detach().numpy(), y, lx, ly, blank=0, compact=False, from_logits=fused)
    assert np.all(np.abs(oc - c.detach().numpy().astype(np.float64)) <= 1e-6 * np.abs(oc))
    # torchaudio runs in fp32 only (it refuses fp64): its lattice and posteriors carry fp32 rounding, up to ~1e-5 on
    # posteriors near 1 at these sizes, so the gradient is held to 3e-5 rather than to the restatement's own accuracy
    assert np.abs(og - inp.grad.numpy()).max() < 3e-5


def test_oracle_compact_equals_padded_and_blank():
    rng = np.random.default_rng(7)
    x, y, lx, ly = _case(rng, 4, 6, 4, 7)
    rows = np.concatenate([x[n, :lx[n], :ly[n] + 1].reshape(-1, 7) for n in range(4)])
    labels = np.concatenate([y[n, :ly[n]] for n in range(4)])
    for fl in (False, True):
        pc, pg = R.rnnt_loss(x, y, lx, ly, from_logits=fl)
        cc, cg = R.rnnt_loss(rows, labels, lx, ly, compact=True, from_logits=fl)
        assert np.array_equal(pc, cc)
        assert np.array_equal(np.concatenate([pg[n, :lx[n], :ly[n] + 1].reshape(-1, 7) for n in range(4)]), cg)
    # beta gives the same log P; another blank id is a relabelling of the vocabulary
    lp = torch.tensor(x).log_softmax(-1).numpy().astype(np.float64)
    for n in range(4):
        T, U = lx[n], ly[n]
        lpb = lp[n, :T, :U + 1, 0]
        lpl = np.take_along_axis(lp[n, :T, :U], np.broadcast_to(y[n, :U][None, :, None], (T, U, 1)), -1)[..., 0]
        a, b, pb, pl = R.lattice(lpb, lpl)
        assert abs(a - b) < 1e-9 * abs(a)
        assert np.allclose((pb + np.pad(pl, ((0, 0), (0, 1)))).sum(), T + U)   # every path takes T + U transitions
    perm = np.roll(np.arange(7), -3)        # token k of the new vocabulary is token perm[k] of the old; blank 0 -> 4
    c0, _ = R.rnnt_loss(x, y, lx, ly, blank=0, from_logits=True)
    c4, _ = R.rnnt_loss(x[..., perm], np.argsort(perm)[y], lx, ly, blank=4, from_logits=True)
    assert np.allclose(c0, c4, rtol=1e-12)


# ---------------------------------------------------------------------------------------------------
# argument checks (no device needed: every one fails before a launch)
# ---------------------------------------------------------------------------------------------------
def _compact_args(V=5):
    lx = torch.tensor([3, 2], dtype=torch.int32)
    ly = torch.tensor([2, 0], dtype=torch.int32)
    x = torch.zeros(3 * 3 + 2 * 1, V)
    y = torch.tensor([1, 2], dtype=torch.int32)
    return x, y, lx, ly


def test_rnnt_dtype_asserts():
    from warp_rnnt import rnnt_loss
    x, y, lx, ly = _compact_args()
    with pytest.raises(AssertionError):
        rnnt_loss(x.double(), y, lx, ly, compact=True)
    with pytest.raises(AssertionError):
        rnnt_loss(x, y.long(), lx, ly, compact=True)
    with pytest.raises(AssertionError):
        rnnt_loss(x, y, lx.long(), ly, compact=True)
    with pytest.raises(AssertionError):
        rnnt_loss(x, y, lx, ly.long(), compact=True)


def test_rnnt_option_checks():
    from warp_rnnt import rnnt_loss
    x, y, lx, ly = _compact_args()
    for red in ("avg", None, "batchmean"):
        with pytest.raises(ValueError, match="reduction"):
            rnnt_loss(x, y, lx, ly, reduction=red, compact=True)
    for blank in (-1, 5, 1.0, True):
        with pytest.raises(ValueError, match="blank"):
            rnnt_loss(x, y, lx, ly, blank=blank, compact=True)
    for kw in ("fastemit_lambda", "average_frames", "gather"):     # options CAT never passes are not accepted
        with pytest.raises(TypeError):
            rnnt_loss(x, y, lx, ly, compact=True, **{kw: 0})


def test_rnnt_host_length_checks():
    from warp_rnnt import rnnt_loss
    x, y, lx, ly = _compact_args()
    with pytest.raises(ValueError, match="rows"):
        rnnt_loss(x[:-1], y, lx, ly, compact=True)
    with pytest.raises(ValueError, match="label lengths sum"):
        rnnt_loss(x, y[:1], lx, ly, compact=True)
    with pytest.raises(ValueError, match=">= 1"):
        rnnt_loss(x, y, torch.tensor([3, 0], dtype=torch.int32), ly, compact=True)
    with pytest.raises(ValueError, match="differ from blank"):
        rnnt_loss(x, torch.tensor([1, 0], dtype=torch.int32), lx, ly, compact=True)
    with pytest.raises(ValueError, match="differ from blank"):
        rnnt_loss(x, torch.tensor([1, 5], dtype=torch.int32), lx, ly, compact=True)
    with pytest.raises(ValueError, match=r"\(N,\)"):
        rnnt_loss(x, y, lx, ly[:1], compact=True)
    # padded layout: shapes and overruns
    xp = torch.zeros(2, 3, 3, 5)
    yp = torch.tensor([[1, 2], [3, 4]], dtype=torch.int32)
    with pytest.raises(ValueError, match="overrun"):
        rnnt_loss(xp, yp, torch.tensor([4, 2], dtype=torch.int32), ly)
    with pytest.raises(ValueError, match="overrun"):
        rnnt_loss(xp, yp, lx, torch.tensor([3, 0], dtype=torch.int32))
    with pytest.raises(ValueError, match=r"\(N, Umax\)"):
        rnnt_loss(xp, yp[:, :1], lx, ly)
    with pytest.raises(ValueError, match="Tmax, Umax"):
        rnnt_loss(xp[0], yp, lx, ly)
    # padding labels past U_n are not checked; valid arguments on the CPU stop at the device check
    yp[1, :] = 0
    with pytest.raises(ValueError, match="CUDA"):
        rnnt_loss(xp, yp, lx, ly)
    with pytest.raises(ValueError, match="CUDA"):
        rnnt_loss(x, y, lx, ly, compact=True)


def test_gather_checks_and_cat():
    import gather
    a, b = torch.zeros(5, 4), torch.zeros(3, 4)
    la, lb = torch.tensor([2, 3]), torch.tensor([1, 2])
    with pytest.raises(ValueError, match="dtype|share"):
        gather.sum(a.double(), b.double(), la, lb)
    with pytest.raises(ValueError, match="same H"):
        gather.sum(a, torch.zeros(3, 5), la, lb)
    with pytest.raises(ValueError, match=r"\(N,\)"):
        gather.sum(a, b, la, lb[:1])
    with pytest.raises(ValueError, match="CUDA"):
        gather.sum(a, b, la, lb)
    x = torch.arange(2 * 4 * 3).reshape(2, 4, 3)
    assert torch.equal(gather.cat(x, torch.tensor([2, 4])), torch.cat([x[0, :2], x[1, :4]]))
    yy = torch.tensor([[1, 2, 0], [3, 0, 0]])
    assert torch.equal(gather.cat(yy, torch.tensor([2, 1])), torch.tensor([1, 2, 3]))
