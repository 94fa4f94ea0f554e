"""CPU: the restatements of the transducer beam search (tests/rnnt_decode_oracle.py) against exhaustive enumeration and each
other, the argument checks of ``cat_b200.rnnt_decode`` (raised before any native call) and the workspace size."""
import numpy as np
import pytest
import torch

from cat_b200 import _lib, rnnt_decode
from cat_b200.rnnt_decode import RNNTDecoder, rnnt_beam_search
from rnnt_decode_oracle import (CatJoiner, JointNet, LogAdd, LSTMPredictor, beam_ref, cat_decode, exhaustive,
                                module_lp)


def _prefix_rows(V, seed, scale=1.0):
    """lp(t, prefix): a log-softmax row drawn from a generator seeded by (seed, t, prefix)"""
    def lp(t, p):
        h = hash((seed, t) + tuple(p)) & 0xffffffff
        z = np.random.default_rng(h).standard_normal(V) * scale
        return z - np.logaddexp.reduce(z)
    return lp


@pytest.mark.parametrize("T", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("seed", [0, 1])
def test_beam_ref_without_pruning_is_exhaustive(T, seed):
    V = 3
    lp = _prefix_rows(V, seed, 2.0)
    ex = exhaustive(T, V, lp)
    got = beam_ref(T, V, 10 ** 6, lp)
    assert len(got) == len(ex)
    for p, s in got:
        assert abs(s - ex[p]) <= 1e-12 * (1 + abs(s)), (p, s, ex[p])
    assert [s for _, s in got] == sorted((s for _, s in got), reverse=True)


def test_beam_ref_ties_go_to_the_lower_flat_index():
    # every row uniform: all candidates tie, so the B kept are flat indices 0..B-1 of the beam
    V, B = 4, 3
    got = beam_ref(2, V, B, lambda t, p: np.full(V, -np.log(V)))
    # frame 0 keeps (), (1,), (2,); frame 1 keeps flat 0..2: () stays, (1,), (2,) extend the empty prefix
    assert [p for p, _ in got] == [(), (1,), (2,)]


def _modules(kind, V=5, H=6, seed=0):
    torch.manual_seed(seed)
    pred = LSTMPredictor(V, H if kind != "logadd" else V).double()
    if kind == "logadd":
        return pred, LogAdd(), V
    if kind == "jointnet":
        return pred, JointNet(H, H, V, 7).double(), H
    return pred, CatJoiner(H, H, V).double(), H


@pytest.mark.parametrize("kind", ["jointnet", "logadd", "cat"])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_cat_restatement_matches_beam_ref(kind, B):
    pred, joiner, He = _modules(kind)
    for p in pred.parameters():
        p.data.mul_(3.0)
    torch.manual_seed(1)
    enc = torch.randn(2, 5, He, dtype=torch.float64) * 2
    lens = torch.tensor([5, 3])
    got = cat_decode(enc, lens, pred, joiner, B)
    for n in range(2):
        lp = module_lp(lambda t: enc[n, t].reshape(1, 1, -1), pred, joiner)
        ref = beam_ref(int(lens[n]), 5, B, lp)
        assert got[n][0] == [list(p) for p, _ in ref]
        for s, (_, r) in zip(got[n][1], ref):
            assert abs(s - r) <= 1e-12 * (1 + abs(r))


class _NoNative:
    """Stands in for the native library: any call fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"native call {name} reached")


@pytest.fixture
def no_native(monkeypatch):
    monkeypatch.setattr(rnnt_decode._lib, "lib", lambda: _NoNative())


@pytest.mark.parametrize("kwargs, match", [
    (dict(lm_module=object(), alpha=0.5), "LM"),
    (dict(est_ilm=True, ilm_weight=0.3), "ILM"),
    (dict(eos_id=7), "eos"),
    (dict(bos_id=1), "bos_id"),
])
def test_decoder_refuses_unsupported_features(kwargs, match, no_native):
    with pytest.raises(NotImplementedError, match=match):
        RNNTDecoder(None, None, **kwargs)


def test_decoder_keeps_cats_rules(no_native):
    d = RNNTDecoder(None, None, lm_module=object(), alpha=0.0, beta=1.0, est_ilm=True, ilm_weight=0.0, eos_id=0,
                    beam_size=4, nbest=9)
    assert d.nbest == 4 and d.eos_id == -1
    assert RNNTDecoder(None, None, beam_size=3).nbest == 3
    for bad in (0, 129, 2.0, True):
        with pytest.raises(ValueError):
            RNNTDecoder(None, None, beam_size=bad)


def test_search_argument_errors_before_native(no_native):
    enc = torch.zeros(2, 3, 4)   # on the CPU: refused before anything else
    with pytest.raises(ValueError, match="CUDA"):
        rnnt_beam_search(enc, torch.tensor([3, 3]), None, None)
    if not torch.cuda.is_available():
        return
    enc = enc.cuda()
    lens = torch.tensor([3, 2])
    for kw, match in ((dict(beam_size=0), "beam_size"), (dict(beam_size=129), "beam_size"),
                      (dict(beam_size=4, nbest=5), "nbest"), (dict(blank=-1), "blank")):
        with pytest.raises(ValueError, match=match):
            rnnt_beam_search(enc, lens, None, None, **kw)
    for bad in (torch.tensor([3, 4]), torch.tensor([-1, 2]), torch.tensor([3]), torch.tensor([3.0, 2.0])):
        with pytest.raises(ValueError, match="frame_lens"):
            rnnt_beam_search(enc, bad, None, None)


def test_unsupported_predictor_state_raises_before_native(no_native):
    if not torch.cuda.is_available():
        pytest.skip("the state check runs after the argument checks, which need a CUDA enc_out")

    class Weird(torch.nn.Module):
        def forward(self, x, state=None):
            return torch.zeros(x.shape[0], 1, 4, device=x.device), [torch.zeros(1)]

    with pytest.raises(NotImplementedError, match="Weird"):
        rnnt_beam_search(torch.zeros(1, 2, 4, device="cuda"), torch.tensor([2]), Weird(), LogAdd())


def test_ws_bytes_bounds():
    L = _lib.lib()
    for N, T, B in ((1, 0, 1), (2, 5, 1), (3, 120, 16), (64, 120, 128)):
        assert L.ccb_rnnt_beam_ws_bytes(N, T, B) > 0
    # the trie: parent and token of 1 + B T nodes, a hash of the next power of two >= 2 (1 + B T) slots, one counter
    cap = 1 + 16 * 120
    h = 1 << (2 * cap - 1).bit_length()
    assert L.ccb_rnnt_beam_ws_bytes(3, 120, 16) == 3 * ((4 * (2 * cap + h + 1) + 255) // 256 * 256)
    for N, T, B in ((0, 5, 4), (2, -1, 4), (2, 5, 0), (2, 5, 129)):
        assert L.ccb_rnnt_beam_ws_bytes(N, T, B) == 0
    assert L.ccb_rnnt_beam_init(2, 5, 129, None, None, None, None, None, None) != 0
    assert "beam" in _lib.last_error()
