"""CPU: the restatements of the CTC-T beam search (tests/ctct_decode_oracle.py) against the CTC-T loss's oracle, torch's CTC
loss and each other, the constructor rules and argument checks of ``cat_b200.ctct_decode`` (raised before any native call)
and the workspace size."""
import itertools

import numpy as np
import pytest
import torch

from cat_b200 import _lib, rnnt_decode
from cat_b200.ctct_decode import CTCTDecoder, ctct_beam_search
from ctct_decode_oracle import beam_ref, cat_decode
from ctct_oracle import utterance
from rnnt_decode_oracle import CatJoiner, JointNet, LogAdd, LSTMPredictor, module_lp


def _prefix_rows(V, seed, scale=1.0):
    """lp(t, prefix): a log-softmax row drawn from a generator seeded by (seed, t, prefix)"""
    def lp(t, p):
        h = hash((seed, t) + tuple(p)) & 0xffffffff
        z = np.random.default_rng(h).standard_normal(V) * scale
        return z - np.logaddexp.reduce(z)
    return lp


def _loss_logp(T, V, lp, y, blank):
    """log P(y) by the CTC-T loss's oracle on y's lattice: row (t, u) is lp(t, y[:u])"""
    rows = np.stack([np.stack([lp(t, tuple(y[:u])) for u in range(len(y) + 1)]) for t in range(T)])
    return utterance(rows, y, blank)[0]


@pytest.mark.parametrize("T, V", [(1, 3), (2, 3), (3, 4), (4, 3), (5, 3), (4, 4)])
@pytest.mark.parametrize("blank", [0, 2])
def test_beam_ref_without_pruning_is_the_ctct_loss(T, V, blank):
    lp = _prefix_rows(V, T * 10 + V + blank, 2.0)
    got = dict(beam_ref(T, V, 10 ** 6, lp, blank=blank))
    labels = [c for c in range(V) if c != blank]
    feasible = set()
    for U in range(T + 1):
        for y in itertools.product(labels, repeat=U):
            ref = _loss_logp(T, V, lp, list(y), blank)
            if ref > -np.inf:
                feasible.add(y)
                assert abs(got[y] - ref) <= 1e-12 * (1 + abs(ref)), (y, got.get(y), ref)
    assert set(got) == feasible
    assert abs(np.logaddexp.reduce(list(got.values()))) <= 1e-12
    assert list(got.values()) == sorted(got.values(), reverse=True)


@pytest.mark.parametrize("blank", [0, 3])
def test_beam_ref_on_prefix_independent_rows_is_ctc(blank):
    T, V = 5, 4
    x = (torch.randn(T, V, dtype=torch.float64, generator=torch.Generator().manual_seed(blank)) * 1.5).log_softmax(-1)
    got = beam_ref(T, V, 10 ** 6, lambda t, p: x[t].numpy(), blank=blank)
    for y, s in got:
        if not y:
            ref = float(x[:, blank].sum())
        else:
            ref = -float(torch.nn.functional.ctc_loss(x[:, None], torch.tensor([y]), torch.tensor([T]),
                                                      torch.tensor([len(y)]), blank=blank, reduction="none"))
        assert abs(s - ref) <= 1e-12 * (1 + abs(ref)), (y, s, ref)


def fold_rows(t, p):
    """Frame 0 keeps [(), (1,)] at beam 2.  At frame 1, () extends to (1,) (key 0) and (2,) (key 1) by equal values, and
    (1,) puts all its mass on (1, 2): its stay is -inf, so the target (1,) holds exactly ()'s extension's mass and ties
    (2,).  It ranks first by its key, the folded extension's 0, not its stay's 1*3+2 = 5."""
    if t == 0:
        return np.log([0.6, 0.3, 0.1])
    if p == ():
        return np.log([0.2, 0.4, 0.4])
    return np.array([-np.inf, -np.inf, 0.0])


def test_beam_ref_folds_an_extension_into_a_later_stay_with_its_key():
    assert [p for p, _ in beam_ref(1, 3, 2, fold_rows)] == [(), (1,)]
    got = beam_ref(2, 3, 2, fold_rows)
    assert [p for p, _ in got] == [(1, 2), (1,)]
    assert got[0][1] == np.log(0.3) and got[1][1] == np.log(0.6) + np.log(0.4)


def repeat_rows(t, p):
    """(1,) enters frame 2 with b / s = 0.7; there its row ranks the repeat 1 first (0.4), 2 (0.3) second and 3 (0.29)
    third, but by path score b lp[1] = 0.28 s < s lp[3].  Ranked by row value, the top-2 is {1, 2}: beam 2 keeps (1, 2) and
    (1, 1), where a ranking by path score would keep (1, 3) instead of (1, 1)."""
    if t == 0:
        return np.log([0.001, 0.997, 0.001, 0.001])
    if p != (1,):
        return np.log(np.full(4, 0.25))
    return np.log([0.7, 0.2998, 1e-4, 1e-4]) if t == 1 else np.log([0.01, 0.4, 0.3, 0.29])


def test_beam_ref_ranks_candidates_by_row_value():
    assert [p for p, _ in beam_ref(3, 4, 2, repeat_rows)] == [(1, 2), (1, 1)]


def test_beam_ref_ties_go_to_the_lower_token_and_key():
    # uniform rows: frame 0's extensions (1,), (2,) (keys 0, 1) tie and precede the stay () (key 3, k = 2), all at -log 3
    V = 4
    flat = lambda t, p: np.full(V, -np.log(V))   # noqa: E731
    assert [p for p, _ in beam_ref(1, V, 2, flat)] == [(1,), (2,)]
    assert [p for p, _ in beam_ref(1, V, 3, flat)] == [(1,), (2,), (3,)]
    assert [p for p, _ in beam_ref(1, V, 8, flat)] == [(1,), (2,), (3,), ()]


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
    (dict(bos_id=1), "bos_id"),
])
def test_decoder_refuses_unsupported_features(kwargs, match, no_native):
    with pytest.raises(NotImplementedError, match=match):
        CTCTDecoder(None, None, **kwargs)


def test_decoder_keeps_cats_rules(no_native):
    # CAT's decode.py passes the tokenizer's eos id; CTCTDecoder has no early stop and ignores it, and the ILM arguments
    d = CTCTDecoder(None, None, lm_module=object(), alpha=0.0, beta=1.0, est_ilm=True, ilm_weight=0.3, eos_id=7,
                    beam_size=4, nbest=9)
    assert d.nbest == 4 and d.eos_id == 7
    assert CTCTDecoder(None, None, beam_size=3).nbest == 3
    assert CTCTDecoder(None, None, blank_id=2, bos_id=2).blank_id == 2
    for bad in (0, 129, 2.0, True):
        with pytest.raises(ValueError):
            CTCTDecoder(None, None, beam_size=bad)


def test_search_argument_errors_before_native(no_native):
    enc = torch.zeros(2, 3, 4)   # on the CPU: refused before anything else
    with pytest.raises(ValueError, match="ctct_beam_search: .*CUDA"):
        ctct_beam_search(enc, torch.tensor([3, 3]), None, None)
    if not torch.cuda.is_available():
        return
    enc = enc.cuda()
    lens = torch.tensor([3, 2])
    for kw, match in ((dict(beam_size=0), "beam_size"), (dict(beam_size=129), "beam_size"),
                      (dict(beam_size=4, nbest=5), "nbest"), (dict(blank=-1), "blank")):
        with pytest.raises(ValueError, match="ctct_beam_search: " + match):
            ctct_beam_search(enc, lens, None, None, **kw)
    for bad in (torch.tensor([3, 4]), torch.tensor([-1, 2]), torch.tensor([3]), torch.tensor([3.0, 2.0])):
        with pytest.raises(ValueError, match="ctct_beam_search: frame_lens"):
            ctct_beam_search(enc, bad, None, None)


def test_unsupported_predictor_state_and_blank_raise_before_native(no_native):
    if not torch.cuda.is_available():
        pytest.skip("these checks run after the argument checks, which need a CUDA enc_out")

    class Weird(torch.nn.Module):
        def forward(self, x, state=None):
            return torch.zeros(x.shape[0], 1, 4, device=x.device), [torch.zeros(1)]

    with pytest.raises(NotImplementedError, match="ctct_beam_search: .*Weird"):
        ctct_beam_search(torch.zeros(1, 2, 4, device="cuda"), torch.tensor([2]), Weird(), LogAdd())

    class Plain(torch.nn.Module):
        def forward(self, x, state=None):
            return torch.zeros(x.shape[0], 1, 4, device=x.device), None

    with pytest.raises(ValueError, match="ctct_beam_search: blank = 4"):
        ctct_beam_search(torch.zeros(1, 2, 4, device="cuda"), torch.tensor([2]), Plain(), LogAdd(), blank=4)


def test_ws_bytes_bounds():
    L = _lib.lib()
    for N, T, B in ((1, 0, 1), (2, 5, 1), (3, 120, 16), (64, 120, 128)):
        assert L.ccb_ctct_beam_ws_bytes(N, T, B) > 0
    # the transducer search's tries first, then per utterance b and n of every slot and B x B candidate tokens, masses and
    # merges
    for N, T, B in ((3, 120, 16), (2, 7, 128), (1, 0, 1)):
        per_utt = (16 * B + 16 * B * B + 255) // 256 * 256
        assert L.ccb_ctct_beam_ws_bytes(N, T, B) == L.ccb_rnnt_beam_ws_bytes(N, T, B) + N * per_utt
    for N, T, B in ((0, 5, 4), (2, -1, 4), (2, 5, 0), (2, 5, 129)):
        assert L.ccb_ctct_beam_ws_bytes(N, T, B) == 0
    assert L.ccb_ctct_beam_init(2, 5, 129, None, None, None, None, None, None) != 0
    assert "ctct_beam_init" in _lib.last_error() and "beam" in _lib.last_error()
    assert L.ccb_ctct_beam_step(None, None, 0, 0, 2, 5, 4, 3, 0, None, 3, None, None, None, None, None, None) != 0
    assert "blank" in _lib.last_error()
