"""CPU: how CTC_CRF_LOSS, WARP_CTC_LOSS and ctc_align pass `utt` (several label sequences per utterance) to the native
layer.  Without `utt` they call exactly what they called before; with it they reach the grouped entries; bad maps are refused
with a clear error; the host grouping round-trips an unsorted map.  The `_C` functions are replaced by fakes, so no GPU runs."""
import pytest
import torch


def _i32(v):
    return torch.tensor(v, dtype=torch.int32)


@pytest.fixture
def fake_core(monkeypatch):
    from cat_b200 import loss as loss_mod
    calls = []

    def scalar_or_costs(kw, m):
        return torch.arange(1.0, m + 1) if kw.get("reduction") == "none" else torch.full((1,), 1.0)

    def crf_fwd(logits, labels, lx, ly, lamb, size_average, **kw):
        calls.append(("ctc_crf_loss_fwd", (lamb, size_average), kw))
        return scalar_or_costs(kw, logits.shape[0]), torch.ones(logits.shape), None

    def crf_fwd_only(logits, labels, lx, ly, lamb, size_average, **kw):
        calls.append(("ctc_crf_loss_fwd_only", (lamb, size_average), kw))
        return scalar_or_costs(kw, logits.shape[0]), None

    def ctc_fwd(logits, labels, lx, ly, size_average, **kw):
        calls.append(("ctc_loss_fwd", (size_average,), kw))
        return scalar_or_costs(kw, logits.shape[0]), torch.ones(logits.shape), torch.zeros(logits.shape[0])

    def ctc_fwd_only(logits, labels, lx, ly, size_average, **kw):
        calls.append(("ctc_loss_fwd_only", (size_average,), kw))
        return scalar_or_costs(kw, logits.shape[0]), torch.zeros(logits.shape[0])

    def align(logits, labels, lx, ly, **kw):
        calls.append(("ctc_align", (), kw))
        return torch.zeros(logits.shape[:2], dtype=torch.int32), torch.zeros(logits.shape[0])

    def crf_seqs(logits, labels, lx, ly, utt, lamb, size_average, **kw):
        calls.append(("ctc_crf_loss_seqs", (lamb, size_average), kw))
        return scalar_or_costs(kw, utt.numel()), torch.ones(logits.shape), ("state" if kw.get("reduction") == "none" else None)

    def crf_seqs_fwd_only(logits, labels, lx, ly, utt, lamb, size_average, **kw):
        calls.append(("ctc_crf_loss_seqs_fwd_only", (lamb, size_average), kw))
        return scalar_or_costs(kw, utt.numel())

    def ctc_seqs(logits, labels, lx, ly, utt, size_average, **kw):
        calls.append(("ctc_loss_seqs", (size_average,), kw))
        none = kw.get("reduction") == "none"
        return scalar_or_costs(kw, utt.numel()), torch.ones(logits.shape), ("state" if none else None)

    def seqs_backward(state, w, dtype):
        calls.append(("seqs_backward", (state,), dict(dtype=dtype)))
        return torch.full((2, 5, 4), float(w.sum()), dtype=dtype)

    def rows_scale(grad, w, lx, dtype):
        calls.append(("grad_rows_scale", (), dict(dtype=dtype)))
        return (grad * w.reshape(-1, 1, 1)).to(dtype)

    def align_seqs(logits, labels, lx, ly, utt, **kw):
        calls.append(("ctc_align_seqs", (), kw))
        return torch.zeros((utt.numel(), logits.shape[1]), dtype=torch.int32), torch.zeros(utt.numel())

    for name, fn in [("ctc_crf_loss_fwd", crf_fwd), ("ctc_crf_loss_fwd_only", crf_fwd_only), ("ctc_loss_fwd", ctc_fwd),
                     ("ctc_loss_fwd_only", ctc_fwd_only), ("ctc_align", align), ("ctc_crf_loss_seqs", crf_seqs),
                     ("ctc_crf_loss_seqs_fwd_only", crf_seqs_fwd_only), ("ctc_loss_seqs", ctc_seqs),
                     ("seqs_backward", seqs_backward), ("ctc_align_seqs", align_seqs), ("grad_rows_scale", rows_scale)]:
        monkeypatch.setattr(loss_mod.core, name, fn)
    return calls


def _batch():
    # two utterances, three sequences: utterance 1 has two, utterance 0 one, handed over unsorted
    return torch.zeros(2, 5, 4), _i32([1, 2, 3, 1, 3]), _i32([5, 4]), _i32([2, 1, 2]), _i32([1, 0, 1])


def _all_calls(y, lab, lx, ly, utt=None):
    import ctc_crf
    kw = {} if utt is None else dict(utt=utt)
    for crit in (ctc_crf.CTC_CRF_LOSS(lamb=0.3), ctc_crf.CTC_CRF_LOSS(lamb=0.3, from_logits=True),
                 ctc_crf.CTC_CRF_LOSS(reduction="none", zero_infinity=True), ctc_crf.WARP_CTC_LOSS(),
                 ctc_crf.WARP_CTC_LOSS(reduction="none")):
        out = crit(y.clone().requires_grad_(True), lab, lx, ly, **kw)
        out.sum().backward()
        with torch.no_grad():
            crit(y, lab, lx, ly, **kw)
    ctc_crf.ctc_align(y, lab, lx, ly, **kw)


def test_utt_none_calls_what_it_called_before(fake_core):
    """utt=None (and no utt) reaches the per-utterance entries with the arguments they always had."""
    y, lab, lx, _, _ = _batch()
    ly = _i32([2, 1])
    lab = lab[:3]
    _all_calls(y, lab, lx, ly)
    without = list(fake_core)
    del fake_core[:]
    _all_calls(y, lab, lx, ly, utt=None)
    assert fake_core == without
    names = [c[0] for c in without]
    assert not any("seqs" in n for n in names)
    assert names == ["ctc_crf_loss_fwd", "ctc_crf_loss_fwd_only"] * 2 + \
        ["ctc_crf_loss_fwd", "grad_rows_scale", "ctc_crf_loss_fwd_only"] + \
        ["ctc_loss_fwd", "ctc_loss_fwd_only", "ctc_loss_fwd", "grad_rows_scale", "ctc_loss_fwd_only", "ctc_align"]
    assert without[0] == ("ctc_crf_loss_fwd", (0.3, True), {})
    assert without[2] == ("ctc_crf_loss_fwd", (0.3, True), dict(from_logits=True))


def test_utt_reaches_the_grouped_entries(fake_core):
    y, lab, lx, ly, utt = _batch()
    _all_calls(y, lab, lx, ly, utt=utt)
    names = [c[0] for c in fake_core]
    assert names == ["ctc_crf_loss_seqs", "ctc_crf_loss_seqs_fwd_only"] * 2 + \
        ["ctc_crf_loss_seqs", "seqs_backward", "ctc_crf_loss_seqs_fwd_only"] + \
        ["ctc_loss_seqs", "ctc_loss_seqs", "ctc_loss_seqs", "seqs_backward", "ctc_loss_seqs", "ctc_align_seqs"]
    assert fake_core[0] == ("ctc_crf_loss_seqs", (0.3, True),
                            dict(from_logits=False, reduction=None, zero_infinity=False))
    assert fake_core[4] == ("ctc_crf_loss_seqs", (0.1, True),
                            dict(from_logits=False, reduction="none", zero_infinity=True))
    assert fake_core[7][2] == dict(reduction=None, zero_infinity=False)
    assert fake_core[8][2] == dict(reduction=None, zero_infinity=False, with_grad=False)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_per_sequence_backward_gets_grad_output(fake_core, dtype):
    """reduction='none' with utt: the backward is seqs_backward(state, grad_output, logits dtype)."""
    import ctc_crf
    y, lab, lx, ly, utt = _batch()
    y = y.to(dtype).requires_grad_(True)
    costs = ctc_crf.CTC_CRF_LOSS(reduction="none")(y, lab, lx, ly, utt=utt)
    assert costs.shape == (3,)
    w = torch.tensor([0.5, -2.0, 4.0])
    (g,) = torch.autograd.grad(costs.mul(w).sum(), y)
    assert fake_core[-1] == ("seqs_backward", ("state",), dict(dtype=dtype))
    assert g.dtype == dtype and float(g[0, 0, 0]) == 2.5


def test_bad_utt_is_refused():
    import ctc_crf
    from cat_b200 import _C
    _, lab, _, ly, utt = _batch()
    with pytest.raises(AssertionError, match="torch.int"):
        ctc_crf.CTC_CRF_LOSS()(torch.zeros(2, 5, 4), lab, _i32([5, 4]), ly, utt=utt.long())
    with pytest.raises(RuntimeError, match="int32 CPU"):
        _C.group_seqs(utt.long(), lab, ly, 2)
    with pytest.raises(RuntimeError, match="int32 CPU"):
        _C.group_seqs([1, 0, 1], lab, ly, 2)
    with pytest.raises(RuntimeError, match="int32 CPU"):
        _C.group_seqs(utt.reshape(3, 1), lab, ly, 2)
    for bad in ([1, 0, 2], [-1, 0, 1]):
        with pytest.raises(RuntimeError, match=r"\[0, N\) = \[0, 2\)"):
            _C.group_seqs(_i32(bad), lab, ly, 2)
    with pytest.raises(RuntimeError, match="one entry per label sequence"):
        _C.group_seqs(_i32([1, 0]), lab, ly, 2)
    with pytest.raises(RuntimeError, match="sum to"):
        _C.group_seqs(utt, lab[:4], ly, 2)
    with pytest.raises(RuntimeError, match="no label sequence"):
        _C.group_seqs(_i32([]), lab[:0], _i32([]), 2)


def test_grouping_round_trips_an_unsorted_map():
    """Stable grouping by row: pos / row / labels / ly / off describe the caller's sequences, and pos un-permutes them."""
    from cat_b200 import _C
    g = torch.Generator().manual_seed(0)
    N, M = 7, 23
    utt = torch.randint(0, N - 1, (M,), generator=g, dtype=torch.int32)      # row N-1 gets no sequence
    ly = torch.randint(0, 5, (M,), generator=g, dtype=torch.int32)
    labels = torch.randint(1, 9, (int(ly.sum()),), generator=g, dtype=torch.int32)
    grp = _C.group_seqs(utt, labels, ly, N)
    assert grp.M == M
    assert sorted(grp.pos.tolist()) == list(range(M))
    assert torch.equal(grp.row, utt[grp.pos.long()])
    assert grp.row.tolist() == sorted(grp.row.tolist())
    for n in range(N):      # stable: the caller's order within a row
        mine = grp.pos[grp.off[n]:grp.off[n + 1]].tolist()
        assert mine == [m for m in range(M) if int(utt[m]) == n]
    assert grp.off[N - 1] == grp.off[N] == M
    off = [0] + torch.cumsum(ly.long(), 0).tolist()
    goff = [0] + torch.cumsum(grp.ly.long(), 0).tolist()
    for j in range(M):
        m = int(grp.pos[j])
        assert grp.ly[j] == ly[m]
        assert torch.equal(grp.labels[goff[j]:goff[j + 1]], labels[off[m]:off[m + 1]])
    # un-permuting: values computed in grouped order land at their caller's index
    vals = torch.arange(M, dtype=torch.float32) * 10
    back = torch.empty(M)
    back[grp.pos.long()] = vals
    assert torch.equal(back[grp.pos.long()], vals)


class _FakeL:
    """Scratch sizes in units: alpha n*t, aux n, numerator workspace m*t*(2*maxl+1)."""
    def ccb_den_alpha_floats(self, n, t): return n * t
    def ccb_den_ckpt_alpha_floats(self, n, t, k): return n * t
    def ccb_den_aux_bytes(self, n, t): return n
    def ccb_ctc_workspace_bytes(self, m, t, maxl): return m * t * (2 * maxl + 1)


def test_planner_sizes_the_numerator_by_sequences(monkeypatch):
    """Slices are cut by utterance; a slice's numerator workspace counts its sequences and their longest label sequence,
    its den scratch its utterances."""
    from cat_b200 import _C
    monkeypatch.setattr(_C, "_scratch_budget", lambda dev, need=0: 1 << 40)
    monkeypatch.setattr(_C, "MAX_UTTS_PER_CALL", 3)
    lx = _i32([10, 9, 8, 7, 6])
    counts = [2, 0, 3, 1, 1]
    off = torch.tensor([0] + torch.cumsum(torch.tensor(counts), 0).tolist())
    ly = _i32([1, 4, 2, 2, 7, 3, 9])        # grouped: row 0 -> [1, 4], row 2 -> [2, 2, 7], row 3 -> [3], row 4 -> [9]
    slices = _C._plan_slices(_FakeL(), lx, ly, 5, 11, None, seq_off=off)
    assert slices == [(0, 3, 10, 7, 0), (3, 5, 7, 9, 0)]
    assert _C._slice_need(_FakeL(), 3, 10, 7, 0, 5) == 4 * 30 + 3 + 5 * 10 * 15
    assert _C._slice_need(_FakeL(), 3, 10, 7, 0) == _C._slice_need(_FakeL(), 3, 10, 7, 0, 3)
    fwd = _C._plan_fwd_only_slices(type("L", (), {"ccb_den_fwd_alpha_floats": lambda s, n: n,
                                                  "ccb_den_aux_bytes": lambda s, n, t: n,
                                                  "ccb_num_fwd_only_bytes": lambda s, m: 4 * m})(),
                                   lx, ly, 5, None, seq_off=off)
    assert fwd == [(0, 3, 10, 7), (3, 5, 7, 9)]


def test_new_symbols_declared():
    from cat_b200 import _lib
    for s in ("ccb_ctc_crf_loss_seqs", "ccb_ctc_crf_loss_seqs_fwd_only", "ccb_ctc_loss_seqs", "ccb_seqs_grad",
              "ccb_ctc_align_seqs"):
        assert s in _lib.SYMBOLS
        assert hasattr(_lib.lib(), s)
