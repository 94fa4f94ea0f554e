"""CPU side of the posterior sampler (``ctc_crf.crf_sample``): argument checks, the seed, ``samples_to_labels``, the plan's
in-arc CSR, and a numpy restatement of the sampler (Philox4x32-10 uniforms, alpha in fp64) that tests/test_gpu_sample.py
compares the kernel against path by path."""
import ctypes as C

import numpy as np
import pytest
import torch

from cat_b200 import _C, _lib, fst, plan

# ---------------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------------
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Philox4x32-10 of counters ctr (4 arrays of uint32 values, broadcast together) under key (k0, k1): 4 uint64 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) & np.uint64(_MASK) for c in ctr)
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = np.uint64(key[0] & _MASK), np.uint64(key[1] & _MASK)
    for _ in range(10):
        p0 = np.uint64(_M0) * c0
        p1 = np.uint64(_M1) * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(_MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(_MASK)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + np.uint64(_W0)) & np.uint64(_MASK)
        k1 = (k1 + np.uint64(_W1)) & np.uint64(_MASK)
    return c0, c1, c2, c3


def uniforms(seed, frame, sample, utt):
    """The kernel's uniform for the state of `frame` of `sample` of utterance `utt` (arrays broadcast): 53 bits in [0, 1)."""
    x0, x1, _, _ = philox4x32_10((frame, sample, utt, 0), (seed & _MASK, seed >> 32))
    return ((x0 >> np.uint64(5)).astype(np.float64) * 67108864.0 + (x1 >> np.uint64(6)).astype(np.float64)) / 9007199254740992.0


def plan_csr(path, n_ctas=132, n_warps=16):
    """The sampler's view of a den plan: in-arc CSR, labels, final weights, start (the numbering of a plan cut for n_ctas)."""
    L = _lib.lib()
    h = L.ccb_plan_create(path.encode(), n_ctas, n_warps)
    assert h, _lib.last_error()
    try:
        info = (C.c_long * 13)()
        assert L.ccb_plan_info(h, info) == 0
        S, start = int(info[2]), int(info[5])

        def get(which, dtype, count):
            a = np.empty(count, dtype=dtype)
            assert L.ccb_plan_copy(h, which, a.ctypes.data_as(C.c_void_p), a.nbytes) == 0
            return a
        in_off = get(19, np.int32, S + 1)
        A = int(in_off[-1])
        return dict(S=S, start=start, in_off=in_off, in_src=get(20, np.int32, A), in_w=get(21, np.float32, A),
                    state_label=get(0, np.int32, S), final_lin=get(1, np.float32, S), orig_state=get(2, np.int32, S))
    finally:
        L.ccb_plan_destroy(h)


def _pick(weights, target, band):
    """Inverse CDF: the first index whose running sum exceeds target; and whether a running sum lies within band of it."""
    cum = np.cumsum(weights)
    i = int(np.searchsorted(cum, target, side="right"))
    i = min(i, len(cum) - 1)
    while weights[i] <= 0:            # (the kernel's rule: only arcs with weight are drawn)
        i -= 1
    return i, int(np.any(np.abs(cum - target) < band))


def sample_ref(P, y, lens, K, seed, n_base=0, band=1e-5):
    """The sampler restated: alpha in fp64 (normalised per frame), the kernel's uniforms and inverse-CDF rule.
    Returns (tokens (N,K,T), lengths (N,K), align (N,K,T), path_logp (N,K) fp64, near (N,K) int: the draws of the path that
    lay within band * total of a CDF boundary, where fp32 alpha on the GPU may pick the neighbour)."""
    from scipy import sparse
    y = np.asarray(y, np.float64)
    N, T, V = y.shape
    S, off, src, w, lab = P["S"], P["in_off"], P["in_src"], P["in_w"].astype(np.float64), P["state_label"]
    fin = P["final_lin"].astype(np.float64)
    A = sparse.csr_matrix((w, src, off.astype(np.int64)), shape=(S, S))   # A[q, p] = w_pq: alpha_t = e_t * (A @ alpha_{t-1})
    tokens = np.full((N, K, T), -1, np.int32)
    align = np.full((N, K, T), -1, np.int32)
    lengths = np.full((N, K), -1, np.int32)
    logp = np.full((N, K), -np.inf)
    near = np.zeros((N, K), np.int64)
    for n in range(N):
        ln = int(lens[n])
        if ln <= 0:
            continue
        a = np.zeros((ln + 1, S))
        a[0, P["start"]] = 1.0
        logs = 0.0
        with np.errstate(invalid="ignore", over="ignore"):
            for t in range(1, ln + 1):
                e = np.exp(y[n, t - 1, lab])
                nxt = (A @ a[t - 1]) * e
                s = nxt.sum()
                if not (s > 0 and np.isfinite(s)):
                    a[t:] = 0
                    break
                a[t] = nxt / s
                logs += np.log(s)
        f = fin * a[ln]
        total = f.sum()
        if not (total > 0 and np.isfinite(total)):
            continue
        logz = np.log(total) + logs
        u_fin = uniforms(seed, ln, np.arange(K), n_base + n)
        u_walk = uniforms(seed, np.arange(ln)[:, None], np.arange(K)[None, :], n_base + n)   # [frame][sample]
        for k in range(K):
            q, nr = _pick(f, u_fin[k] * total, band * total)
            score = np.log(fin[q])
            labs = np.empty(ln, np.int32)
            for t in range(ln, 0, -1):
                labs[t - 1] = lab[q]
                score += y[n, t - 1, lab[q]]
                arcs = slice(off[q], off[q + 1])
                v = w[arcs] * a[t - 1, src[arcs]]
                tot = v.sum()
                i, nr2 = _pick(v, u_walk[t - 1, k] * tot, band * tot)
                nr += nr2
                score += np.log(w[off[q] + i])
                q = int(src[off[q] + i])
            assert q == P["start"]
            toks = [int(l) for j, l in enumerate(labs) if l != 0 and (j == 0 or labs[j - 1] != l)]
            align[n, k, :ln] = labs
            tokens[n, k, :len(toks)] = toks
            lengths[n, k] = len(toks)
            logp[n, k] = score - logz
            near[n, k] = nr
    return tokens, lengths, align, logp, near


# ---------------------------------------------------------------------------------------------------------------------
# Philox and the seed
# ---------------------------------------------------------------------------------------------------------------------
def test_philox_known_answers():
    """The Random123 known-answer vectors of Philox4x32-10."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((_MASK,) * 4, (_MASK, _MASK), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        got = tuple(int(x) for x in philox4x32_10(ctr, key))
        assert got == want, [hex(x) for x in got]


def test_uniforms_lie_in_unit_interval_and_differ_by_counter():
    u = uniforms(0x0123456789ABCDEF, np.arange(200)[:, None], np.arange(50)[None, :], 7)
    assert u.shape == (200, 50) and u.min() >= 0.0 and u.max() < 1.0
    assert len(np.unique(u)) == u.size
    assert abs(u.mean() - 0.5) < 0.01
    assert not np.array_equal(uniforms(1, 3, 4, 5), uniforms(1, 3, 4, 6))


def test_seed_is_drawn_from_the_generator_reproducibly():
    g = torch.Generator().manual_seed(1234)
    a, b = _C.draw_seed(g), _C.draw_seed(g)
    g.manual_seed(1234)
    assert _C.draw_seed(g) == a and a != b
    assert 0 <= a < (1 << 64)
    torch.manual_seed(99)
    c = _C.draw_seed()
    torch.manual_seed(99)
    assert _C.draw_seed(None) == c
    with pytest.raises(RuntimeError, match="CPU torch.Generator"):
        _C.draw_seed(object())


# ---------------------------------------------------------------------------------------------------------------------
# arguments (checked before anything touches a device)
# ---------------------------------------------------------------------------------------------------------------------
class _FakeCuda(torch.Tensor):
    pass


def test_argument_checks(monkeypatch):
    # the checks run on shapes and CPU tensors; a CPU stand-in that claims to be on the GPU reaches every one of them
    def fake(shape, dtype=torch.float32):
        t = torch.zeros(shape, dtype=dtype)
        return t.as_subclass(_FakeCuda)
    monkeypatch.setattr(_FakeCuda, "is_cuda", property(lambda self: True))
    y = fake((2, 5, 4))
    lx = torch.tensor([5, 3], dtype=torch.int32)
    assert _C._check_sample_args(y, lx, 3) == (2, 5, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C._check_sample_args(torch.zeros(2, 5, 4), lx, 1)
    with pytest.raises(RuntimeError, match="dtype"):
        _C._check_sample_args(fake((2, 5, 4), torch.float64), lx, 1)
    with pytest.raises(RuntimeError, match=r"\(N,T,V\)"):
        _C._check_sample_args(fake((2, 5)), lx, 1)
    with pytest.raises(RuntimeError, match="empty"):
        _C._check_sample_args(fake((0, 5, 4)), lx[:0], 1)
    with pytest.raises(RuntimeError, match="int32 CPU"):
        _C._check_sample_args(y, lx.long(), 1)
    with pytest.raises(RuntimeError, match="int32 CPU"):
        _C._check_sample_args(y, lx[:1], 1)
    with pytest.raises(RuntimeError, match=r"\[0, T\]"):
        _C._check_sample_args(y, torch.tensor([6, 1], dtype=torch.int32), 1)
    with pytest.raises(RuntimeError, match=r"\[0, T\]"):
        _C._check_sample_args(y, torch.tensor([-1, 1], dtype=torch.int32), 1)
    for bad in (0, -2, 1.5, True, None):
        with pytest.raises(RuntimeError, match="num_samples"):
            _C._check_sample_args(y, lx, bad)


# ---------------------------------------------------------------------------------------------------------------------
# samples_to_labels
# ---------------------------------------------------------------------------------------------------------------------
def test_samples_to_labels_by_hand():
    tokens = torch.full((2, 3, 5), -1, dtype=torch.int32)
    lengths = torch.tensor([[2, -1, 0], [3, 1, -1]], dtype=torch.int32)
    tokens[0, 0, :2] = torch.tensor([4, 2])
    tokens[1, 0, :3] = torch.tensor([1, 1, 3])
    tokens[1, 1, :1] = torch.tensor([7])
    labels, ly, utt = _C.samples_to_labels(tokens, lengths)
    assert labels.tolist() == [4, 2, 1, 1, 3, 7]
    assert ly.tolist() == [2, 0, 3, 1]
    assert utt.tolist() == [0, 0, 1, 1]
    assert labels.dtype == ly.dtype == utt.dtype == torch.int32
    assert not labels.is_cuda and not ly.is_cuda and not utt.is_cuda
    labels, ly, utt = _C.samples_to_labels(tokens[:, 1:2], lengths[:, 1:2])   # only infeasible samples but one
    assert labels.tolist() == [7] and ly.tolist() == [1] and utt.tolist() == [1]
    with pytest.raises(RuntimeError, match="tokens must be"):
        _C.samples_to_labels(tokens, lengths[:, :2])


# ---------------------------------------------------------------------------------------------------------------------
# the plan's in-arc CSR
# ---------------------------------------------------------------------------------------------------------------------
def _check_csr(path, g, n_ctas, n_warps):
    P = plan_csr(path, n_ctas, n_warps)
    S, off, src, w = P["S"], P["in_off"], P["in_src"], P["in_w"]
    assert off[0] == 0 and np.all(np.diff(off) >= 0) and src.min() >= 0 and src.max() < S
    dst = np.repeat(np.arange(S), np.diff(off))
    # every arc of the split graph once: a file arc p -> q with label l is an arc from every copy of p into the copy of q
    # that carries label l (the loader's in-label split)
    orig, lab = P["orig_state"], P["state_label"]
    copies = {}
    for s in range(S):
        copies.setdefault(int(orig[s]), []).append(s)
    src_f, dst_f, lab_f, lw = g.log_arcs()
    want = []
    for p, q, l, x in zip(src_f, dst_f, lab_f, lw):
        qs = [s for s in copies[int(q)] if lab[s] == l]
        assert len(qs) == 1
        for ps in copies[int(p)]:
            want.append((ps, qs[0], np.float32(np.exp(np.float32(x)))))
    got = sorted(zip(src.tolist(), dst.tolist(), w.tolist()))
    want = sorted((a, b, float(c)) for a, b, c in want)
    assert len(got) == len(want) == int(off[-1])
    assert [(a, b) for a, b, _ in got] == [(a, b) for a, b, _ in want]
    np.testing.assert_allclose([c for _, _, c in got], [c for _, _, c in want], rtol=1e-6, atol=0)
    # labels of every arc's destination: the arc's label
    assert np.all(lab[dst] >= 0)
    return P


@pytest.mark.parametrize("n_ctas,n_warps", [(132, 16), (4, 2)])
def test_in_arc_csr_lists_every_split_arc_once(tmp_graphs, fixture_fst, n_ctas, n_warps):
    for name in ("tlm_small", "random_split"):
        path, g, _ = tmp_graphs[name]
        _check_csr(path, g, n_ctas, n_warps)
    _check_csr(fixture_fst, fst.read_fst(fixture_fst), n_ctas, n_warps)


def test_in_arc_csr_unchanged_by_hub_rows(tmp_graphs, monkeypatch):
    """Hub rows are a kernel layout; the CSR is the plain graph whatever the hub threshold."""
    path, g, _ = tmp_graphs["tlm_small"]
    a = plan_csr(path)
    monkeypatch.setenv("CCB_HUB_IN_ARCS", "10")
    monkeypatch.setenv("CCB_PART_ARCS", "7")
    assert plan.load_plan(path).hub_states.size > 0
    b = _check_csr(path, g, 132, 16)
    assert a["in_off"][-1] == b["in_off"][-1]


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against exhaustive enumeration (so that the GPU comparison rests on a checked reference)
# ---------------------------------------------------------------------------------------------------------------------
def test_restatement_draws_the_path_posterior(tmp_path):
    """On a tiny T o LM graph, the restatement's path frequencies match exp(path_logp), and path_logp is a distribution's
    log-probability: every frame-label path's exact posterior from enumeration."""
    lm = fst.make_random_lm(H=2, V=3, d=2, seed=4)
    g = fst.compose_ctc_lm(lm)
    p = str(tmp_path / "tiny.fst")
    fst.write_fst(p, g)
    P = plan_csr(p)
    rng = np.random.default_rng(0)
    T = 3
    x = rng.standard_normal((1, T, 3))
    y = (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)
    K = 4000
    tokens, lengths, align, logp, near = sample_ref(P, y, [T], K, seed=77)
    assert (lengths >= 0).all()
    rows = {tuple(r) for r in align[0].tolist()}
    probs = {}
    for k in range(K):
        probs.setdefault(tuple(align[0, k].tolist()), []).append(logp[0, k])
    # the same frame labels can come from several paths only through different states; here each label row is one path
    for key, lps in probs.items():
        assert np.ptp(lps) < 1e-9
    expect = np.array([np.exp(v[0]) for v in probs.values()])
    count = np.array([len(v) for v in probs.values()])
    assert expect.sum() <= 1 + 1e-9
    assert np.all(np.abs(count / K - expect) < 5 * np.sqrt(expect * (1 - expect) / K) + 1e-3)
    assert len(rows) > 3
