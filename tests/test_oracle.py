"""CPU: pin the fp64 oracle -- fixture known answers, torch's CTC as an independent numerator check,
the self-consistency invariants the reference computes but never compares (SURVEY.md 4), and the golden
vectors recorded from the reference's own CUDA code on the GPU box (tests/golden/ref_cuda_golden.npz)."""
import os

import numpy as np
import pytest
import torch

from cat_b200 import fst
from oracle import oracle

from conftest import GOLDEN


def test_fixture_known_answers(fixture_fst, fixture_inputs):
    fi = fixture_inputs
    g = fst.read_fst(fixture_fst)
    loss, grad, parts = oracle.ctc_crf(g, fi["y"], fi["labels"], fi["lx"], fi["ly"], fi["lamb"])
    assert abs(parts["logz_alpha"][0] - (-6.25832785)) < 1e-6
    assert abs(parts["logz_beta"][0] - (-6.25832785)) < 1e-6
    assert abs(parts["logp_ctc"][0] - (-3.74228025)) < 1e-6
    assert abs(loss - (-2.47862480)) < 1e-6
    np.testing.assert_allclose(grad[0, 0], [0.658503, 0.311666, -0.980169, 0, 0], atol=1e-6)
    np.testing.assert_allclose(grad[0, 4], [0.060326, 0, 0, 0, -0.070326], atol=1e-6)
    np.testing.assert_allclose(parts["gamma_den"].sum(-1), 1.0, atol=1e-12)
    np.testing.assert_allclose(parts["gamma_ctc"].sum(-1), 1.0, atol=1e-12)


@pytest.mark.parametrize("seed,N,T,V,lens,ly", [
    (0, 4, 100, 5, [100, 80, 55, 9], [8, 8, 3, 8]),          # BASELINE config 1 shape (yesno: N=4,T=100,V=5)
    (1, 3, 30, 12, [30, 11, 30], [10, 0, 29]),                # L = 0 and a nearly full lattice
    (2, 2, 7, 4, [7, 6], [4, 3]),
])
def test_ctc_matches_torch(seed, N, T, V, lens, ly):
    """log p = -nll; gamma_ctc = exp(y) - d nll / d y (torch folds the softmax Jacobian in)."""
    rng = np.random.default_rng(seed)
    y, _, lens, _ = oracle.synth_batch(N, T, V, seed=seed, lens=lens)
    ly = np.asarray(ly, np.int32)
    labels = rng.integers(1, V, size=int(ly.sum())).astype(np.int32)
    lp, gam = oracle.ctc(y, labels, ly, lens)
    yt = torch.tensor(y, dtype=torch.float64).transpose(0, 1).contiguous().requires_grad_(True)
    nll = torch.nn.functional.ctc_loss(yt, torch.tensor(labels, dtype=torch.long), torch.tensor(lens, dtype=torch.long),
                                       torch.tensor(ly, dtype=torch.long), reduction="none", zero_infinity=False)
    feasible = torch.isfinite(nll)
    nll[feasible].sum().backward()
    for n in range(N):
        if feasible[n]:
            assert abs(lp[n] + nll[n].item()) < 1e-9 * max(1, abs(lp[n]))
            ref = (torch.tensor(y[n], dtype=torch.float64).exp() - yt.grad[:, n]).numpy()[:lens[n]]
            np.testing.assert_allclose(gam[n, :lens[n]], ref, atol=1e-9)
        else:
            assert np.isinf(lp[n]) and lp[n] < 0
            assert not gam[n].any()


def test_ctc_repeats_and_infeasible():
    V = 6
    y, _, lens, _ = oracle.synth_batch(3, 6, V, seed=4, lens=[6, 6, 5])
    labels = np.array([2, 2, 3,   1, 1, 1, 1,   4, 4, 4], np.int32)    # repeats need blanks between them
    ly = np.array([3, 4, 3], np.int32)
    lp, gam = oracle.ctc(y, labels, ly, lens)
    assert np.isfinite(lp[0])                 # L + repeats = 4 <= 6
    assert np.isinf(lp[1]) and lp[1] < 0      # 4 + 3 = 7 > 6   (gpu_ctc_kernels.h:108-109)
    assert np.isfinite(lp[2])                 # 3 + 2 = 5 == 5: the start/end special case (:144)
    np.testing.assert_allclose(gam[2, :5].sum(-1), 1.0, atol=1e-12)
    assert not gam[1].any()


def test_den_invariants(tmp_graphs):
    for name in ("tlm_small", "random_split"):
        _, g, V = tmp_graphs[name]
        y, _, lens, _ = oracle.synth_batch(3, 25, V, seed=8, lens=[25, 14, 1])
        la, lb, gd = oracle.den(g, y, lens)
        np.testing.assert_allclose(la, lb, rtol=1e-12)
        for n in range(3):
            np.testing.assert_allclose(gd[n, :lens[n]].sum(-1), 1.0, atol=1e-10)
            assert not gd[n, lens[n]:].any()


def test_assembly_matches_reference_formula(tmp_graphs):
    _, g, V = tmp_graphs["tlm_small"]
    y, labels, lens, ly = oracle.synth_batch(3, 30, V, seed=2, lens=[30, 20, 12])
    for sa in (True, False):
        loss, grad, p = oracle.ctc_crf(g, y, labels, lens, ly, lamb=0.1, size_average=sa)
        sc = 1 / 3 if sa else 1.0
        assert abs(loss - sc * (p["logz_alpha"] - 1.1 * p["logp_ctc"]).sum()) < 1e-9
        np.testing.assert_allclose(grad, sc * (p["gamma_den"] - 1.1 * p["gamma_ctc"]), atol=1e-12)


def test_against_reference_cuda_golden():
    """Golden vectors produced by the reference's own CUDA code (oracle/_ref) on the GPU with
    tests/golden/make_ref_golden.py: the oracle must reproduce the reference's outputs."""
    path = os.path.join(GOLDEN, "ref_cuda_golden.npz")
    if not os.path.exists(path):
        pytest.skip("golden vectors not recorded yet")
    z = np.load(path, allow_pickle=False)
    cases = sorted({k.split("/")[0] for k in z.files})
    assert cases
    for c in cases:
        g = fst.read_fst(os.path.join(GOLDEN, str(z[f"{c}/graph"])))
        y, labels, lx, ly = z[f"{c}/y"], z[f"{c}/labels"], z[f"{c}/lx"], z[f"{c}/ly"]
        lamb = float(z[f"{c}/lamb"])
        loss, grad, parts = oracle.ctc_crf(g, y, labels, lx, ly, lamb)
        assert abs(loss - float(z[f"{c}/ref_loss"])) <= 1e-4 * max(1, abs(loss)), c
        assert np.abs(grad - z[f"{c}/ref_grad"]).max() < 1e-3, c
        np.testing.assert_allclose(parts["logz_alpha"], z[f"{c}/ref_logz_alpha"], rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(parts["logp_ctc"], z[f"{c}/ref_logp_ctc"], rtol=1e-4, atol=1e-4)


def test_oracle_from_logits_matches_autograd_chain(fixture_fst):
    """oracle.ctc_crf_from_logits (raw encoder outputs, SURVEY 8f-1) == torch autograd through log_softmax of the
    oracle's own d loss / d y, and a per-frame constant added to the logits changes nothing."""
    from cat_b200 import fst
    from oracle import oracle
    g = fst.read_fst(fixture_fst)
    rng = np.random.default_rng(3)
    N, T, V = 2, 7, 5
    z = (2.0 * rng.standard_normal((N, T, V)) + 3.0).astype(np.float32)
    labels = np.array([1, 2, 3, 2], np.int32)
    lx, ly = np.array([7, 5], np.int32), np.array([3, 1], np.int32)
    loss, dz, _ = oracle.ctc_crf_from_logits(g, z, labels, lx, ly, 0.05)
    zt = torch.tensor(z, dtype=torch.float64, requires_grad=True)
    y = zt.log_softmax(-1)
    oloss, gy, _ = oracle.ctc_crf(g, y.detach().numpy().astype(np.float32), labels, lx, ly, 0.05)
    y.backward(torch.tensor(gy))
    assert abs(loss - oloss) < 1e-9
    np.testing.assert_allclose(dz, zt.grad.numpy(), atol=1e-9)
    loss2, dz2, _ = oracle.ctc_crf_from_logits(g, z + rng.standard_normal((N, T, 1)).astype(np.float32), labels, lx, ly, 0.05)
    assert abs(loss - loss2) < 1e-5
    np.testing.assert_allclose(dz, dz2, atol=1e-5)


def test_den_oracle_equals_brute_force_path_sum(fixture_fst):
    """The denominator restatement against first principles on the reference's own den_lm.fst: logZ = log of the sum over
    EVERY start->final path of exp(sum of arc weights + emissions + final weight) (den_calculate.cu:75-161 computes the
    same sum by dynamic programming), enumerated path by path; the occupancies likewise."""
    g = fst.read_fst(fixture_fst)
    src, dst, lab, lw = g.log_arcs()
    ew = g.end_weight()
    out = [[] for _ in range(g.num_states)]
    for a in range(g.num_arcs):
        out[src[a]].append(a)
    rng = np.random.default_rng(9)
    T, V = 8, 5
    x = rng.standard_normal((1, T, V))
    y = (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)
    total = 0.0
    occ = np.zeros((T, V))
    n_paths = 0

    def walk(q, t, score, labs):
        nonlocal total, n_paths
        if t == T:
            if np.isfinite(ew[q]):
                p = float(np.exp(np.float64(score) + np.float64(ew[q])))
                total += p
                n_paths += 1
                for tt, k in enumerate(labs):
                    occ[tt, k] += p
            return
        for a in out[q]:
            walk(dst[a], t + 1, score + float(lw[a]) + float(y[0, t, lab[a]]), labs + [int(lab[a])])

    walk(g.start, 0, 0.0, [])
    assert n_paths > 20
    la, lb, gamma = oracle.den(g, y, [T])
    assert abs(la[0] - np.log(total)) < 1e-9 and abs(lb[0] - np.log(total)) < 1e-9
    np.testing.assert_allclose(gamma[0], occ / total, atol=1e-9)


@pytest.mark.parametrize("name,scale", [("tlm_small", 3.0), ("random_split", 3.0), ("tlm_mid", 3.0), ("tlm_mid", 20.0)])
def test_linear_domain_oracle_equals_log_domain_oracle(tmp_graphs, fixture_fst, fixture_inputs, name, scale):
    """The fp64 scaled-linear evaluation used by the at-size GPU tests (oracle_den_linear) is the same function as the
    log-domain restatement of den_calculate.cu (oracle_den): logZ from alpha, logZ from beta and every occupancy, on
    structured, unstructured and peaky inputs, ragged lengths included, plus the reference's own fixture."""
    path, g, V = tmp_graphs[name]
    y, _, lens, _ = oracle.synth_batch(5, 40, V, seed=13, lens=[40, 33, 17, 2, 1], scale=scale)
    la, lb, gd = oracle.den(g, y, lens)
    fa, fb, fg = oracle.den(g, y, lens, fast=True)
    np.testing.assert_allclose(fa, la, rtol=1e-11, atol=1e-9)
    np.testing.assert_allclose(fb, lb, rtol=1e-11, atol=1e-9)
    np.testing.assert_allclose(fg, gd, atol=1e-10)
    fi = fixture_inputs
    gf = fst.read_fst(fixture_fst)
    a = oracle.den(gf, fi["y"], fi["lx"])
    b = oracle.den(gf, fi["y"], fi["lx"], fast=True)
    for u, v in zip(a, b):
        np.testing.assert_allclose(v, u, rtol=1e-12, atol=1e-12)
    assert abs(b[0][0] - (-6.25832785)) < 1e-6
