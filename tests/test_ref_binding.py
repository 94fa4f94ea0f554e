"""The drop-in boundary as a CAT maintainer would use it: the reference's OWN pybind module -- src/ctc_crf/binding.cpp,
compiled unmodified by oracle/Makefile (`make -C oracle ref_binding`, setup.py:27-37 with the two `libraries` swapped) --
linked against this repository's libctc_crf_b200.so instead of libfst_den.so + libwarpctc.so.

CPU: the module exists, exports binding.cpp's four functions and resolves its native symbols from OUR library.
GPU: the call sequence of the reference's `_CTC_CRF.forward` (ctc_crf/__init__.py:58-90, restated here line by line because
the reference tree is not on the GPU box) driven through that module on the reference's own test input (test/main.py:14-42)
gives the survey's known answer, loss = -2.478625, and the oracle's gradient."""
import importlib.util
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT

SO = os.path.join(ROOT, "oracle", "_ref", "ctc_crf_refbinding", "_C.so")


def _load():
    if not os.path.exists(SO):
        from cat_b200 import build
        build.build()
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "ref_binding"], stdout=subprocess.DEVNULL)
        if not os.path.exists(SO):
            pytest.skip("oracle/_ref/ctc_crf_refbinding/_C.so not built (needs the reference sources at build time, oracle/Makefile REF)")
    spec = importlib.util.spec_from_file_location("_C", SO)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_reference_binding_links_against_this_library():
    core = _load()
    for name in ("gpu_ctc", "gpu_den", "init_env", "release_env"):       # binding.cpp:118-126
        assert callable(getattr(core, name))
    maps = open("/proc/self/maps").read()
    assert "cat_b200/libctc_crf_b200.so" in maps                           # Init/compute_alpha/... come from our library
    assert "libfst_den" not in maps and "libwarpctc" not in maps


@pytest.mark.gpu
def test_reference_forward_sequence_through_reference_binding(fixture_fst, fixture_inputs):
    from oracle import oracle
    from cat_b200 import fst
    core = _load()
    fi = fixture_inputs
    gpus = torch.IntTensor([0])
    core.init_env(fixture_fst, gpus)                                        # CRFContext.__init__, __init__.py:147-166
    try:
        lamb = fi["lamb"]
        logits = torch.tensor(fi["y"], device="cuda:0")
        labels = torch.tensor(fi["labels"], dtype=torch.int32)
        input_lengths = torch.tensor(fi["lx"], dtype=torch.int32)
        label_lengths = torch.tensor(fi["ly"], dtype=torch.int32)
        # --- _CTC_CRF.forward, __init__.py:58-90 ---
        logits = logits.contiguous()
        batch_size = logits.size(0)
        costs_alpha_den = torch.zeros(logits.size(0)).type_as(logits)
        costs_beta_den = torch.zeros(logits.size(0)).type_as(logits)
        grad_den = torch.zeros(logits.size()).type_as(logits)
        costs_ctc = torch.zeros(logits.size(0))
        act = torch.transpose(logits, 0, 1).contiguous()
        grad_ctc = torch.zeros(act.size()).type_as(logits)
        core.gpu_ctc(act, grad_ctc, labels, label_lengths, input_lengths, logits.size(0), costs_ctc, 0)
        core.gpu_den(logits, grad_den, input_lengths.cuda(), costs_alpha_den, costs_beta_den)
        grad_ctc = torch.transpose(grad_ctc, 0, 1)
        costs_ctc = costs_ctc.to(logits.get_device())
        grad_all = grad_den - (1 + lamb) * grad_ctc
        costs_all = costs_alpha_den - (1 + lamb) * costs_ctc
        costs = torch.FloatTensor([costs_all.sum()]).to(logits.get_device())
        grad_all = grad_all / batch_size
        costs = costs / batch_size
        # --- known answers (SURVEY.md 8c) and the oracle ---
        assert abs(float(costs.item()) - (-2.47862480)) < 1e-4
        assert abs(float(costs_alpha_den[0]) - (-6.25832785)) < 1e-4
        assert abs(float(costs_beta_den[0]) - (-6.25832785)) < 1e-4
        assert abs(float(costs_ctc[0]) - (-3.74228025)) < 1e-4
        oloss, ograd, _ = oracle.ctc_crf(fst.read_fst(fixture_fst), fi["y"], fi["labels"], fi["lx"], fi["ly"], lamb)
        assert np.abs(grad_all.cpu().numpy() - ograd).max() < 1e-3
        # a batch that is NOT a multiple of 32 with binding.cpp's own (T+1)*N*DEN_NUM_STATES alpha buffer, twice in a row
        N, T, V = 5, 7, 5
        y, labs, lens, ly = oracle.synth_batch(N, T, V, seed=3, lens=[7, 6, 5, 4, 2])      # (shorter ones cannot reach a final state)
        lg = torch.tensor(y, device="cuda:0")
        for _ in range(2):
            gd = torch.zeros_like(lg)
            ca, cb = torch.zeros(N, device="cuda:0"), torch.zeros(N, device="cuda:0")
            core.gpu_den(lg, gd, torch.tensor(lens).cuda(), ca, cb)
            la, lb, g_or = oracle.den(fst.read_fst(fixture_fst), y, lens)
            np.testing.assert_allclose(ca.cpu().numpy(), la, rtol=1e-4, atol=1e-4)
            np.testing.assert_allclose(cb.cpu().numpy(), lb, rtol=1e-4, atol=1e-4)
            assert np.abs(gd.cpu().numpy() - g_or).max() < 1e-3
    finally:
        core.release_env(gpus)
