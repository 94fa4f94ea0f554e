import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

GOLDEN = os.path.join(ROOT, "tests", "golden")
FIXTURE_FST = os.path.join(GOLDEN, "den_lm_fixture.fst")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def fixture_fst():
    return FIXTURE_FST


@pytest.fixture(scope="session")
def fixture_inputs():
    """The reference's only test case: src/ctc_crf/test/main.py:16-28 (values restated, not copied code)."""
    p = np.array([[[0.1, 0.1, 0.5, 0.1, 0.2],
                   [0.5, 0.1, 0.1, 0.2, 0.2],
                   [0.1, 0.7, 0.1, 0.05, 0.05],
                   [0.6, 0.1, 0.1, 0.1, 0.1],
                   [0.1, 0.1, 0.1, 0.6, 0.1]]], dtype=np.float32)
    return dict(y=np.log(p), labels=np.array([2, 1, 4], np.int32), lx=np.array([5], np.int32),
                ly=np.array([3], np.int32), lamb=0.01)


@pytest.fixture(scope="session")
def tmp_graphs(tmp_path_factory):
    """Small den graphs written once per session: T-compose-LM shaped and an unstructured one."""
    from cat_b200 import fst
    d = tmp_path_factory.mktemp("graphs")
    out = {}
    g = fst.make_synthetic_den(50, 6, 12, seed=7)
    fst.write_fst(str(d / "tlm_small.fst"), g)
    out["tlm_small"] = (str(d / "tlm_small.fst"), g, 12)
    g = fst.make_random_den(40, 300, 7, seed=3)
    fst.write_fst(str(d / "random_split.fst"), g)
    out["random_split"] = (str(d / "random_split.fst"), g, 7)
    g = fst.make_synthetic_den(600, 12, 40, seed=11)
    fst.write_fst(str(d / "tlm_mid.fst"), g)
    out["tlm_mid"] = (str(d / "tlm_mid.fst"), g, 40)
    return out
