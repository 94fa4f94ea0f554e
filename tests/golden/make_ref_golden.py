"""Records golden vectors from the REFERENCE'S OWN CUDA CODE (oracle/_ref: den_calculate.cu + ctc_entrypoint.cu
compiled unmodified for sm_90a) on seeded inputs.  Needs a GPU:

    gpurun -- 'python tests/golden/make_ref_golden.py'     # writes gpurun_out/ref_cuda_golden.npz
    cp gpurun_out/ref_cuda_golden.npz tests/golden/        # commit

The den graphs of the cases are small files committed next to this script (written by this script when absent).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from cat_b200 import fst  # noqa: E402
from oracle import oracle, ref_cuda  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def cases():
    p = np.array([[[0.1, 0.1, 0.5, 0.1, 0.2], [0.5, 0.1, 0.1, 0.2, 0.2], [0.1, 0.7, 0.1, 0.05, 0.05],
                   [0.6, 0.1, 0.1, 0.1, 0.1], [0.1, 0.1, 0.1, 0.6, 0.1]]], dtype=np.float32)
    yield "fixture", "den_lm_fixture.fst", None, (np.log(p), np.array([2, 1, 4], np.int32), np.array([5], np.int32),
                                                   np.array([3], np.int32)), 0.01
    yield "tlm_a", "golden_tlm_a.fst", (60, 5, 12), oracle.synth_batch(4, 40, 12, seed=11, lens=[40, 31, 18, 6]), 0.1
    yield "tlm_b", "golden_tlm_b.fst", (300, 10, 40), oracle.synth_batch(6, 80, 40, seed=12, lens=[80, 80, 66, 41, 23, 9]), 0.01


def main():
    out = {}
    for name, gfile, gspec, (y, labels, lx, ly), lamb in cases():
        gpath = os.path.join(GOLDEN, gfile)
        if not os.path.exists(gpath):
            fst.write_fst(gpath, fst.make_synthetic_den(*gspec, seed=7))
        ctx = ref_cuda.RefContext(gpath, 0)
        costs, grad, parts = ref_cuda.ctc_crf_forward(ctx, torch.tensor(y, device="cuda"), torch.tensor(labels),
                                                      torch.tensor(lx), torch.tensor(ly), lamb, True)
        torch.cuda.synchronize()
        ctx.close()
        out[f"{name}/graph"] = np.array(gfile)
        out[f"{name}/y"] = y
        out[f"{name}/labels"] = labels
        out[f"{name}/lx"] = lx
        out[f"{name}/ly"] = ly
        out[f"{name}/lamb"] = np.array(lamb)
        out[f"{name}/ref_loss"] = np.array(costs.item())
        out[f"{name}/ref_grad"] = grad.cpu().numpy()
        out[f"{name}/ref_logz_alpha"] = parts["logz_alpha"].cpu().numpy()
        out[f"{name}/ref_logz_beta"] = parts["logz_beta"].cpu().numpy()
        out[f"{name}/ref_logp_ctc"] = parts["logp_ctc"].cpu().numpy()
        print(name, "ref loss", costs.item(), "ctc status", parts["ctc_status"])
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    np.savez_compressed(os.path.join(ROOT, "gpurun_out", "ref_cuda_golden.npz"), **out)
    print("wrote gpurun_out/ref_cuda_golden.npz")


if __name__ == "__main__":
    main()
