"""TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

Drives ``oracle/_ref/libctc_crf_ref.so`` -- the reference's own den_calculate.cu + ctc_entrypoint.cu compiled
UNMODIFIED for sm_90a (oracle/Makefile) -- exactly the way the reference's binding.cpp:65-117 and
ctc_crf/__init__.py:58-90 drive it (same allocations, same call order, same post-processing), with torch
tensors for memory.  This is the parity target named in BASELINE.json ("the reference's own CUDA ctc_crf").
Needs a GPU; never imported by the product.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# "patched": the reference sources with the two sm_70+ defects patched at build time (oracle/Makefile): the
#            shfl.sync membermask in moderngpu's intrinsics and the non-volatile warp-synchronous reduction in
#            alpha_lld_kernal.  "unmodified": the sources exactly as they are (see oracle/Makefile for what goes wrong).
VARIANT = os.environ.get("CCB_REF_VARIANT", "patched")
_SO = os.path.join(_HERE, "_ref", "libctc_crf_ref.so" if VARIANT == "unmodified" else "libctc_crf_ref_patched.so")
_lib = None
ATOMIC_CONST = 32   # binding.cpp:17-18


class _ctcOptions(C.Structure):
    _fields_ = [("stream", C.c_void_p), ("blank_label", C.c_int)]


def available() -> bool:
    return os.path.exists(_SO)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError(f"{_SO} missing: run `make -C oracle ref` where the reference sources are present (oracle/Makefile REF)")
        L = C.CDLL(_SO)
        vp, ip = C.c_void_p, C.POINTER(C.c_int)
        L.Init.argtypes = [C.c_char_p, C.c_int, ip]; L.Init.restype = None
        L.Release.argtypes = [C.c_int, ip]; L.Release.restype = None
        L.compute_alpha.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]; L.compute_alpha.restype = None
        L.compute_beta_and_grad.argtypes = [vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
        L.compute_beta_and_grad.restype = None
        L.compute_ctc_loss.argtypes = [vp, vp, ip, ip, ip, C.c_int, C.c_int, C.POINTER(C.c_float), vp, _ctcOptions]
        L.compute_ctc_loss.restype = C.c_int
        L.get_workspace_size.argtypes = [ip, ip, C.c_int, C.c_int, _ctcOptions, C.POINTER(C.c_size_t)]
        L.get_workspace_size.restype = C.c_int
        _lib = L
    return _lib


def _iptr(t):
    return C.cast(t.data_ptr(), C.POINTER(C.c_int))


class RefContext:
    """ctc_crf/__init__.py:147-171 (CRFContext) over the reference library."""

    def __init__(self, den_lm: str, gpu: int = 0):
        self._gpus = torch.IntTensor([gpu])
        lib().Init(den_lm.encode(), 1, _iptr(self._gpus))
        self.num_states = C.c_int.in_dll(lib(), "DEN_NUM_STATES").value
        self.num_arcs = C.c_int.in_dll(lib(), "DEN_NUM_ARCS").value

    def close(self):
        if self._gpus is not None:
            lib().Release(1, _iptr(self._gpus))
            self._gpus = None


def gpu_den(ctx: RefContext, logits, grad_net, input_lengths, costs_alpha, costs_beta):
    """binding.cpp:65-84"""
    N, T, V = logits.shape
    dev = logits.device
    S = ctx.num_states
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    alpha = torch.empty((T + 1, N, S), dtype=torch.float32, device=dev)
    beta = torch.empty((2, N, S), dtype=torch.float32, device=dev)
    grad_storage = torch.empty((ATOMIC_CONST, N, V), dtype=torch.float32, device=dev)
    L = lib()
    L.compute_alpha(alpha.data_ptr(), logits.data_ptr(), N, T, S, V, input_lengths.data_ptr(), costs_alpha.data_ptr(), stream)
    L.compute_beta_and_grad(beta.data_ptr(), alpha.data_ptr(), logits.data_ptr(), costs_alpha.data_ptr(),
                            grad_storage.data_ptr(), grad_net.data_ptr(), N, T, S, V, input_lengths.data_ptr(),
                            costs_beta.data_ptr(), stream)


def gpu_ctc(probs, grads, labels, label_sizes, sizes, minibatch_size, costs, blank_label):
    """binding.cpp:86-117 (status codes are ignored there; surfaced here)"""
    V = probs.size(2)
    dev = probs.device
    opts = _ctcOptions(stream=torch.cuda.current_stream(dev).cuda_stream, blank_label=blank_label)
    nbytes = C.c_size_t(0)
    L = lib()
    L.get_workspace_size(_iptr(label_sizes), _iptr(sizes), V, minibatch_size, opts, C.byref(nbytes))
    ws = torch.empty(nbytes.value // 4 + 1, dtype=torch.float32, device=dev)
    return L.compute_ctc_loss(probs.data_ptr(), grads.data_ptr(), _iptr(labels), _iptr(label_sizes), _iptr(sizes), V,
                              minibatch_size, C.cast(costs.data_ptr(), C.POINTER(C.c_float)), ws.data_ptr(), opts)


def ctc_crf_forward(ctx: RefContext, logits, labels, input_lengths, label_lengths, lamb=0.1, size_average=True):
    """ctc_crf/__init__.py:58-90 (_CTC_CRF.forward), returning (costs[1], grad_all, parts)."""
    logits = logits.contiguous()
    batch_size = logits.size(0)
    costs_alpha_den = torch.zeros(logits.size(0)).type_as(logits)
    costs_beta_den = torch.zeros(logits.size(0)).type_as(logits)
    grad_den = torch.zeros(logits.size()).type_as(logits)
    costs_ctc = torch.zeros(logits.size(0))
    act = torch.transpose(logits, 0, 1).contiguous()
    grad_ctc = torch.zeros(act.size()).type_as(logits)
    status = gpu_ctc(act, grad_ctc, labels, label_lengths, input_lengths, logits.size(0), costs_ctc, 0)
    gpu_den(ctx, logits, grad_den, input_lengths.cuda(), costs_alpha_den, costs_beta_den)
    grad_ctc = torch.transpose(grad_ctc, 0, 1)
    costs_ctc = costs_ctc.to(logits.device)
    grad_all = grad_den - (1 + lamb) * grad_ctc
    costs_all = costs_alpha_den - (1 + lamb) * costs_ctc
    costs = costs_all.sum().reshape(1)
    if size_average:
        grad_all = grad_all / batch_size
        costs = costs / batch_size
    parts = dict(logz_alpha=costs_alpha_den, logz_beta=costs_beta_den, logp_ctc=costs_ctc, gamma_den=grad_den,
                 gamma_ctc=grad_ctc, ctc_status=status)
    return costs, grad_all, parts
