"""cat_b200 -- H100-native implementation of the CTC-CRF loss hot path of thu-spmi/CAT (src/ctc_crf).

``import ctc_crf`` (the top-level shim package) gives the reference's names; this package holds the
implementation: ``csrc/`` (sm_90a CUDA kernels + C ABI), ``_C`` (mirror of binding.cpp), ``loss``
(mirror of ctc_crf/__init__.py), ``fst`` (den-graph files), ``dist`` (minibatch sharding over GPUs).
"""
from .loss import CRFContext, CTC_CRF_LOSS, WARP_CTC_LOSS, ctc_align, __version__  # noqa: F401
