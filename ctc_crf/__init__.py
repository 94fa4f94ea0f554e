"""Drop-in for the reference's ``ctc_crf`` package (src/ctc_crf/ctc_crf/__init__.py): callers such as
cat/ctc/train.py:118,137 keep ``from ctc_crf import CTC_CRF_LOSS, CRFContext`` unchanged."""
from cat_b200 import _C  # noqa: F401
from cat_b200.loss import (CRFContext, CTC_CRF_LOSS, WARP_CTC_LOSS, _CTC_CRF, _CTC_CRF_LOGITS, _WARP_CTC_GPU,  # noqa: F401
                           CTCBeamDecoder, crf_sample, ctc_align, ctc_beam_search, samples_to_labels, __version__)
from cat_b200.ngram import NGramLM  # noqa: F401
from cat_b200.wfst import DecodingGraph, WfstResult, fst_decode  # noqa: F401
