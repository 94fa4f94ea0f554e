"""Drop-in for the ``warp_rnnt`` package CAT's transducer trainers import (cat/rnnt/train.py:22,217): ``rnnt_loss`` with
``compact=True`` over the joiner's compact output, or the padded (N, T, U+1, V) layout, and ``rnnt_loss_simple``, the loss
of the ``LogAdd`` joiner taken from the encoder and predictor outputs without the joint tensor."""
from cat_b200.rnnt import rnnt_loss  # noqa: F401
from cat_b200.rnnt_simple import rnnt_loss_simple  # noqa: F401

__all__ = ["rnnt_loss", "rnnt_loss_simple"]
