"""Drop-in for the ``warp_ctct`` package CAT's transducer trainer imports for ``"trainer": {"topo": "ctct"}``
(cat/rnnt/train.py): ``ctct_loss`` over the joiner's output, compact or padded, and ``ctct_simple_loss``, the loss of the
``LogAdd`` joiner taken from the encoder and predictor outputs without the joint tensor."""
from cat_b200.ctct import ctct_loss, ctct_simple_loss  # noqa: F401

__all__ = ["ctct_loss", "ctct_simple_loss"]
