"""Drop-in for the ``gather`` package (torch-gather) CAT's compact joiner imports (cat/rnnt/joiner.py:12,108-139):
``gather.cat`` and ``gather.sum``."""
from cat_b200.rnnt import gather_cat as cat  # noqa: F401
from cat_b200.rnnt import gather_sum as sum  # noqa: F401,A001

__all__ = ["cat", "sum"]
