"""The loss under CAT's own mixed precision: fp16 autocast around the model with a GradScaler step
(cat/shared/manager.py:29,280,533,547,620-627), restated by tools/trainer_smoke.py --amp --amp-dtype float16.  With
--from-logits the criterion takes the encoder's fp16 logits as they are."""
import os
import sys

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(ROOT, "tools"))


@pytest.mark.parametrize("flags", [["--amp", "--amp-dtype", "float16"], ["--amp", "--amp-dtype", "float16", "--from-logits"]])
def test_trainer_smoke_fp16_amp(flags):
    import numpy as np
    import trainer_smoke
    log = trainer_smoke.run(trainer_smoke.parse(["--steps", "30"] + flags))
    assert len(log) == 30 and np.isfinite(log).all()
    assert sum(log[-5:]) < sum(log[:5])            # (run() itself raises unless the loss fell by >= 10 %)
