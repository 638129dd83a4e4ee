"""-m gpu: where the training kernels read and write.  Every case of dw_train_footprint_cases runs on guarded buffers
(footprint_util.Guarded, as test_gpu_footprint.py runs the inference entry points): the outputs equal the bit-exact
restatement, every guard byte and every input byte is unchanged, no output element keeps the sentinel, and the call
returned LP_OK.  One more case shows the harness sees a one-image overrun of lp_dw_nchw_fwd."""
import numpy as np
import pytest
import torch

import dw_train_emul as dte
import dw_train_footprint_cases as tfc
from footprint_util import Guarded
from litepose_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", tfc.CASES, ids=[c.id for c in tfc.CASES])
def test_footprint(case):
    g = Guarded()
    rcs = case.run(g)
    assert all(rc == _lib.LP_OK for rc in rcs), "%s returned %s: %s" % (case.id, rcs, _lib.load().lp_last_error())
    errs = g.verify(case.ref(), case.untouched)
    assert not errs, "%s:\n  %s" % (case.id, "\n  ".join(errs))


def test_detects_fwd_overrun():
    """one more image than the output holds: that image's planes land in the back guard"""
    n, c, h, w = 2, 3, 9, 13
    rng = np.random.default_rng(1)
    x = rng.standard_normal((n + 1, c, h, w)).astype(np.float32)
    wt = rng.standard_normal((c, 3, 3)).astype(np.float32)
    g = Guarded()
    xd, wd = g.inp("x", x), g.inp("w", wt)
    y = g.out("y", (n, c, h, w), np.float32)
    rc = _lib.load().lp_dw_nchw_fwd(xd.data_ptr(), wd.data_ptr(), y.data_ptr(), n + 1, c, h, w, 3, 1, _lib.LP_DT_F32,
                                    torch.cuda.current_stream().cuda_stream)
    assert rc == _lib.LP_OK
    errs = g.verify({"y": dte.fwd(x[:n], wt, 1)})
    assert any(e.startswith("y: back guard modified") for e in errs), errs
    assert not [e for e in errs if not e.startswith("y: back guard")], errs
