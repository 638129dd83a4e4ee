"""-m gpu: where the train-mode BatchNorm kernels read and write.  Every case of bn_nchw_train_footprint_cases runs on
guarded buffers (footprint_util.Guarded, as test_gpu_footprint.py runs the inference entry points): the outputs, the
running statistics updated in place included, equal the bit-exact restatement, every guard byte and every input byte
is unchanged, no output element keeps the sentinel, and the call returned LP_OK."""
import pytest

import bn_nchw_train_footprint_cases as bfc
from footprint_util import Guarded
from litepose_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", bfc.CASES, ids=[c.id for c in bfc.CASES])
def test_footprint(case):
    g = Guarded()
    rcs = case.run(g)
    assert all(rc == _lib.LP_OK for rc in rcs), "%s returned %s: %s" % (case.id, rcs, _lib.load().lp_last_error())
    errs = g.verify(case.ref(), case.untouched)
    assert not errs, "%s:\n  %s" % (case.id, "\n  ".join(errs))
