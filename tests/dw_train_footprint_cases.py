"""The footprint table of the training entry points (include/litepose_b200_train.h, _lib.TRAIN_SIGNATURES), in the
form of tests/footprint_cases.py: every case runs its call on guarded buffers (footprint_util.Guarded) and names its
reference, the bit-exact restatement dw_train_emul.  test_gpu_dw_train_footprint.py runs them; importing this module
needs no GPU (test_dw_train_host.py checks that every launching training symbol has a case)."""
import functools
import zlib

import numpy as np

import dw_train_emul as dte
from footprint_cases import Case
from footprint_util import SKEW
from litepose_b200 import _lib

F16, F32 = np.float16, np.float32
CASES = []


def _L():
    return _lib.load()


def _s():
    import torch
    return torch.cuda.current_stream().cuda_stream


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


# (n, c, h, w, k, stride, fp16, odd element offset): a plane taller than one wgrad range with ragged tiles, H and W
# below k, 1 x 1 planes, the widest kernel at both strides
DWT = [(2, 3, 131, 37, 3, 1, False, False), (3, 5, 4, 3, 5, 2, True, True), (2, 4, 1, 1, 7, 1, False, True),
       (1, 6, 40, 70, 7, 2, True, False), (2, 2, 33, 65, 5, 1, True, False)]


def _dwt_case(n, c, h, w, k, s, fp16, odd):
    dt = F16 if fp16 else F32
    ho, wo = dte.out_size(h, s), dte.out_size(w, s)
    skew = SKEW + np.dtype(dt).itemsize if odd else None        # the element alignment the header documents
    code = _lib.LP_DT_F16 if fp16 else _lib.LP_DT_F32

    @functools.lru_cache(None)
    def inputs():
        rng = _rng("dw_train", n, c, h, w, k, s, fp16)
        return (rng.standard_normal((n, c, h, w)).astype(dt), (rng.standard_normal((c, k, k)) / k).astype(dt),
                rng.standard_normal((n, c, ho, wo)).astype(dt))

    def fwd(A):
        x, wt, _ = inputs()
        xd, wd = A.inp("x", x, skew=skew), A.inp("w", wt, skew=skew)
        y = A.out("y", (n, c, ho, wo), dt, skew=skew)
        return [_L().lp_dw_nchw_fwd(xd.data_ptr(), wd.data_ptr(), y.data_ptr(), n, c, h, w, k, s, code, _s())]

    def dgrad(A):
        _, wt, dy = inputs()
        dd, wd = A.inp("dy", dy, skew=skew), A.inp("w", wt, skew=skew)
        dx = A.out("dx", (n, c, h, w), dt, skew=skew)
        return [_L().lp_dw_nchw_dgrad(dd.data_ptr(), wd.data_ptr(), dx.data_ptr(), n, c, h, w, k, s, code, _s())]

    def wgrad(A):
        x, _, dy = inputs()
        xd, dd = A.inp("x", x, skew=skew), A.inp("dy", dy, skew=skew)
        dw = A.out("dw", (c, k, k), dt, skew=skew)
        nb = _L().lp_dw_nchw_wgrad_workspace_bytes(n, c, h, w, k, s)
        ws = A.ws("workspace", nb, skew=4 if odd else 256)
        return [_L().lp_dw_nchw_wgrad(xd.data_ptr(), dd.data_ptr(), dw.data_ptr(), n, c, h, w, k, s, code,
                                      ws.data_ptr(), nb, _s())]

    sfx = "k%d-s%d-n%d-c%d-%dx%d-%s%s" % (k, s, n, c, h, w, "fp16" if fp16 else "fp32", "-odd" if odd else "")
    CASES.append(Case("dw_nchw_fwd-" + sfx, ["lp_dw_nchw_fwd"], fwd,
                      lambda: {"y": dte.fwd(inputs()[0], inputs()[1], s)}))
    CASES.append(Case("dw_nchw_dgrad-" + sfx, ["lp_dw_nchw_dgrad"], dgrad,
                      lambda: {"dx": dte.dgrad(inputs()[2], inputs()[1], s, h, w)}))
    CASES.append(Case("dw_nchw_wgrad-" + sfx, ["lp_dw_nchw_wgrad"], wgrad,
                      lambda: {"dw": dte.wgrad(inputs()[0], inputs()[2], k, s)}))


for _c in DWT:
    _dwt_case(*_c)


def launching_symbols():
    """every symbol of _lib.TRAIN_SIGNATURES that launches device work (all but *_workspace_bytes)"""
    return {s for s in _lib.TRAIN_SIGNATURES if not s.endswith("_workspace_bytes")}


def covered_symbols():
    return {e for c in CASES for e in c.entries}
