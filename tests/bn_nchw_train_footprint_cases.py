"""The footprint table of the train-mode BatchNorm entry points (include/litepose_b200_train_bn.h,
_lib.TRAIN_BN_SIGNATURES), in the form of tests/footprint_cases.py: every case runs its call on guarded buffers
(footprint_util.Guarded) and names its reference, the bit-exact restatement bn_nchw_train_emul.
test_gpu_bn_nchw_train_footprint.py runs them; importing this module needs no GPU (test_bn_nchw_train_host.py checks
that every launching symbol has a case)."""
import functools
import zlib

import numpy as np

import bn_nchw_train_emul as bte
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


# (n, c, h, w, act, fp16, odd element offset): a channel past one reduction range with a ragged last one, 1 x 1 planes,
# an odd plane below one warp, a plane of more than one apply CTA
BNT = [(3, 5, 61, 53, 2, False, False), (7, 3, 1, 1, 1, True, True), (16, 6, 7, 7, 0, False, True),
       (2, 4, 40, 70, 2, True, False)]


def _bnt_case(n, c, h, w, act, fp16, odd):
    dt = F16 if fp16 else F32
    skew = SKEW + np.dtype(dt).itemsize if odd else None        # the element alignment the header documents
    pskew = SKEW + 4 if odd else None
    code = _lib.LP_DT_F16 if fp16 else _lib.LP_DT_F32

    @functools.lru_cache(None)
    def inputs():
        rng = _rng("bn_nchw_train", n, c, h, w, act, fp16)
        x = (rng.standard_normal((n, c, h, w)) * 2 + rng.standard_normal((1, c, 1, 1))).astype(dt)
        prm = [rng.uniform(0.5, 1.5, c), rng.standard_normal(c) * 0.5, rng.standard_normal(c) * 0.1,
               rng.uniform(0.75, 1.25, c)]
        return (x,) + tuple(p.astype(F32) for p in prm) + (rng.standard_normal((n, c, h, w)).astype(dt),)

    @functools.lru_cache(None)
    def ref_fwd():
        x, g, b, rm, rv, _ = inputs()
        return bte.fwd(x, g, b, rm, rv, 0.1, 1e-5, act)

    def fwd(A):
        x, g, b, rm, rv, _ = inputs()
        xd = A.inp("x", x, skew=skew)
        gd, bd = A.inp("gamma", g, skew=pskew), A.inp("beta", b, skew=pskew)
        # the running statistics are read and written in place: outputs initialised with the old values
        rmd = A.out("running_mean", (c,), F32, skew=pskew, init=rm)
        rvd = A.out("running_var", (c,), F32, skew=pskew, init=rv)
        y = A.out("y", (n, c, h, w), dt, skew=skew)
        sv = A.out("saved", (4, c), F32, skew=pskew)
        nb = _L().lp_bn_nchw_workspace_bytes(n, c, h, w)
        ws = A.ws("workspace", nb, skew=8 if odd else 256)
        return [_L().lp_bn_nchw_fwd(xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), rmd.data_ptr(), rvd.data_ptr(), 0.1,
                                    1e-5, y.data_ptr(), sv.data_ptr(), n, c, h, w, act, code, ws.data_ptr(), nb,
                                    _s())]

    def bwd(A):
        x, g, _, _, _, dy = inputs()
        saved = ref_fwd()[1]
        xd, dd = A.inp("x", x, skew=skew), A.inp("dy", dy, skew=skew)
        gd, sd = A.inp("gamma", g, skew=pskew), A.inp("saved", saved, skew=pskew)
        dx = A.out("dx", (n, c, h, w), dt, skew=skew)
        dg, db = A.out("dgamma", (c,), F32, skew=pskew), A.out("dbeta", (c,), F32, skew=pskew)
        nb = _L().lp_bn_nchw_workspace_bytes(n, c, h, w)
        ws = A.ws("workspace", nb, skew=8 if odd else 256)
        return [_L().lp_bn_nchw_bwd(xd.data_ptr(), dd.data_ptr(), gd.data_ptr(), sd.data_ptr(), dx.data_ptr(),
                                    dg.data_ptr(), db.data_ptr(), n, c, h, w, act, code, ws.data_ptr(), nb, _s())]

    def ref_bwd():
        x, g, _, _, _, dy = inputs()
        dx, dg, db = bte.bwd(x, dy, g, ref_fwd()[1], act)
        return {"dx": dx, "dgamma": dg, "dbeta": db}

    sfx = "act%d-n%d-c%d-%dx%d-%s%s" % (act, n, c, h, w, "fp16" if fp16 else "fp32", "-odd" if odd else "")
    CASES.append(Case("bn_nchw_fwd-" + sfx, ["lp_bn_nchw_fwd"], fwd,
                      lambda: dict(zip(("y", "saved", "running_mean", "running_var"), ref_fwd()))))
    CASES.append(Case("bn_nchw_bwd-" + sfx, ["lp_bn_nchw_bwd"], bwd, ref_bwd))


for _c in BNT:
    _bnt_case(*_c)


def launching_symbols():
    """every symbol of _lib.TRAIN_BN_SIGNATURES that launches device work (all but *_workspace_bytes)"""
    return {s for s in _lib.TRAIN_BN_SIGNATURES if not s.endswith("_workspace_bytes")}


def covered_symbols():
    return {e for c in CASES for e in c.entries}
