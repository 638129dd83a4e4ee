"""The footprint table: for every C-ABI entry point that launches work, a few cases run inside guarded buffers
(footprint_util.Guarded) against the reference its own test uses.

A case is Case(id, entries, run, ref, untouched, prec):
  run(A)   allocates every tensor of the call through A (Guarded or Plain) and launches; -> list of return codes;
  ref()    the expected outputs, name -> array (the emulators: dw_emul, mma_emul, conv_ref, bn_train_emul, glue_emul, the
           transforms goldens), or None: the same calls on plain tensors (Plain) are the reference - the parser,
           fast-grouping, payload and planting entry points, which their own tests hold to the oracles that way;
  untouched  outputs whose header contract leaves some entries unwritten (there the sentinel must survive exactly);
  prec     the lp_set_dw_precision setting of the case.
The inputs are drawn when the case runs (numpy only on the host; parser stages take their inputs from the earlier
stages run on plain tensors), so importing this module needs no GPU: the CPU coverage test reads `entries`."""
import functools
import zlib

import numpy as np

import bn_train_emul as bte
import conv_ref as cr
import dw_emul as de
import glue_emul as ge
import mma_emul as me
import simplenet_emul as se
from footprint_util import SKEW, sentinel_array
from litepose_b200 import _lib

F16, F32, F64, I32, I64, U8 = np.float16, np.float32, np.float64, np.int32, np.int64, np.uint8


class Case(object):
    def __init__(self, cid, entries, run, ref=None, untouched=(), prec=-1):
        self.id, self.entries, self.run, self.ref, self.untouched, self.prec = cid, tuple(entries), run, ref, \
            tuple(untouched), prec


def _L():
    return _lib.load()


def _s():
    import torch
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def _u16(a):
    return np.ascontiguousarray(a, F16).view(np.uint16)


def _addr(a):
    return None if a is None else a.ctypes.data


# ---------------------------------------------------------------- host packing (numpy in, numpy out)
def pack_pw(w, bias):
    """lp_pw1x1_pack of w [N, K] fp16 and bias [N] fp32 (or None) -> (packed fp16, packed bias fp32)"""
    lib = _L()
    n, k = w.shape
    w16 = _u16(w)
    b = None if bias is None else np.ascontiguousarray(bias, F32)
    wp = np.zeros(lib.lp_pw1x1_packed_elems(k, n), np.uint16)
    bp = np.zeros(lib.lp_pw1x1_packed_bias_elems(n), F32)
    _lib.check(lib.lp_pw1x1_pack(w16.ctypes.data, _addr(b), k, n, wp.ctypes.data, bp.ctypes.data), "pw1x1_pack")
    return wp.view(F16), bp


def pack_wexp(we):
    lib = _L()
    ce, cin = we.shape
    w16 = _u16(we)
    out = np.zeros(lib.lp_block_s1_wexp_elems(cin, ce), np.uint16)
    _lib.check(lib.lp_block_s1_pack_wexp(w16.ctypes.data, cin, ce, out.ctypes.data), "block_s1_pack_wexp")
    return out.view(F16)


def pack_deconv(wr, ww, b, cr_, cw, co):
    lib = _L()
    wr16 = _u16(wr)
    ww16 = _u16(ww) if cw else None
    wp = np.zeros(lib.lp_deconv_packed_elems(cr_, cw, co), np.uint16)
    bp = np.zeros(lib.lp_deconv_packed_bias_elems(co), F32)
    _lib.check(lib.lp_deconv_pack(wr16.ctypes.data, _addr(ww16), b.ctypes.data, cr_, cw, co, wp.ctypes.data,
                                  bp.ctypes.data), "deconv_pack")
    return wp.view(F16), bp


def pack_head(w1, w2, c1, c2, co):
    lib = _L()
    h1 = _u16(w1)
    h2 = _u16(w2) if c2 else None
    wp = np.zeros(lib.lp_head_packed_elems(c1, c2, co), np.uint16)
    _lib.check(lib.lp_head_pack(h1.ctypes.data, _addr(h2), c1, c2, co, wp.ctypes.data), "head_pack")
    return wp.view(F16)


def pack_head_fused(d1, b1, d2, b2, w1, w2, c1, c2, co):
    lib = _L()
    dwc = np.zeros(lib.lp_head_fused_dw_elems(c1, c2), np.uint16)
    bdc = np.zeros(dwc.size // 25, F32)
    pwc = np.zeros(lib.lp_head_fused_pw_elems(c1, c2, co), np.uint16)
    a1, a2 = _u16(d1), _u16(d2) if c2 else None
    v1, v2 = _u16(w1), _u16(w2) if c2 else None
    _lib.check(lib.lp_head_fused_pack(a1.ctypes.data, b1.ctypes.data, _addr(a2), _addr(b2) if c2 else None, v1.ctypes.data,
                                      _addr(v2), c1, c2, co, dwc.ctypes.data, bdc.ctypes.data, pwc.ctypes.data),
               "head_fused_pack")
    return dwc.view(F16), bdc, pwc.view(F16)


CASES = []


def _add(*a, **kw):
    CASES.append(Case(*a, **kw))


# ---------------------------------------------------------------- stem
# (n, h, w, fp32, odd element offset of x): the vector path (fp16 W % 8 == 0, fp32 W % 4 == 0, aligned base), the
# generic path (W % 8 == 4, W % 4 == 2, the base one element off), H = W = 2
STEM = [(2, 36, 128, False, False), (2, 36, 128, True, False), (2, 52, 100, False, False), (2, 52, 98, True, False),
        (1, 36, 128, False, True), (1, 36, 128, True, True), (3, 2, 2, False, False)]


def _stem_case(n, h, w, fp32, odd, flip, raw):
    def inputs():
        rng = _rng("stem", n, h, w, fp32, odd, flip, raw)
        x = rng.standard_normal((n, 3, h, w)).astype(F32 if fp32 else F16)
        wt = (rng.standard_normal((32, 27)) * 0.3).astype(F16)
        b = (rng.standard_normal(32) * 0.2).astype(F32)
        return x, wt, b
    inputs = functools.lru_cache(None)(inputs)

    def run(A):
        x, wt, b = inputs()
        xd = A.inp("x", x, skew=SKEW + x.itemsize if odd else None)
        wd = A.inp("w", wt)
        y = A.out("y", (n, h // 2, w // 2, 32), F16)
        if raw:
            return [_L().lp_stem_conv3x3_s2_act(xd.data_ptr(), int(fp32), flip, wd.data_ptr(), None, y.data_ptr(), n,
                                                h, w, _lib.ACT_NONE, _s())]
        bd = A.inp("bias", b)
        return [_L().lp_stem_conv3x3_s2(xd.data_ptr(), int(fp32), flip, wd.data_ptr(), bd.data_ptr(), y.data_ptr(), n,
                                        h, w, _s())]

    def ref():
        x, wt, b = inputs()
        return {"y": bte.stem_raw(x, wt, flip) if raw else cr.stem_conv(x, wt, b, flip)}
    name = "lp_stem_conv3x3_s2_act" if raw else "lp_stem_conv3x3_s2"
    _add("%s-n%d-%dx%d-%s%s-flip%d" % (name[3:], n, h, w, "fp32" if fp32 else "fp16", "-odd" if odd else "", flip),
         [name], run, ref)


for _c in STEM:
    for _f in (0, 1):
        _stem_case(*_c, _f, False)
for _c in (STEM[0], STEM[3], STEM[5]):
    _stem_case(*_c, 1, True)


# (n, h, w, C0, fp32 x, flip): ragged tile rows, Wo = 18 with C0 = 8, a 1 x 2 output
STEM_FUSED = [(2, 36, 64, 16, False, 0), (1, 52, 36, 8, True, 1), (3, 2, 4, 8, False, 1), (1, 36, 64, 32, True, 0)]


def _stem_fused_case(n, h, w, c0, fp32, flip):
    ho, wo = h // 2, w // 2

    @functools.lru_cache(None)
    def inputs():
        rng = _rng("stem_fused", n, h, w, c0)
        x = rng.standard_normal((n, 3, h, w)).astype(F32)
        w1 = (rng.standard_normal((32, 27)) * 0.3).astype(F16)
        b1 = (rng.standard_normal(32) * 0.2).astype(F32)
        wdw = (rng.standard_normal((9, 32)) * 0.3).astype(F16)
        bdw = (rng.standard_normal(32) * 0.2).astype(F32)
        w3 = (rng.standard_normal((c0, 32)) / 32 ** 0.5).astype(F16)
        b3 = (rng.standard_normal(c0) * 0.1).astype(F32)
        w1p = np.zeros((32, 64), F16)
        w1p[:, :27] = w1
        return (x if fp32 else x.astype(F16)), w1p, b1, wdw, bdw, w3, b3

    def run(A):
        x, w1p, b1, wdw, bdw, w3, b3 = inputs()
        w3k, b3k = pack_pw(w3, b3)
        t = [A.inp("x", x), A.inp("w1p", w1p), A.inp("b1", b1), A.inp("w_dw", wdw), A.inp("b_dw", bdw),
             A.inp("w_pw", w3k), A.inp("b_pw", b3k)]
        y = A.out("y", (n, ho, wo, c0), F16)
        return [_L().lp_stem_fused_f16(t[0].data_ptr(), int(fp32), flip, *[v.data_ptr() for v in t[1:]], y.data_ptr(),
                                       n, h, w, c0, _s())]

    def ref():
        # the chain lp_stem_fused_f16 replaces (test_gpu_stem_deconv_exact), each part by its emulator
        x, w1p, b1, wdw, bdw, w3, b3 = inputs()
        m = n * ho * wo
        e = me.pw1x1(cr.stem_im2col(x.astype(F16), flip), w1p[:, :32], b1, None, de.ACT_RELU6)
        d = de.dwconv(e.reshape(n, ho, wo, 32), wdw, bdw, 3, 1, de.ACT_RELU6, 2)
        return {"y": me.pw1x1(d.reshape(m, 32), w3, b3).reshape(n, ho, wo, c0)}
    _add("stem_fused-n%d-%dx%d-c%d-%s-flip%d" % (n, h, w, c0, "fp32" if fp32 else "fp16", flip), ["lp_stem_fused_f16"],
         run, ref)


for _c in STEM_FUSED:
    _stem_fused_case(*_c)


# ---------------------------------------------------------------- depthwise
def _dw_shape(k, s, i):
    """ragged against the tiles with a partial slab, W < 8 with W % 4 != 0, the widest channel count, the smallest map"""
    if s == 1:
        return [(3, 40, 37, 45), (3, 8, 9, 6), (1, 720, 9, 13), (3, 24, 5, 5)][i % 4]
    return [(3, 40, 38, 42), (3, 8, 6, 10), (1, 720, 10, 14), (3, 24, 2, 2)][i % 4]


def _dw_case(k, s, prec, i):
    n, c, h, w = _dw_shape(k, s, i)
    act = i % 3
    kind = ("relu6", "signed", "tiny")[i % 3]
    narrow = i % 3 == 1          # y and w at the 4-byte alignment the entry point documents for them

    @functools.lru_cache(None)
    def inputs():
        return de.make_inputs(n, c, h, w, k, kind, 31 * i + k)

    def run(A):
        x, wt, b = inputs()
        xd, wd, bd = A.inp("x", x), A.inp("w", wt, skew=4 if narrow else None), A.inp("bias", b)
        y = A.out("y", (n, h // s, w // s, c), F16, skew=4 if narrow else None)
        return [_L().lp_dwconv_f16(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), y.data_ptr(), n, c, h, w, k, s, act,
                                   _s())]

    def ref():
        x, wt, b = inputs()
        return {"y": de.dwconv(x, wt, b, k, s, act, prec)}
    _add("dwconv-k%d-s%d-prec%d-n%d-c%d-%dx%d-act%d%s" % (k, s, prec, n, c, h, w, act, "-align4" if narrow else ""),
         ["lp_dwconv_f16"], run, ref, prec=prec)


for _i, (_k, _st, _pr) in enumerate([(k, s, p) for k in (3, 5, 7) for s in (1, 2) for p in (0, 1, 2)]):
    _dw_case(_k, _st, _pr, _i)


# ---------------------------------------------------------------- pointwise GEMM
# (m, k, n, act, residual): one row and K = 8; M and N tails with a second K block; N = 168 in two chunks; streaming
# weights; the widest N
PW = [(1, 8, 8, 0, False), (65, 72, 24, 1, True), (65, 72, 168, 0, True), (63, 448, 256, 0, True),
      (65, 960, 160, 2, True), (300, 32, 1024, 2, False)]


def pw_inputs(m, k, n, res, seed):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((m, k)).astype(F16)
    wt = (rng.standard_normal((n, k)) / k ** 0.5).astype(F16)
    b = (rng.standard_normal(n) * 0.3).astype(F32)
    r = rng.standard_normal((m, n)).astype(F16) if res else None
    return a, wt, b, r


def _pw_case(m, k, n, act, res):
    inputs = functools.lru_cache(None)(lambda: pw_inputs(m, k, n, res, m + 7 * k + n))

    def run(A):
        a, wt, b, r = inputs()
        wp, bp = pack_pw(wt, b)
        ad, wd, bd = A.inp("a", a), A.inp("w", wp), A.inp("bias", bp)
        rd = A.inp("residual", r) if res else None
        out = A.out("out", (m, n), F16)
        return [_L().lp_pw1x1_f16(ad.data_ptr(), wd.data_ptr(), bd.data_ptr(), _p(rd), out.data_ptr(), m, k, n, act,
                                  _s())]

    def ref():
        a, wt, b, r = inputs()
        return {"out": me.pw1x1(a, wt, b, r, act)}
    _add("pw1x1-m%d-k%d-n%d-act%d-res%d" % (m, k, n, act, res), ["lp_pw1x1_f16"], run, ref)


for _c in PW:
    _pw_case(*_c)


# ---------------------------------------------------------------- fused blocks
# (n, h, w, Ce, Co, residual): ragged tiles with Co = 64 (dw_project_kernel), the wide kernel with Co = 120 and 160
DW7P = [(2, 37, 45, 40, 64, True), (1, 8, 16, 288, 120, True), (3, 20, 40, 96, 160, False)]


def _dw7p_case(n, h, w, ce, co, res):
    @functools.lru_cache(None)
    def inputs():
        rng = np.random.default_rng(ce * 3 + co + h + n)
        x, wd, bd = de.make_inputs(n, ce, h, w, 7, "relu6", ce + h)
        wp = (rng.standard_normal((co, ce)) / ce ** 0.5).astype(F16)
        bp = (rng.standard_normal(co) * 0.1).astype(F32)
        r = rng.standard_normal((n, h, w, co)).astype(F16) if res else None
        return x, wd, bd, wp, bp, r

    def run(A):
        x, wd, bd, wp, bp, r = inputs()
        wk, bk = pack_pw(wp, bp)
        t = [A.inp("x", x), A.inp("w_dw", wd), A.inp("b_dw", bd), A.inp("w_proj", wk), A.inp("b_proj", bk)]
        rd = A.inp("residual", r) if res else None
        out = A.out("out", (n, h, w, co), F16)
        return [_L().lp_dw7_project_f16(*[v.data_ptr() for v in t], _p(rd), out.data_ptr(), n, h, w, ce, co, _s())]

    def ref():
        x, wd, bd, wp, bp, r = inputs()
        d = de.dwconv(x, wd, bd, 7, 1, de.ACT_RELU6, 2).reshape(-1, ce)
        return {"out": me.pw1x1(d, wp, bp, None if r is None else r.reshape(-1, co)).reshape(n, h, w, co)}
    _add("dw7_project-n%d-%dx%d-ce%d-co%d-res%d" % (n, h, w, ce, co, res), ["lp_dw7_project_f16"], run, ref)


for _c in DW7P:
    _dw7p_case(*_c)


# (n, h, w, Cin, Ce, Co, stride): stride 1 ragged in both axes and the widest stage; stride 2 ragged, a 2 x 3 output,
# Cin = 8 with a partial slab, three projection chunks
BLOCKS = [(3, 40, 52, 16, 96, 16, 1), (2, 20, 28, 48, 288, 48, 1), (3, 40, 52, 16, 96, 16, 2), (2, 4, 6, 16, 96, 16, 2),
          (2, 16, 20, 8, 48, 16, 2), (1, 24, 32, 16, 96, 40, 2)]


def _block_case(n, h, w, cin, ce, co, stride):
    ho, wo = h // stride, w // stride

    @functools.lru_cache(None)
    def inputs():
        rng = np.random.default_rng(cin * 5 + ce * 3 + co + h + w + n)
        x = rng.standard_normal((n, h, w, cin)).astype(F16)
        we = (rng.standard_normal((ce, cin)) / cin ** 0.5).astype(F16)
        be = (rng.standard_normal(ce) * 0.2).astype(F32)
        _, wd, bd = de.make_inputs(1, ce, 1, 1, 7, "relu6", ce + h)
        wp = (rng.standard_normal((co, ce)) / ce ** 0.5).astype(F16)
        bp = (rng.standard_normal(co) * 0.1).astype(F32)
        return x, we, be, wd, bd, wp, bp

    def run(A):
        x, we, be, wd, bd, wp, bp = inputs()
        wk, bk = pack_pw(wp, bp)
        t = [A.inp("x", x), A.inp("w_exp", pack_wexp(we)), A.inp("b_exp", be), A.inp("w_dw", wd), A.inp("b_dw", bd),
             A.inp("w_proj", wk), A.inp("b_proj", bk)]
        out = A.out("out", (n, ho, wo, co), F16)
        p = [v.data_ptr() for v in t]
        if stride == 1:
            return [_L().lp_block_s1_f16(*p, 1, out.data_ptr(), n, h, w, cin, ce, co, _s())]
        return [_L().lp_block_s2_f16(*p, out.data_ptr(), n, h, w, cin, ce, co, _s())]

    def ref():
        x, we, be, wd, bd, wp, bp = inputs()
        e = me.pw1x1(x.reshape(-1, cin), we, be, None, de.ACT_RELU6).reshape(n, h, w, ce)
        d = de.dwconv(e, wd, bd, 7, stride, de.ACT_RELU6, 2).reshape(-1, ce)
        r = x.reshape(-1, cin) if stride == 1 else None
        return {"out": me.pw1x1(d, wp, bp, r).reshape(n, ho, wo, co)}
    name = "lp_block_s%d_f16" % stride
    _add("block_s%d-n%d-%dx%d-cin%d-ce%d-co%d" % (stride, n, h, w, cin, ce, co), [name], run, ref)


for _c in BLOCKS:
    _block_case(*_c)


# ---------------------------------------------------------------- fusion deconv
# (n, h, w, Cr, Cw, Co): the row kernel (W = 64 exactly, a partial strip, K = 64 with Co = 32), the tiled kernel
# (W = 63, half-filled K slices, a second K block of 8 channels), one branch on either kernel
DECONV = [(1, 3, 64, 16, 16, 16), (1, 2, 200, 24, 16, 8), (2, 4, 96, 40, 24, 32), (2, 12, 63, 16, 16, 16),
          (2, 8, 16, 40, 24, 40), (1, 20, 24, 72, 40, 64), (1, 3, 64, 32, 0, 16), (2, 8, 16, 40, 0, 24)]


def _deconv_case(n, h, w, cr_, cw, co, act):
    rows = cr.uses_rows_kernel(cr_, cw, co, w)
    inputs = functools.lru_cache(None)(lambda: cr.deconv_inputs(n, h, w, cr_, cw, co, 3 * n + h + w + cr_ + cw + co))

    def run(A):
        xr, xw, wr, ww, b = inputs()
        wp, bp = pack_deconv(wr, ww, b, cr_, cw, co)
        rd = A.inp("refined", xr)
        rwd = A.inp("raw", xw) if cw else None
        wd, bd = A.inp("w", wp), A.inp("bias", bp)
        out = A.out("out", (n, 2 * h, 2 * w, co), F16)
        if act is None:
            return [_L().lp_fusion_deconv_f16(rd.data_ptr(), _p(rwd), wd.data_ptr(), bd.data_ptr(), out.data_ptr(), n, h,
                                              w, cr_, cw, co, _s())]
        return [_L().lp_fusion_deconv_act_f16(rd.data_ptr(), _p(rwd), wd.data_ptr(), bd.data_ptr(), out.data_ptr(), n,
                                              h, w, cr_, cw, co, act, _s())]

    def ref():
        xr, xw, wr, ww, b = inputs()
        if act == _lib.ACT_NONE:
            return {"out": bte.deconv_raw(xr, xw, wr, ww, b)}
        if cw == 0:
            return {"out": se.deconv_single(xr, wr, b, rows)}
        return {"out": me.deconv(xr, xw, wr, ww, b, rows)}
    name = "lp_fusion_deconv_f16" if act is None else "lp_fusion_deconv_act_f16"
    _add("%s-%s-n%d-%dx%d-cr%d-cw%d-co%d" % (name[3:-4], "rows" if rows else "tiled", n, h, w, cr_, cw, co), [name],
         run, ref)


for _c in DECONV:
    _deconv_case(*_c, None)
for _c in (DECONV[1], DECONV[4]):
    _deconv_case(*_c, _lib.ACT_NONE)


# ---------------------------------------------------------------- heads
# (n, h, w, C1, C2, Co, fp32): Co 17 and 34 (odd, and two chunks), partial slices, one branch
HEADS = [(2, 16, 16, 16, 16, 17, True), (1, 24, 40, 32, 32, 34, False), (2, 5, 7, 8, 16, 30, True),
         (2, 12, 20, 24, 0, 17, False)]


def _head_case(n, h, w, c1, c2, co, fp32):
    p = n * h * w
    odt = F32 if fp32 else F16

    @functools.lru_cache(None)
    def inputs():
        rng = np.random.default_rng(n + h + w + c1 + c2 + co)
        a1 = np.maximum(rng.standard_normal((n, h, w, c1)), 0).astype(F16)
        a2 = np.maximum(rng.standard_normal((n, h, w, c2)), 0).astype(F16)
        w1 = (rng.standard_normal((co, c1)) / c1 ** 0.5).astype(F16)
        w2 = (rng.standard_normal((co, c2)) / max(c2, 1) ** 0.5).astype(F16)
        return a1, a2, w1, w2

    def run(A):
        a1, a2, w1, w2 = inputs()
        d1 = A.inp("a1", a1)
        d2 = A.inp("a2", a2) if c2 else None
        wd = A.inp("w", pack_head(w1, w2, c1, c2, co))
        out = A.out("out", (n, co, h, w), odt)
        return [_L().lp_head_pw_dual_f16(d1.data_ptr(), _p(d2), wd.data_ptr(), out.data_ptr(), int(fp32), n, h, w, c1,
                                         c2, co, _s())]

    def ref():
        a1, a2, w1, w2 = inputs()
        if c2:
            r = me.head_dual(a1.reshape(p, c1), a2.reshape(p, c2), w1, w2, fp32)
        else:
            r = se.head_single(a1.reshape(p, c1), w1, fp32)
        return {"out": r.reshape(n, h, w, co).transpose(0, 3, 1, 2)}
    _add("head_pw_dual-n%d-%dx%d-c1_%d-c2_%d-co%d-%s" % (n, h, w, c1, c2, co, "fp32" if fp32 else "fp16"),
         ["lp_head_pw_dual_f16"], run, ref)


for _c in HEADS:
    _head_case(*_c)


HEADS_FUSED = [(2, 20, 36, 24, 16, 17, True), (1, 37, 45, 72, 40, 34, False), (1, 16, 24, 40, 0, 17, True)]


def _head_fused_case(n, h, w, c1, c2, co, fp32):
    p = n * h * w
    odt = F32 if fp32 else F16

    @functools.lru_cache(None)
    def inputs():
        seed = c1 * 7 + c2 + co
        rng = np.random.default_rng(seed)
        x1, d1, b1 = de.make_inputs(n, c1, h, w, 5, "signed", seed + 1)
        if c2:
            x2, d2, b2 = de.make_inputs(n, c2, h, w, 5, "signed", seed + 2)
        else:
            x2 = d2 = b2 = None
        w1 = (rng.standard_normal((co, c1)) / c1 ** 0.5).astype(F16)
        w2 = (rng.standard_normal((co, c2)) / c2 ** 0.5).astype(F16) if c2 else None
        return x1, d1, b1, x2, d2, b2, w1, w2

    def run(A):
        x1, d1, b1, x2, d2, b2, w1, w2 = inputs()
        dwc, bdc, pwc = pack_head_fused(d1, b1, d2, b2, w1, w2, c1, c2, co)
        s1 = A.inp("a1", x1)
        s2 = A.inp("a2", x2) if c2 else None
        t = [A.inp("dw_cat", dwc), A.inp("bdw_cat", bdc), A.inp("pw", pwc)]
        out = A.out("out", (n, co, h, w), odt)
        return [_L().lp_head_fused_f16(s1.data_ptr(), _p(s2), *[v.data_ptr() for v in t], out.data_ptr(), int(fp32), n,
                                       h, w, c1, c2, co, _s())]

    def ref():
        # lp_dwconv_f16 (k5, ReLU, fp32 taps) then lp_head_pw_dual_f16, each by its emulator (test_gpu_dw_exact)
        x1, d1, b1, x2, d2, b2, w1, w2 = inputs()
        t1 = de.dwconv(x1, d1, b1, 5, 1, de.ACT_RELU, 0).reshape(p, c1)
        if c2:
            t2 = de.dwconv(x2, d2, b2, 5, 1, de.ACT_RELU, 0).reshape(p, c2)
            r = me.head_dual(t1, t2, w1, w2, fp32)
        else:
            r = se.head_single(t1, w1, fp32)
        return {"out": r.reshape(n, h, w, co).transpose(0, 3, 1, 2)}
    _add("head_fused-n%d-%dx%d-c1_%d-c2_%d-co%d-%s" % (n, h, w, c1, c2, co, "fp32" if fp32 else "fp16"),
         ["lp_head_fused_f16"], run, ref)


for _c in HEADS_FUSED:
    _head_fused_case(*_c)


# ---------------------------------------------------------------- train-mode BatchNorm
BN = [(2, 720), (777, 24), (2049, 200)]


def _bn_inputs(m, c):
    rng = np.random.default_rng(m * 3 + c)
    x = (rng.standard_normal((m, c)) * 2 + 0.5).astype(F16)
    gamma = rng.uniform(0.5, 1.5, c).astype(F32)
    beta = rng.standard_normal(c).astype(F32)
    rmean = rng.standard_normal(c).astype(F32)
    rvar = rng.uniform(0.5, 2, c).astype(F32)
    res = rng.standard_normal((m, c)).astype(F16)
    return x, gamma, beta, rmean, rvar, res


def _bn_stats_case(m, c):
    inputs = functools.lru_cache(None)(lambda: _bn_inputs(m, c))

    def run(A):
        x, gamma, beta, rmean, rvar, _ = inputs()
        xd = A.inp("x", x)
        t = [A.inp("gamma", gamma), A.inp("beta", beta), A.inp("running_mean", rmean), A.inp("running_var", rvar)]
        o = [A.out(k, (c,), F32) for k in ("scale", "shift", "new_mean", "new_var")]
        nf = A.out("nonfinite", (1,), I32, init=np.zeros(1, I32))
        nb = _L().lp_bn_stats_workspace_bytes(m, c)
        ws = A.ws("workspace", nb, skew=16)
        return [_L().lp_bn_stats_f16(xd.data_ptr(), m, c, *[v.data_ptr() for v in t], 0.1, 1e-5,
                                     *[v.data_ptr() for v in o], nf.data_ptr(), ws.data_ptr(), nb, _s())]

    def ref():
        x, gamma, beta, rmean, rvar, _ = inputs()
        scale, shift, nm, nv, bad = bte.stats(x, gamma, beta, rmean, rvar, 0.1, 1e-5)
        return {"scale": scale, "shift": shift, "new_mean": nm, "new_var": nv, "nonfinite": np.array([int(bad)], I32)}
    _add("bn_stats-m%d-c%d" % (m, c), ["lp_bn_stats_f16"], run, ref)


def _bn_apply_case(m, c, act, res, inplace):
    @functools.lru_cache(None)
    def inputs():
        x, gamma, beta, rmean, rvar, r = _bn_inputs(m, c)
        scale, shift = bte.stats(x, gamma, beta, rmean, rvar, 0.1, 1e-5)[:2]
        return x, scale, shift, r

    def run(A):
        x, scale, shift, r = inputs()
        if inplace:                                   # y == x: the in-place form the header allows
            y = xd = A.out("y", x.shape, F16, init=x)
        else:
            xd, y = A.inp("x", x), A.out("y", x.shape, F16)
        sd, hd = A.inp("scale", scale), A.inp("shift", shift)
        rd = A.inp("residual", r) if res else None
        return [_L().lp_bn_apply_f16(xd.data_ptr(), sd.data_ptr(), hd.data_ptr(), _p(rd), y.data_ptr(), m, c, act,
                                     _s())]

    def ref():
        x, scale, shift, r = inputs()
        return {"y": bte.apply(x, scale, shift, act, r if res else None)}
    _add("bn_apply-m%d-c%d-act%d-res%d%s" % (m, c, act, res, "-inplace" if inplace else ""), ["lp_bn_apply_f16"], run,
         ref)


for _c in BN:
    _bn_stats_case(*_c)
_bn_apply_case(777, 24, 2, True, False)
_bn_apply_case(2049, 200, 1, False, False)
_bn_apply_case(2, 720, 0, True, True)


# ---------------------------------------------------------------- pre-processing: the warp
def _warp_golden(i):
    from litepose_b200.lib.utils import transforms as T
    from oracle.make_golden_transforms import PRE_CASES, pre_image
    import os
    seed, h, w, size = PRE_CASES[i]
    img = pre_image(seed, h, w)
    (wr, hr), center, scale = T.get_multi_scale_size(img, size, 1.0, 1.0)
    minv = T.invert_affine(T.get_affine_transform(center, scale, 0, (wr, hr)))
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "transforms.npz"))
    pre = "p%02d_" % i
    return img, np.asarray(minv, F64).reshape(6), (wr, hr), {0: g[pre + "resized"], 1: g[pre + "tensor"],
                                                             2: g[pre + "tensor"].astype(F16)}


_MEAN = np.array([0.485, 0.456, 0.406], F32)       # valid.py:181-184 (the goldens' normalisation)
_STD = np.array([0.229, 0.224, 0.225], F32)
_OUT_DT = {0: U8, 1: F32, 2: F16}


def _warp_case(i, mode, odd):
    def run(A):
        img, minv, (wr, hr), _ = _warp_golden(i)
        h, w = img.shape[:2]
        src = A.inp("img", np.stack([img, img]), skew=SKEW + 1 if odd else None)
        m = A.inp("minv", np.stack([minv, minv]))
        shape = (2, hr, wr, 3) if mode == 0 else (2, 3, hr, wr)
        out = A.out("out", shape, _OUT_DT[mode])
        return [_L().lp_warp_affine_normalize_u8(src.data_ptr(), 2, h, w, m.data_ptr(), wr, hr, _MEAN.ctypes.data,
                                                 _STD.ctypes.data, out.data_ptr(), mode, _s())]

    def ref():
        g = _warp_golden(i)[3][mode]
        return {"out": np.stack([g, g])}
    _add("warp-p%d-mode%d%s" % (i, mode, "-odd" if odd else ""), ["lp_warp_affine_normalize_u8"], run, ref)


def _warp_ragged_case(idx, mode, odd):
    from litepose_b200.mixed import WARP_DESC

    def layout():
        gs = [_warp_golden(i) for i in idx]
        desc = np.zeros(len(idx), WARP_DESC)
        src, so, do = [], 0, 0
        for k, (img, minv, (wr, hr), _) in enumerate(gs):
            desc[k]["src_offset"], desc[k]["src_h"], desc[k]["src_w"] = so, img.shape[0], img.shape[1]
            desc[k]["minv"], desc[k]["dst_offset"], desc[k]["out_h"], desc[k]["out_w"] = minv, do, hr, wr
            src.append(img.reshape(-1))
            so += img.size
            do += hr * wr * 3
        return gs, desc, np.concatenate(src), do

    def run(A):
        gs, desc, src, total = layout()
        s = A.inp("img", src, skew=SKEW + 1 if odd else None)
        d = A.desc("desc", desc)
        out = A.out("out", (total,), _OUT_DT[mode])
        mw, mh = max(g[2][0] for g in gs), max(g[2][1] for g in gs)
        return [_L().lp_warp_affine_normalize_ragged_u8(s.data_ptr(), len(idx), d.data_ptr(), mw, mh, _MEAN.ctypes.data,
                                                        _STD.ctypes.data, out.data_ptr(), mode, _s())]

    def ref():
        gs = layout()[0]
        return {"out": np.concatenate([g[3][mode].reshape(-1) for g in gs])}
    _add("warp_ragged-%s-mode%d%s" % ("_".join(map(str, idx)), mode, "-odd" if odd else ""),
         ["lp_warp_affine_normalize_ragged_u8"], run, ref)


_warp_case(0, 0, False)
_warp_case(3, 1, True)
_warp_case(1, 2, False)
_warp_case(0, 0, True)
_warp_ragged_case((0, 3, 2), 0, True)
_warp_ragged_case((1, 4), 1, False)
_warp_ragged_case((3, 0), 2, False)


# ---------------------------------------------------------------- glue (input side; the outputs have guards already)
GLUE = ["x4_16", "generic_61x93", "ms_1_2", "unproj_shared_tag", "generic_no_tag"]


def _glue_case(name):
    case = next(c for c in ge.CASES if c["name"] == name)
    J, N, Hd, Wd = case["J"], case["N"], case["Hd"], case["Wd"]
    T = 2 if case["flip"] else 1
    tshape = (N, 1 if case["tag_shared"] else J, Hd, Wd, T)
    inputs = functools.lru_cache(None)(lambda: ge.case_inputs(case, "randn", 17))

    def run(A):
        det = A.out("det", (N, J, Hd, Wd), F32)
        tag = A.out("tag", tshape, F32)
        fidx = A.inp("flip_index", np.array(ge.flip_index(J), I32))          # read for the J joints written
        rcs = []
        for ci, ((h, w, acc, div, wt), arrs) in enumerate(zip(case["calls"], inputs())):
            o0, o1, f0, f1 = [None if a is None else A.inp("%s_%d" % (k, ci), a)
                              for k, a in zip(("o0", "o1", "f0", "f1"), arrs)]
            if case["entry"] == "f32":
                rcs.append(_L().lp_glue_f32(o0.data_ptr(), o1.data_ptr(), _p(f0), _p(f1), fidx.data_ptr(), N, J, h, w,
                                            int(case["flip"]), Hd, Wd, det.data_ptr(), tag.data_ptr(), _s()))
            else:
                rcs.append(_L().lp_glue_scale_f32(o0.data_ptr(), o1.data_ptr(), _p(f0), _p(f1), fidx.data_ptr(), N, J,
                                                  case["Jm"], int(case["tag_shared"]), h, w, int(case["flip"]), Hd, Wd,
                                                  int(acc), div, det.data_ptr(), tag.data_ptr() if wt else None, _s()))
        return rcs

    def ref():
        det, tag = ge.run_case(case, inputs())
        t = sentinel_array(tshape, F32)
        if tag is not None:                    # the tag planes a call does not write stay NaN in the emulation
            t = np.where(np.isnan(tag), t, tag).astype(F32)
        return {"det": det, "tag": t}
    entry = "lp_glue_f32" if case["entry"] == "f32" else "lp_glue_scale_f32"
    _add("glue-%s" % name, [entry], run, ref, untouched=("tag",))


for _g in GLUE:
    _glue_case(_g)


# ---------------------------------------------------------------- the parser chain
J, K, TT, NMS = 14, 30, 2, 5
DET_THR, TAG_THR = 0.1, 1.0
PCAP = J * K
JOINT_ORDER = np.array([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13], I32)


@functools.lru_cache(None)
def parser_maps(n, h, w, seed):
    from litepose_b200 import synth
    det, tag = synth.plant_crowd_batch(n, J, h, w, TT, num_people=4, seed=seed)
    return np.ascontiguousarray(det, F32), np.ascontiguousarray(tag, F32)


@functools.lru_cache(None)
def ragged_maps(sizes, seed):
    """det / tag arenas of differently sized maps, host hw [N,2] and the MAP_DESC descriptors"""
    from litepose_b200.mixed import MAP_DESC
    ds, ts = [], []
    desc = np.zeros(len(sizes), MAP_DESC)
    do = to = 0
    for k, (h, w) in enumerate(sizes):
        d, t = parser_maps(1, h, w, seed + k)
        desc[k]["h"], desc[k]["w"], desc[k]["det_offset"], desc[k]["tag_offset"] = h, w, do, to
        ds.append(d.reshape(-1))
        ts.append(t.reshape(-1))
        do += d.size
        to += t.size
    return np.concatenate(ds), np.concatenate(ts), np.array(sizes, I32).reshape(-1, 2), desc


def _topk(A, det, tag, n, h, w, odd=False):
    d = A.inp("det", det, skew=SKEW + 4 if odd else None)
    t = A.inp("tag", tag, skew=SKEW + 4 if odd else None)
    val, ind, tk = A.out("val_k", (n, J, K), F32), A.out("ind_k", (n, J, K), I32), A.out("tag_k", (n, J, K, TT), F32)
    nb = _L().lp_nms_topk_workspace_bytes(n, J, h, w, K)
    ws = A.ws("ws_topk", nb)
    return [_L().lp_nms_topk_f32(d.data_ptr(), t.data_ptr(), n, J, h, w, TT, NMS, K, DET_THR, val.data_ptr(),
                                 ind.data_ptr(), tk.data_ptr(), ws.data_ptr(), nb, _s())]


def _topk_ragged(A, sizes, seed, odd=False):
    det, tag, hw, desc = ragged_maps(sizes, seed)
    n = len(sizes)
    d = A.inp("det", det, skew=SKEW + 4 if odd else None)
    t = A.inp("tag", tag, skew=SKEW + 4 if odd else None)
    dd = A.desc("desc", desc)
    val, ind, tk = A.out("val_k", (n, J, K), F32), A.out("ind_k", (n, J, K), I32), A.out("tag_k", (n, J, K, TT), F32)
    nb = _L().lp_nms_topk_ragged_workspace_bytes(n, hw.ctypes.data, J, K)
    ws = A.ws("ws_topk", nb)
    return [_L().lp_nms_topk_ragged_f32(d.data_ptr(), t.data_ptr(), n, hw.ctypes.data, dd.data_ptr(), J, TT, NMS, K,
                                        DET_THR, val.data_ptr(), ind.data_ptr(), tk.data_ptr(), ws.data_ptr(), nb,
                                        _s())]


def _plain(run):
    """the outputs of ``run`` on plain tensors"""
    from footprint_util import Plain
    A = Plain()
    rcs = run(A)
    assert all(rc == _lib.LP_OK for rc in rcs), rcs
    return A.outputs()


def _match(A, tk, n, w, desc=None):
    val, ind, tg = A.inp("val_k", tk["val_k"]), A.inp("ind_k", tk["ind_k"]), A.inp("tag_k", tk["tag_k"])
    jo = A.inp("joint_order", JOINT_ORDER)
    ans, num = A.out("ans", (n, PCAP, J, 3 + TT), F32), A.out("num", (n,), I32)
    nb = _L().lp_tag_match_workspace_bytes(n, J, K, TT, PCAP)
    ws = A.ws("ws_match", nb)
    common = (jo.data_ptr(), DET_THR, TAG_THR, 1, 0, K, PCAP, ans.data_ptr(), num.data_ptr(), ws.data_ptr(), nb, _s())
    if desc is None:
        return [_L().lp_tag_match_f32(val.data_ptr(), ind.data_ptr(), tg.data_ptr(), n, J, K, TT, w, *common)]
    dd = A.desc("desc", desc)
    return [_L().lp_tag_match_ragged_f32(val.data_ptr(), ind.data_ptr(), tg.data_ptr(), n, J, K, TT, dd.data_ptr(),
                                         *common)]


def _refine(A, det, tag, mt, n, h, w, hw=None, desc=None):
    d, t = A.inp("det", det), A.inp("tag", tag)
    num = A.inp("num", mt["num"])
    ans = A.out("ans", mt["ans"].shape, F32, init=mt["ans"])
    sc = A.out("scores", (n, PCAP), F32)
    nb = _L().lp_adjust_refine_workspace_bytes(n, J, PCAP)
    ws = A.ws("ws_ref", nb)
    tail = (PCAP, ans.data_ptr(), num.data_ptr(), sc.data_ptr(), 1, 1, ws.data_ptr(), nb, _s())
    if desc is None:
        return [_L().lp_adjust_refine_f32(d.data_ptr(), t.data_ptr(), n, J, h, w, TT, *tail)]
    dd = A.desc("desc", desc)
    return [_L().lp_adjust_refine_ragged_f32(d.data_ptr(), t.data_ptr(), n, hw.ctypes.data, dd.data_ptr(), J, TT,
                                             *tail)]


# (n, h, w, odd element offset of det / tag): W % 4 == 0 (vector loads) and W % 4 != 0, the base 4 bytes off
PARSER = [(2, 64, 96, False), (1, 40, 90, False), (2, 64, 96, True)]
RAGGED = [((64, 96), (48, 60), (33, 80)), ((40, 90), (64, 64))]


def _parser_cases(n, h, w, odd):
    det, tag = parser_maps(n, h, w, h + w)
    tk = functools.lru_cache(None)(lambda: _plain(lambda A: _topk(A, det, tag, n, h, w)))
    mt = functools.lru_cache(None)(lambda: _plain(lambda A: _match(A, tk(), n, w)))
    sfx = "n%d-%dx%d%s" % (n, h, w, "-odd" if odd else "")
    _add("nms_topk-" + sfx, ["lp_nms_topk_f32"], lambda A: _topk(A, det, tag, n, h, w, odd))
    if not odd:
        _add("tag_match-" + sfx, ["lp_tag_match_f32"], lambda A: _match(A, tk(), n, w), untouched=("ans",))
        _add("adjust_refine-" + sfx, ["lp_adjust_refine_f32"], lambda A: _refine(A, det, tag, mt(), n, h, w),
             untouched=("ans", "scores"))


def _parser_ragged_cases(sizes, odd):
    det, tag, hw, desc = ragged_maps(sizes, 7)
    n = len(sizes)
    tk = functools.lru_cache(None)(lambda: _plain(lambda A: _topk_ragged(A, sizes, 7)))
    mt = functools.lru_cache(None)(lambda: _plain(lambda A: _match(A, tk(), n, 0, desc)))
    sfx = "_".join("%dx%d" % s for s in sizes) + ("-odd" if odd else "")
    _add("nms_topk_ragged-" + sfx, ["lp_nms_topk_ragged_f32"], lambda A: _topk_ragged(A, sizes, 7, odd))
    if not odd:
        _add("tag_match_ragged-" + sfx, ["lp_tag_match_ragged_f32"], lambda A: _match(A, tk(), n, 0, desc),
             untouched=("ans",))
        _add("adjust_refine_ragged-" + sfx, ["lp_adjust_refine_ragged_f32"],
             lambda A: _refine(A, det, tag, mt(), n, 0, 0, hw, desc), untouched=("ans", "scores"))


for _c in PARSER:
    _parser_cases(*_c)
for _c in RAGGED:
    _parser_ragged_cases(_c, False)
_parser_ragged_cases(RAGGED[0], True)


# ---------------------------------------------------------------- fast grouping
FM, FTHR, FWIN, FTAG = 10, 0.1, 3, 1.0


def _peaks(A, n, h, w):
    det, tag = parser_maps(n, h, w, 5 * h + w)
    inp, tm = A.inp("input", det), A.inp("tmap", np.ascontiguousarray(tag[..., 0]))
    o = _peak_outs(A, n)
    return [_L().lp_find_peaks_f32(inp.data_ptr(), tm.data_ptr(), n, J, h, w, FM, FTHR, FWIN, *[t.data_ptr() for t in o],
                                   _s())]


def _peak_outs(A, n):
    return [A.out("count", (n, J), I32), A.out("val", (n, J, FM), F32), A.out("tag", (n, J, FM), F32),
            A.out("ind", (n, J, FM, 2), I32)]


def _peaks_maps(A, n, h, w, sizes=None):
    if sizes is None:
        det, tag = parser_maps(n, h, w, 5 * h + w)
        hw = desc = None
    else:
        det, tag, hw, desc = ragged_maps(sizes, 11)
        n = len(sizes)
    d, t = A.inp("det", det), A.inp("tag_map", tag)
    dd = None if desc is None else A.desc("desc", desc)
    o = _peak_outs(A, n)
    return [_L().lp_find_peaks_maps_f32(d.data_ptr(), t.data_ptr(), n, h, w, None if hw is None else hw.ctypes.data,
                                        _p(dd), J, TT, J, FM, FTHR, FWIN, *[v.data_ptr() for v in o], _s())]


def _assign(A, pk, n):
    t = [A.inp("count", pk["count"]), A.inp("val", pk["val"]), A.inp("tag", pk["tag"]), A.inp("ind", pk["ind"]),
         A.inp("joint_order", JOINT_ORDER)]
    num, ans, st = A.out("num_person", (n,), I32), A.out("ans", (n, FM, J, 4), F32), A.out("status", (n,), I32)
    return [_L().lp_assign_f32(*[v.data_ptr() for v in t], n, J, FM, FTAG, num.data_ptr(), ans.data_ptr(), st.data_ptr(),
                               _s())]


def _fast_cases(n, h, w):
    sfx = "n%d-%dx%d" % (n, h, w)
    pk = functools.lru_cache(None)(lambda: _plain(lambda A: _peaks(A, n, h, w)))
    _add("find_peaks-" + sfx, ["lp_find_peaks_f32"], lambda A: _peaks(A, n, h, w), untouched=("val", "tag", "ind"))
    _add("find_peaks_maps-" + sfx, ["lp_find_peaks_maps_f32"], lambda A: _peaks_maps(A, n, h, w),
         untouched=("val", "tag", "ind"))
    _add("assign-" + sfx, ["lp_assign_f32"], lambda A: _assign(A, pk(), n), untouched=("ans",))

    @functools.lru_cache(None)
    def assigned():
        def run(A):
            # as the pipeline runs it: ans zeroed first (lp_assign_f32 writes only what it assigns)
            t = [A.inp(k, pk()[k]) for k in ("count", "val", "tag", "ind")] + [A.inp("joint_order", JOINT_ORDER)]
            num, st = A.out("num_person", (n,), I32), A.out("status", (n,), I32)
            ans = A.out("ans", (n, FM, J, 4), F32, init=np.zeros((n, FM, J, 4), F32))
            return [_L().lp_assign_f32(*[v.data_ptr() for v in t], n, J, FM, FTAG, num.data_ptr(), ans.data_ptr(),
                                       st.data_ptr(), _s())]
        return _plain(run)

    def pack(A):
        a = assigned()
        t = [A.inp("ans", a["ans"]), A.inp("num_person", a["num_person"]), A.inp("status", a["status"])]
        out = A.out("packed", (n, FM * J * 4 + 2), F32)
        return [_L().lp_pack_fast_payload_f32(*[v.data_ptr() for v in t], n, FM, J, out.data_ptr(), _s())]
    _add("pack_fast_payload-" + sfx, ["lp_pack_fast_payload_f32"], pack)


_fast_cases(2, 64, 96)
_fast_cases(1, 40, 90)
_add("find_peaks_maps-ragged", ["lp_find_peaks_maps_f32"], lambda A: _peaks_maps(A, 0, 0, 0, RAGGED[0]),
     untouched=("val", "tag", "ind"))


# ---------------------------------------------------------------- payload, planting, final predictions
def _payload_case(n, pcap, keep, seed):
    row = J * (3 + TT)

    @functools.lru_cache(None)
    def inputs():
        rng = np.random.default_rng(seed)
        ans = rng.standard_normal((n, pcap, J, 3 + TT)).astype(F32)
        num = rng.integers(0, pcap + 3, n).astype(I32)         # a count may exceed keep (and pcap)
        num[0] = 0
        scores = rng.standard_normal((n, pcap)).astype(F32)
        return ans, num, scores

    def run(A):
        ans, num, scores = inputs()
        t = [A.inp("ans", ans), A.inp("num", num), A.inp("scores", scores)]
        out = A.out("packed", (n, keep * row + keep + 1), F32)
        return [_L().lp_pack_payload_f32(*[v.data_ptr() for v in t], n, pcap, row, keep, out.data_ptr(), _s())]
    _add("pack_payload-n%d-pcap%d-keep%d" % (n, pcap, keep), ["lp_pack_payload_f32"], run, untouched=("packed",))


_payload_case(3, 20, 20, 1)
_payload_case(4, 30, 7, 2)


def _plant_case(n, h, w, seed):
    @functools.lru_cache(None)
    def inputs():
        rng = np.random.default_rng(seed)
        det = rng.random((n, J, h, w)).astype(F32)
        tag = rng.standard_normal((n, J, h, w, TT)).astype(F32)
        di = rng.integers(0, det.size, 300).astype(I64)
        di[:20] = di[0]                                        # repeated det indices: the max wins, in any order
        ti = rng.choice(tag.size, 200, replace=False).astype(I64)
        return det, tag, di, rng.random(300).astype(F32) * 2, ti, rng.standard_normal(200).astype(F32)

    def run(A):
        det, tag, di, dv, ti, tv = inputs()
        d, t = A.out("det", det.shape, F32, init=det), A.out("tag", tag.shape, F32, init=tag)
        a = [A.inp("det_index", di), A.inp("det_value", dv), A.inp("tag_index", ti), A.inp("tag_value", tv)]
        return [_L().lp_plant_crowd_f32(d.data_ptr(), a[0].data_ptr(), a[1].data_ptr(), di.size, t.data_ptr(),
                                        a[2].data_ptr(), a[3].data_ptr(), ti.size, _s())]
    _add("plant_crowd-n%d-%dx%d" % (n, h, w), ["lp_plant_crowd_f32"], run)


_plant_case(2, 32, 48, 3)


def _transform_case(idx, pcap):
    """the golden get_final_preds vectors of the transforms cases ``idx`` (test_transforms), one image each, every
    image with its own matrix"""
    @functools.lru_cache(None)
    def inputs():
        import os
        from litepose_b200.lib.utils import transforms as T
        from oracle.make_golden_transforms import keypoints
        g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "transforms.npz"))
        ans = np.full((len(idx), pcap, 14, 5), -3.0, F32)
        want = ans.copy()
        num = np.zeros(len(idx), I32)
        trans = []
        for k, i in enumerate(idx):
            wr, hr = (int(v) for v in g["c%02d_size" % i])
            persons = keypoints(100 + i, 1 + i % 4, 14, 2, wr, hr)
            num[k] = len(persons)
            ans[k, :len(persons)] = np.stack(persons)
            want[k, :len(persons)] = g["c%02d_final" % i]
            trans.append(T.get_affine_transform(g["c%02d_center" % i], g["c%02d_scale" % i], 0, [wr, hr], inv=1))
        return ans, num, np.stack(trans).reshape(-1, 6).astype(F64), want

    def run(A):
        ans, num, trans, _ = inputs()
        a = A.out("ans", ans.shape, F32, init=ans)
        nd, td = A.inp("num", num), A.inp("trans", trans)
        return [_L().lp_transform_preds_f32(a.data_ptr(), nd.data_ptr(), td.data_ptr(), ans.shape[0], ans.shape[1], 14,
                                            5, _s())]
    _add("transform_preds-n%d-pcap%d" % (len(idx), pcap), ["lp_transform_preds_f32"], run, lambda: {"ans": inputs()[3]})


_transform_case(tuple(range(10)), 6)
_transform_case((3, 6, 7), 4)


# ---------------------------------------------------------------- coverage bookkeeping
NOT_LAUNCHING = {"lp_version", "lp_last_error", "lp_device_check", "lp_launch_count", "lp_reset_launch_count",
                 "lp_set_dw_precision", "lp_get_dw_precision"}


def launching_symbols():
    """every symbol of _lib.SIGNATURES that launches device work: all but the packers, *_elems, *_supported,
    *_workspace_bytes and the library-state functions above"""
    from litepose_b200._lib import SIGNATURES
    return {s for s in SIGNATURES if s not in NOT_LAUNCHING and
            not s.endswith(("_pack", "_pack_wexp", "_elems", "_supported", "_workspace_bytes"))}


def covered_symbols():
    return {e for c in CASES for e in c.entries}
