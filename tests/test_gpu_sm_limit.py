"""-m gpu: every persistent kernel gives the same bits at any SM count (lp_set_sm_limit).

The persistent kernels size their grids from the SM count: the grid decides which tiles each CTA walks, how often the
mbarrier rings' parities wrap, where the deconv row kernel's row runs begin, whether lp_pw1x1_f16 keeps its weights
resident, and how early a dependent launch starts.  A tile's arithmetic does not depend on the CTA that computes it, so
under every limit each entry point must equal its emulator, bit for bit.

(a) Each grid-sizing entry point against its emulator under the limits 1, 2, 3, 7, 16, 66, 114, 131 and one above the
    device's count (plus the limits at which a kernel changes its partition), at shapes where the partition matters.
    The emulator is computed once per shape; every limit's output must equal it, and equal the default grid's output
    as bits.
(b) LitePoseEngine.run equals net_emul.forward for the NET_CASES of test_gpu_mma_exact at limits 1, 7 and 114, every
    traced intermediate compared, so that the first tensor that differs names the op at fault.
(c) The benchmark's geometry (LitePose-S, 512 x 512, fp16, batch 32, flip): LitePosePipeline.step() and the packed
    payload (its persons and the count; the slots past the count are not part of the result), the det / tag maps and
    a replay of the captured graph at limits 7 and 114 equal the default grid's, bit for bit; a mixed-size
    infer_images list at limit 114 equals the default grid's.
(d) The limit really reaches the launches: each kernel's grid, read from a torch.profiler trace, is at most the limit
    (3x for the fused stem, 8x for lp_bn_apply_f16), and the getter reports the limit in a freshly started thread."""
import json
import os
import tempfile
import threading

import numpy as np
import pytest
import torch

import bn_train_emul as bte
import conv_ref as cr
import dw_emul as de
import mma_emul as me
from litepose_b200 import _lib
from gpu_util import pack_pw, stream
from test_gpu_block_s2 import _Block, _inputs as _s2_inputs
from test_gpu_dw_exact import _dw7_project, _head_fused, _head_inputs, _proj_inputs
from test_gpu_mma_exact import NET_CASES, _net, _pw_inputs, _pw_run, assert_equal_values, run_deconv, run_head

pytestmark = pytest.mark.gpu

LIMITS = [1, 2, 3, 7, 16, 66, 114, 131]


@pytest.fixture(autouse=True)
def restore_library_state():
    """every test starts and ends at the device's SM count and the per-kernel-size depthwise arithmetic"""
    lib = _lib.load()
    lib.lp_set_sm_limit(0)
    lib.lp_set_dw_precision(-1)
    try:
        yield
    finally:
        lib.lp_set_sm_limit(0)
        lib.lp_set_dw_precision(-1)


def _device_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _limits(extra=()):
    """LIMITS, the kernel's own partition edges and one limit above the device's count"""
    return sorted(set(LIMITS) | set(extra)) + [_device_sms() + 1]


def _set_limit(n):
    lib = _lib.load()
    lib.lp_set_sm_limit(n)
    want = _device_sms() if n <= 0 else min(n, _device_sms())
    assert lib.lp_get_sm_limit() == want, (n, lib.lp_get_sm_limit(), want)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32}[a.itemsize])


def _check_every_limit(run, want, what, extra=(), sel=None):
    """run() -> the entry point's output as numpy.  Under every limit it equals the emulator's ``want`` (on the
    elements ``sel`` picks, all by default) and the default grid's output, bit for bit."""
    _set_limit(0)
    default = run()
    pick = (lambda a: a) if sel is None else sel
    assert_equal_values(pick(default), want, "%s default grid" % what)
    bad = []
    for lim in _limits(extra):
        _set_limit(lim)
        got = run()
        neq = _bits(got) != _bits(default)
        if neq.any():
            bad.append("limit %d: %d of %d elements differ from the default grid (first at %s)" % (
                lim, neq.sum(), neq.size, np.argwhere(neq)[0]))
        else:
            assert_equal_values(pick(got), want, "%s limit %d" % (what, lim))
    _set_limit(0)
    assert not bad, "%s: %s" % (what, "; ".join(bad))


# ---------------------------------------------------------------- (a) each entry point against its emulator
# (m, k, n, act, res, extra limits): N = 720 (6 chunks) and 960 (8 chunks) of 128 MMA columns, odd m_tiles (17 of 64
# rows).  K <= 320 keeps the weights resident when n_chunks <= SMs (cpc = SMs / n_chunks CTAs per chunk), below that
# they stream with several chunks; K = 960 streams at every grid.
PW_CASES = [
    (1083, 120, 720, 2, True, (5, 6, 12, 13)),
    (1083, 64, 960, 1, True, (8, 9, 17)),
    (171, 960, 720, 0, True, (5, 6)),
    (1083, 40, 160, 2, False, ()),
]


@pytest.mark.parametrize("m,k,n,act,res,extra", PW_CASES)
def test_pw1x1_every_limit(m, k, n, act, res, extra):
    a, wt, b, r = _pw_inputs(m, k, n, res, m + 7 * k + n, wide=m >= 1000)
    _check_every_limit(lambda: _pw_run(a, wt, b, r, act), me.pw1x1(a, wt, b, r, act),
                       "pw1x1 m%d k%d n%d act%d res%d" % (m, k, n, act, res), extra)


# deconv row kernel: items = strips * N * H rows, CTA b walks items [b*per + min(b, extra), ...) with per = items / grid
# (n, h, w, cr, cw, co, extra limits, what the partition edges are)
DECONV_ROWS_SM_CASES = [
    # 2 strips x 2 images x 7 rows = 28 items: limit 2 -> runs of 14 end at the strip boundary; 4 -> runs of 7 end at
    # image boundaries; 3, 7 -> mid-strip starts; 16 -> per = 1 (every item starts a run); 66 and up -> items < limit
    (2, 7, 200, 24, 16, 8, (4, 14, 27, 28, 29)),
    # 3 strips (the last 4 pixels wide) x 2 images x 9 rows = 54 items: 3 -> runs of 18 = one strip; 6 -> runs of 9 =
    # one image; 2 -> 27, across a strip boundary; 16 -> 3 or 4; 66 -> grid 54, per = 1
    (2, 9, 260, 16, 8, 24, (6, 18, 27, 53, 54)),
    (1, 1, 128, 16, 8, 24, ()),           # H = 1: every run is one row
]


def _deconv_run(xr, xw, wr, ww, b, act=None):
    """lp_fusion_deconv_f16 (act None) or lp_fusion_deconv_act_f16 -> [N,2H,2W,Co]"""
    if act is None:
        return run_deconv(xr, xw, wr, ww, b)
    lib = _lib.load()
    n, h, w, cr_ = xr.shape
    cw, co = xw.shape[3], wr.shape[1]
    wp = np.zeros(lib.lp_deconv_packed_elems(cr_, cw, co), np.uint16)
    bp = np.zeros(lib.lp_deconv_packed_bias_elems(co), np.float32)
    _lib.check(lib.lp_deconv_pack(wr.view(np.uint16).ctypes.data, ww.view(np.uint16).ctypes.data, b.ctypes.data, cr_,
                                  cw, co, wp.ctypes.data, bp.ctypes.data), "deconv_pack")
    out = torch.full((n, 2 * h, 2 * w, co), float("nan"), dtype=torch.float16, device="cuda")
    rd, rwd, wd, bd = _dev(xr), _dev(xw), _dev(wp.view(np.float16)), _dev(bp)
    _lib.check(lib.lp_fusion_deconv_act_f16(rd.data_ptr(), rwd.data_ptr(), wd.data_ptr(), bd.data_ptr(), out.data_ptr(),
                                            n, h, w, cr_, cw, co, act, stream()), "deconv_act")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _check_deconv_every_limit(n, h, w, cr_, cw, co, rows, extra=()):
    """lp_fusion_deconv_f16 against mma_emul.deconv, lp_fusion_deconv_act_f16 (act none) against
    bn_train_emul.deconv_raw"""
    assert cr.uses_rows_kernel(cr_, cw, co, w) == rows
    xr, xw, wr, ww, b = cr.deconv_inputs(n, h, w, cr_, cw, co, 3 * n + h + w + cr_ + cw + co)
    what = "deconv %s n%d %dx%d cr%d cw%d co%d" % ("rows" if rows else "tiled", n, h, w, cr_, cw, co)
    _check_every_limit(lambda: _deconv_run(xr, xw, wr, ww, b), me.deconv(xr, xw, wr, ww, b, rows), what, extra)
    _check_every_limit(lambda: _deconv_run(xr, xw, wr, ww, b, _lib.ACT_NONE), bte.deconv_raw(xr, xw, wr, ww, b),
                       what + " act none", extra)


@pytest.mark.parametrize("n,h,w,cr_,cw,co,extra", DECONV_ROWS_SM_CASES)
def test_deconv_rows_every_limit(n, h, w, cr_, cw, co, extra):
    _check_deconv_every_limit(n, h, w, cr_, cw, co, True, extra)


# the tiled kernel (gemm_tc_kernel): 32 x 4 pixel tiles, 2 x 10 x 4 = 80 tiles; Co = 40 > 32 at W = 100, 16 x 8 pixel
# tiles, 7 x 5 = 35 tiles
DECONV_TILED_SM_CASES = [(4, 40, 63, 16, 16, 16), (1, 36, 100, 24, 16, 40)]


@pytest.mark.parametrize("n,h,w,cr_,cw,co", DECONV_TILED_SM_CASES)
def test_deconv_tiled_every_limit(n, h, w, cr_, cw, co):
    _check_deconv_every_limit(n, h, w, cr_, cw, co, False)


# (n, h, w, C1, C2, Co, fp32): 16 x 8 pixel tiles; 45 and 67 tiles
HEAD_PW_SM_CASES = [(3, 37, 45, 24, 40, 17, True), (1, 536, 16, 32, 32, 34, False)]


@pytest.mark.parametrize("n,h,w,c1,c2,co,fp32", HEAD_PW_SM_CASES)
def test_head_pw_dual_every_limit(n, h, w, c1, c2, co, fp32):
    rng = np.random.default_rng(n + h + w + c1 + c2 + co)
    p = n * h * w
    a1 = np.maximum(rng.standard_normal((p, c1)), 0).astype(np.float16)
    a2 = np.maximum(rng.standard_normal((p, c2)) * 2.0 ** rng.integers(-12, 4, (p, 1)), 0).astype(np.float16)
    w1 = (rng.standard_normal((co, c1)) / c1 ** 0.5).astype(np.float16)
    w2 = (rng.standard_normal((co, c2)) / c2 ** 0.5).astype(np.float16)
    _check_every_limit(lambda: run_head(a1, a2, w1, w2, fp32, n, h, w), me.head_dual(a1, a2, w1, w2, fp32),
                       "head_pw_dual n%d %dx%d c1 %d c2 %d co %d" % (n, h, w, c1, c2, co))


# (n, h, w, Ce, Co, res): Co <= 64 runs dw_project_kernel (16 x 16 tiles: 67 and 75 tiles), wider Co
# dw_project_wide_kernel (16 x 8 tiles: 67 and 18 tiles)
DW7_PROJECT_SM_CASES = [(67, 16, 16, 96, 16, True), (5, 48, 80, 144, 24, True), (67, 8, 16, 288, 120, True),
                        (2, 20, 40, 432, 72, False)]


@pytest.mark.parametrize("n,h,w,ce,co,res", DW7_PROJECT_SM_CASES)
def test_dw7_project_every_limit(n, h, w, ce, co, res):
    x, wd, bd, wp, bp, r = _proj_inputs(n, h, w, ce, co, res, ce * 3 + co + h + n)
    xd, wdd, bdd, rd = _dev(x), _dev(wd), _dev(bd), _dev(r) if res else None
    wpk, bpk = pack_pw(torch.from_numpy(wp), torch.from_numpy(bp))

    def run():
        out = _dw7_project(xd, wdd, bdd, wpk, bpk, rd, n, h, w, ce, co)
        torch.cuda.synchronize()
        return out.cpu().numpy().reshape(-1, co)
    d = de.dwconv(x, wd, bd, 7, 1, de.ACT_RELU6, de.default_prec(7))
    want = me.pw1x1(d.reshape(-1, ce), wp, bp, None if r is None else r.reshape(-1, co))
    _check_every_limit(run, want, "dw7_project n%d %dx%d ce%d co%d res%d" % (n, h, w, ce, co, res))


# (n, h, w, C1, C2, Co, fp32): 16 x 16 tiles, 67 and 27 tiles
HEAD_FUSED_SM_CASES = [(67, 16, 16, 24, 16, 28, True), (3, 37, 45, 72, 40, 34, False)]


@pytest.mark.parametrize("n,h,w,c1,c2,co,fp32", HEAD_FUSED_SM_CASES)
def test_head_fused_every_limit(n, h, w, c1, c2, co, fp32):
    x1, d1, b1, x2, d2, b2, w1, w2 = _head_inputs(n, h, w, c1, c2, co, c1 * 7 + c2 + co)
    t1 = de.dwconv(x1, d1, b1, 5, 1, de.ACT_RELU, de.default_prec(5)).reshape(-1, c1)
    t2 = de.dwconv(x2, d2, b2, 5, 1, de.ACT_RELU, de.default_prec(5)).reshape(-1, c2)
    want = me.head_dual(t1, t2, w1, w2, fp32)
    _check_every_limit(lambda: _head_fused(x1, d1, b1, x2, d2, b2, w1, w2, n, h, w, c1, c2, co, fp32)
                       .transpose(0, 2, 3, 1).reshape(-1, co), want,
                       "head_fused n%d %dx%d c1 %d c2 %d co %d fp32 %d" % (n, h, w, c1, c2, co, fp32))


def _emulated_images(n):
    """the images the emulator runs for a batch of n: all of a small batch, the first and the last of a large one"""
    return list(range(n)) if n <= 2 else [0, n - 1]


# test_gpu_block_pipeline.SCHEDULE_SHAPES: odd slab counts (3, 5), the streaming layout (Ce = 288, 320), 1 to 1024
# 16 x 16 tiles; and 67 single-tile images
BLOCK_S1_SM_CASES = [
    (16, 128, 128, 16, 96, 16, True), (8, 64, 64, 32, 192, 32, True), (20, 32, 32, 48, 288, 48, True),
    (4, 64, 64, 32, 160, 32, False), (5, 48, 48, 16, 96, 16, False), (1, 32, 48, 32, 192, 32, True),
    (1, 16, 16, 16, 32, 16, False), (2, 32, 32, 32, 64, 48, False), (1, 16, 16, 64, 160, 64, True),
    (3, 48, 48, 40, 320, 56, False), (67, 16, 16, 16, 96, 16, True),
]


@pytest.mark.parametrize("n,h,w,cin,ce,co,res", BLOCK_S1_SM_CASES)
def test_block_s1_every_limit(n, h, w, cin, ce, co, res):
    lib = _lib.load()
    assert lib.lp_block_s1_supported(cin, ce, co) == 1
    rng = np.random.default_rng(cin * 5 + ce * 3 + co + h + n)
    x = rng.standard_normal((n, h, w, cin)).astype(np.float16)
    we = (rng.standard_normal((ce, cin)) / cin ** 0.5).astype(np.float16)
    be = (rng.standard_normal(ce) * 0.2).astype(np.float32)
    _, wd, bd = de.make_inputs(1, ce, 1, 1, 7, "relu6", ce + h)
    wp = (rng.standard_normal((co, ce)) / ce ** 0.5).astype(np.float16)
    bp = (rng.standard_normal(co) * 0.1).astype(np.float32)
    xd, wdd, bdd, bed = _dev(x), _dev(wd), _dev(bd), _dev(be)
    wpk, bpk = pack_pw(torch.from_numpy(wp), torch.from_numpy(bp))
    wek = np.zeros(lib.lp_block_s1_wexp_elems(cin, ce), np.uint16)
    _lib.check(lib.lp_block_s1_pack_wexp(we.view(np.uint16).ctypes.data, cin, ce, wek.ctypes.data))
    wed = torch.from_numpy(wek).view(torch.float16).cuda()

    def run():
        out = torch.full((n, h, w, co), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(lib.lp_block_s1_f16(xd.data_ptr(), wed.data_ptr(), bed.data_ptr(), wdd.data_ptr(), bdd.data_ptr(),
                                       wpk.data_ptr(), bpk.data_ptr(), 1 if res else 0, out.data_ptr(), n, h, w, cin,
                                       ce, co, stream()), "block_s1")
        torch.cuda.synchronize()
        return out.cpu().numpy()
    img = _emulated_images(n)
    xs = x[img]
    e = me.pw1x1(xs.reshape(-1, cin), we, be, None, de.ACT_RELU6).reshape(len(img), h, w, ce)
    d = de.dwconv(e, wd, bd, 7, 1, de.ACT_RELU6, de.default_prec(7))
    want = me.pw1x1(d.reshape(-1, ce), wp, bp, xs.reshape(-1, cin) if res else None).reshape(len(img), h, w, co)
    _check_every_limit(run, want, "block_s1 n%d %dx%d cin%d ce%d co%d res%d" % (n, h, w, cin, ce, co, res),
                       sel=lambda a: a[img])


# (n, h, w, Cin, Ce, Co): 16 x 8 output tiles; 18, 16, 67 and 75 tiles; one and five slabs
BLOCK_S2_SM_CASES = [(3, 40, 52, 16, 96, 16), (2, 64, 64, 16, 160, 16), (67, 16, 32, 16, 96, 32),
                     (5, 76, 92, 8, 48, 40), (2, 64, 64, 16, 32, 16)]


@pytest.mark.parametrize("n,h,w,cin,ce,co", BLOCK_S2_SM_CASES)
def test_block_s2_every_limit(n, h, w, cin, ce, co):
    assert _lib.load().lp_block_s2_supported(cin, ce, co) == 1
    seed = cin * 5 + ce * 3 + co + h + w + n
    blk = _Block(n, h, w, cin, ce, co, seed)
    x, we, be, wd, bd, wp, bp = _s2_inputs(n, h, w, cin, ce, co, seed)
    img = _emulated_images(n)
    e = me.pw1x1(x[img].reshape(-1, cin), we, be, None, de.ACT_RELU6).reshape(len(img), h, w, ce)
    d = de.dwconv(e, wd, bd, 7, 2, de.ACT_RELU6, de.default_prec(7))
    want = me.pw1x1(d.reshape(-1, ce), wp, bp).reshape(len(img), h // 2, w // 2, co)
    _check_every_limit(blk.fused, want, "block_s2 n%d %dx%d cin%d ce%d co%d" % (n, h, w, cin, ce, co),
                       sel=lambda a: a[img])


# (n, h, w, C0, flip): grid 3 x SMs over 8 x 8 output tiles
STEM_SM_CASES = [(3, 100, 100, 24, 0), (2, 130, 260, 16, 1), (1, 36, 64, 8, 1)]


def _stem_case(n, h, w, c0, flip):
    """(run, emulated output [n*Ho*Wo, C0]) of lp_stem_fused_f16 on an fp16 image"""
    from test_gpu_stem_deconv_exact import _stem_inputs
    lib = _lib.load()
    assert lib.lp_stem_fused_supported(h, w, c0) == 1
    x, w1, b1, wdw, bdw, w3, b3 = _stem_inputs(n, h, w, c0, n * 1000 + h * 7 + w + c0 + flip)
    x16 = x.astype(np.float16)
    ho, wo = h // 2, w // 2
    w1p = np.zeros((32, 64), np.float16)
    w1p[:, :27] = w1
    xd, w1d, b1d, wdd, bdd = _dev(x16), _dev(w1p), _dev(b1), _dev(wdw), _dev(bdw)
    w3k, b3k = pack_pw(torch.from_numpy(w3), torch.from_numpy(b3))

    def run():
        y = torch.full((n, ho, wo, c0), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(lib.lp_stem_fused_f16(xd.data_ptr(), 0, flip, w1d.data_ptr(), b1d.data_ptr(), wdd.data_ptr(),
                                         bdd.data_ptr(), w3k.data_ptr(), b3k.data_ptr(), y.data_ptr(), n, h, w, c0,
                                         stream()), "stem_fused")
        torch.cuda.synchronize()
        return y.cpu().numpy().reshape(-1, c0)
    e = me.pw1x1(cr.stem_im2col(x16, flip), w1p[:, :32], b1, None, de.ACT_RELU6).reshape(n, ho, wo, 32)
    d = de.dwconv(e, wdw, bdw, 3, 1, de.ACT_RELU6, de.default_prec(3))
    return run, me.pw1x1(d.reshape(-1, 32), w3, b3)


@pytest.mark.parametrize("n,h,w,c0,flip", STEM_SM_CASES)
def test_stem_fused_every_limit(n, h, w, c0, flip):
    run, want = _stem_case(n, h, w, c0, flip)
    _check_every_limit(run, want, "stem_fused n%d %dx%d c0 %d flip %d" % (n, h, w, c0, flip))


# (M, C, act, residual, in place): grid min(ceil(M*C/8 / 256), 8 x SMs), a grid-stride loop over 8-channel vectors
BN_APPLY_SM_CASES = [(9000, 720, _lib.ACT_RELU6, True, False), (9000, 720, _lib.ACT_NONE, False, False),
                     (9000, 720, _lib.ACT_RELU, True, True), (5000, 40, _lib.ACT_RELU6, False, True),
                     (777, 24, _lib.ACT_RELU, True, False)]


def _bn_case(m, c, act, res, in_place):
    lib = _lib.load()
    rng = np.random.default_rng(m + c + act)
    x = (rng.standard_normal((m, c)) * np.exp(rng.standard_normal(c))).astype(np.float16)
    scale = rng.uniform(0.5, 1.5, c).astype(np.float32)
    shift = (rng.standard_normal(c) * 0.3).astype(np.float32)
    r = rng.standard_normal((m, c)).astype(np.float16) if res else None
    xd, sd, hd, rd = _dev(x), _dev(scale), _dev(shift), _dev(r) if res else None

    def run():
        src = xd.clone()
        y = src if in_place else torch.full_like(xd, float("nan"))
        _lib.check(lib.lp_bn_apply_f16(src.data_ptr(), sd.data_ptr(), hd.data_ptr(), None if rd is None else rd.data_ptr(),
                                       y.data_ptr(), m, c, act, stream()), "lp_bn_apply_f16")
        torch.cuda.synchronize()
        return y.cpu().numpy()
    return run, bte.apply(x, scale, shift, act, r)


@pytest.mark.parametrize("m,c,act,res,in_place", BN_APPLY_SM_CASES)
def test_bn_apply_every_limit(m, c, act, res, in_place):
    run, want = _bn_case(m, c, act, res, in_place)
    _check_every_limit(run, want, "bn_apply m%d c%d act%d res%d in_place%d" % (m, c, act, res, in_place))


# ---------------------------------------------------------------- (b) the whole forward under a limit
_net_emul_cache = {}


@pytest.mark.parametrize("case", NET_CASES, ids=["-".join(map(str, c)) for c in NET_CASES])
def test_engine_forward_equals_net_emul_under_limits(case):
    import net_emul
    from litepose_b200 import engine, synth
    arch_name, n, h, w, dt, out_fp32, flip = case
    arch, sd = _net(arch_name, h)
    x = synth.make_frames(n, h, seed=h + w + n, width=w)
    x = x.half() if dt == "fp16" else x
    trace = []
    want = net_emul.forward(sd, arch, x.numpy(), flip, out_fp32, trace)
    name = "-".join(map(str, case))
    for lim in (1, 7, 114):
        _set_limit(lim)
        eng = engine.LitePoseEngine(sd, arch, "cuda")          # a fresh engine: nothing launched before the limit
        got = eng.run(x.cuda(), flip=flip, out_fp32=out_fp32)
        torch.cuda.synchronize()
        plan = next(iter(eng.plans.values()))
        keep = plan["keep"]
        fused_stem = any(op.name == "stem_fused" for op in plan["ops"])
        inner = [keep[0]] + [t for t in keep[1 if fused_stem else 3:] if t.dim() == 4]
        assert len(inner) == len(trace), (len(inner), [nm for nm, _ in trace])
        for t, (nm, wt) in zip(inner, trace):        # the first tensor that differs names the op at fault
            assert_equal_values(t.cpu().numpy(), wt, "%s limit %d %s" % (name, lim, nm))
        for i, (g, wt) in enumerate(zip(got, want)):
            assert_equal_values(g.cpu().numpy(), wt, "%s limit %d output %d" % (name, lim, i))
        del eng, got, plan, keep, inner


# ---------------------------------------------------------------- (c) the benchmark's geometry under a limit
def _bench_pipe():
    """LitePose-S 512 x 512, batch 32, flip test, graphs, keep 64, five planted persons: bench.py's configuration"""
    from litepose_b200 import synth
    from litepose_b200.config import get_arch, get_cfg
    from litepose_b200.lib.models.pose_mobilenet import get_pose_net
    from litepose_b200.pipeline import LitePosePipeline
    cfg = get_cfg(input_size=512)
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch("S")), 1)).eval().cuda()
    return LitePosePipeline(model, cfg, use_graphs=True, keep=64)


def _payload_defined(packed, keep, row):
    """mask of the packed payload's defined floats: per image the keypoints and scores of its first min(count, keep)
    persons and the count.  The slots past the count are not part of the result (unpack never reads them) and carry
    whatever the parser's buffers held: lp_adjust_refine_f32 writes the scores of the persons it found only."""
    mask = np.zeros(packed.shape, bool)
    mask[:, -1] = True
    for i, c in enumerate(packed[:, -1]):
        p = min(int(c), keep)
        mask[i, :p * row] = True
        mask[i, keep * row:keep * row + p] = True
    return mask


def test_bench_geometry_same_bits_under_limits():
    from litepose_b200 import synth
    from litepose_b200.pipeline import PlantedCrowd
    frames = synth.make_frames(32, 512, seed=1234).half().pin_memory()
    plant = PlantedCrowd(32, 14, 512, 512, 2, num_people=5, seed=77, device="cuda")
    x_dev = frames.cuda()
    runs = {}
    for lim in (0, 7, 114):
        _set_limit(lim)
        pipe = _bench_pipe()                                   # fresh: its graphs are captured under the limit
        packed = pipe.step_device(x_dev, plant).clone()
        maps = [pipe._last_state[k].clone() for k in ("det", "tag")]   # the network passes + glue, every element defined
        host = pipe.step(frames, plant)
        again = pipe.step_device(x_dev, plant).clone()          # a replay of the graph captured under the limit
        torch.cuda.synchronize()
        runs[lim] = ([packed.cpu().numpy(), again.cpu().numpy()], [m.cpu().numpy() for m in maps], host)
        keep, row = pipe.keep, pipe.row
        del pipe
    (ref_packed, _), ref_maps, ref_host = runs[0]
    assert ref_packed[:, -1].sum() > 0, "no person found: the comparison would be vacuous"
    defined = _payload_defined(ref_packed, keep, row)
    for lim in (0, 7, 114):
        packeds, maps, host = runs[lim]
        for what, got, want in (("det", maps[0], ref_maps[0]), ("tag", maps[1], ref_maps[1])):
            neq = _bits(got) != _bits(want)
            assert not neq.any(), "limit %d %s: %d of %d elements differ from the default grid (first at %s)" % (
                lim, what, neq.sum(), neq.size, np.argwhere(neq)[0])
        for what, got in zip(("packed", "packed replay"), packeds):
            assert np.array_equal(got[:, -1], ref_packed[:, -1]), "limit %d %s: person counts differ" % (lim, what)
            neq = (_bits(got) != _bits(ref_packed)) & defined
            assert not neq.any(), "limit %d %s: %d of %d payload floats differ from the default grid" % (
                lim, what, neq.sum(), defined.sum())
        assert len(host) == len(ref_host)
        for i, (g, e) in enumerate(zip(host, ref_host)):
            assert g[-1] == e[-1], (lim, i)
            assert np.array_equal(_bits(np.asarray(g[0], np.float32)), _bits(np.asarray(e[0], np.float32))), (lim, i)
            assert np.array_equal(_bits(np.asarray(g[1], np.float32)), _bits(np.asarray(e[1], np.float32))), (lim, i)


def test_mixed_size_list_same_under_limit():
    from test_gpu_submit_images import LIST_A, _cfg_case, _images, _pipe, _plants, _same
    imgs = _images(LIST_A, seed=5)
    results = {}
    for lim in (0, 114):
        _set_limit(lim)
        pipe = _pipe(_cfg_case("shipped"), keep=2)
        results[lim] = pipe.infer_images(imgs, plant=_plants(pipe, [im.shape[:2] for im in imgs]))
        del pipe
    assert sum(r[-1] for r in results[0]) > 0
    _same(results[114], results[0], "infer_images list at limit 114")


# ---------------------------------------------------------------- (d) the limit reaches the launches
def _block_s1_call(n, h, w, cin, ce, co):
    """lp_block_s1_f16 on zeros (the trace and the timing below need its launch, not its values) -> run"""
    lib = _lib.load()
    xd = torch.zeros((n, h, w, cin), dtype=torch.float16, device="cuda")
    wek = torch.zeros(lib.lp_block_s1_wexp_elems(cin, ce), dtype=torch.float16, device="cuda")
    wdd = torch.zeros((49, ce), dtype=torch.float16, device="cuda")
    bed, bdd = torch.zeros(ce, device="cuda"), torch.zeros(ce, device="cuda")
    wpk, bpk = pack_pw(torch.zeros(co, ce), torch.zeros(co))
    out = torch.empty((n, h, w, co), dtype=torch.float16, device="cuda")

    def run():
        _lib.check(lib.lp_block_s1_f16(xd.data_ptr(), wek.data_ptr(), bed.data_ptr(), wdd.data_ptr(), bdd.data_ptr(),
                                       wpk.data_ptr(), bpk.data_ptr(), 1, out.data_ptr(), n, h, w, cin, ce, co,
                                       stream()), "block_s1")
    return run


def _small_calls():
    """one call of every grid-sizing entry point -> [(entry point, kernel, grid bound per SM, run)], each on more tiles
    than the limits of test_limit_reaches_every_launch"""
    calls = []
    a, wt, b, r = _pw_inputs(1083, 120, 720, True, 1)
    calls.append(("lp_pw1x1_f16", "pw_gemm_kernel", 1, lambda: _pw_run(a, wt, b, r, 2)))
    rows = cr.deconv_inputs(2, 9, 260, 16, 8, 24, 5)
    calls.append(("lp_fusion_deconv_f16 rows", "deconv_rows_kernel", 1, lambda: _deconv_run(*rows)))
    calls.append(("lp_fusion_deconv_act_f16 rows", "deconv_rows_kernel", 1,
                  lambda: _deconv_run(*rows, act=_lib.ACT_NONE)))
    tiled = cr.deconv_inputs(4, 40, 63, 16, 16, 16, 6)
    calls.append(("lp_fusion_deconv_f16 tiled", "gemm_tc_kernel", 1, lambda: _deconv_run(*tiled)))
    calls.append(("lp_fusion_deconv_act_f16 tiled", "gemm_tc_kernel", 1,
                  lambda: _deconv_run(*tiled, act=_lib.ACT_NONE)))
    rng = np.random.default_rng(2)
    h1 = [np.maximum(rng.standard_normal((536 * 16, c)), 0).astype(np.float16) for c in (32, 32)]
    h2 = [(rng.standard_normal((34, 32)) / 32 ** 0.5).astype(np.float16) for _ in range(2)]
    calls.append(("lp_head_pw_dual_f16", "gemm_tc_kernel", 1, lambda: run_head(*h1, *h2, True, 1, 536, 16)))
    x, wd, bd, wp, bp, rr = _proj_inputs(67, 16, 16, 96, 16, True, 7)
    px = [_dev(x), _dev(wd), _dev(bd)] + list(pack_pw(torch.from_numpy(wp), torch.from_numpy(bp))) + [_dev(rr)]
    calls.append(("lp_dw7_project_f16 narrow", "dw_project_kernel", 1, lambda: _dw7_project(*px, 67, 16, 16, 96, 16)))
    x, wd, bd, wp, bp, rr = _proj_inputs(67, 8, 16, 288, 120, True, 8)
    pw_ = [_dev(x), _dev(wd), _dev(bd)] + list(pack_pw(torch.from_numpy(wp), torch.from_numpy(bp))) + [_dev(rr)]
    calls.append(("lp_dw7_project_f16 wide", "dw_project_wide_kernel", 1,
                  lambda: _dw7_project(*pw_, 67, 8, 16, 288, 120)))
    head = _head_inputs(67, 16, 16, 24, 16, 28, 3)
    calls.append(("lp_head_fused_f16", "dw_project_kernel", 1, lambda: _head_fused(*head, 67, 16, 16, 24, 16, 28, True)))
    calls.append(("lp_block_s1_f16", "block_s1_kernel", 1, _block_s1_call(67, 16, 16, 16, 96, 16)))
    blk = _Block(67, 16, 32, 16, 96, 32, 9)
    calls.append(("lp_block_s2_f16", "block_s2_kernel", 1, blk.fused))
    stem_run, _ = _stem_case(2, 130, 260, 16, 1)
    calls.append(("lp_stem_fused_f16", "stem_fused_kernel", 3, stem_run))
    bn_run, _ = _bn_case(9000, 720, _lib.ACT_RELU6, True, False)
    calls.append(("lp_bn_apply_f16", "bn_apply_kernel", 8, bn_run))
    return calls


class _NoGridInTrace(Exception):
    pass


def _traced_kernels(run):
    """[(kernel name, grid size or None)] of the kernels in a torch.profiler trace of run(), in launch order"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    out = []
    for ev in sorted((ev for ev in events if ev.get("cat") == "kernel"), key=lambda ev: ev.get("ts", 0)):
        grid = (ev.get("args") or {}).get("grid")
        out.append((ev.get("name", ""), None if grid is None else
                    (grid[0] * grid[1] * grid[2] if isinstance(grid, list) else int(grid))))
    return out


def _launch_grids(calls):
    """one trace of every call of ``calls`` -> the grid of each call's kernel, in call order.  A trace that misses
    some of the launches (the profiler dropped device records) is taken again, up to three times.  Raises
    _NoGridInTrace when the trace carries no grid dimensions at all."""
    def run():
        for c in calls:
            c[3]()
    want = [c[1] for c in calls]
    for _ in range(3):
        kernels = [(nm, g) for nm, g in _traced_kernels(run) if any(k in nm for k in want)]
        found = [next(k for k in want if k in nm) for nm, _ in kernels]
        if found == want:
            break
    assert found == want, "kernels in three traces of the calls: last %s, launched %s" % (found, want)
    if all(g is None for _, g in kernels):
        raise _NoGridInTrace()
    return [g for _, g in kernels]


def test_limit_reaches_every_launch():
    calls = _small_calls()
    for c in calls:                                  # load the modules and warm up outside the traces
        c[3]()
    grids = {}
    for lim in (0, 3, 16):
        _set_limit(lim)
        try:
            got = _launch_grids(calls)
        except _NoGridInTrace:
            pytest.skip("this torch build's trace carries no grid dimensions "
                        "(test_limit_slows_a_single_sm_grid observes the limit on the device instead)")
        for c, g in zip(calls, got):
            grids[c[0], lim] = g
    _set_limit(0)
    sms = _device_sms()
    for label, kernel, per_sm, _ in calls:
        default = grids[label, 0]
        assert default <= per_sm * sms, (label, default)
        if kernel != "pw_gemm_kernel":               # more tiles than the limits: the default grid is larger
            assert default > 16 * per_sm, (label, default)
        for lim in (3, 16):
            got = grids[label, lim]
            assert got <= per_sm * lim, "%s: grid %d at limit %d (bound %d)" % (label, got, lim, per_sm * lim)
            if kernel != "pw_gemm_kernel":
                assert got == per_sm * lim, "%s: grid %d at limit %d, %d expected" % (label, got, lim, per_sm * lim)
    # lp_pw1x1_f16 at N = 720 (6 chunks), 17 m-tiles: resident with min(SMs / 6, 9) CTAs per chunk at the default grid
    # and at limit 16, streaming on every SM below 6
    assert grids["lp_pw1x1_f16", 0] == 6 * min(sms // 6, 9)
    assert grids["lp_pw1x1_f16", 16] == 12 and grids["lp_pw1x1_f16", 3] == 3


def test_limit_slows_a_single_sm_grid():
    """an observation made on the device, independent of the trace: a 1024-tile lp_block_s1_f16 launch takes far
    longer on one SM than on all of them"""
    run = _block_s1_call(16, 128, 128, 16, 96, 16)

    def timed():
        run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            run()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)
    t_all = timed()
    _set_limit(1)
    t_one = timed()
    assert t_one > 16 * t_all, "one SM: %.3f ms, all %d SMs: %.3f ms" % (t_one, _device_sms(), t_all)


def test_getter_reports_the_limit_in_a_fresh_thread():
    lib = _lib.load()
    for lim in (1, 7, 114, _device_sms() + 1):
        _set_limit(lim)
        seen = []
        t = threading.Thread(target=lambda: (torch.cuda.set_device(torch.cuda.current_device()),
                                             seen.append(lib.lp_get_sm_limit())))
        t.start()
        t.join()
        assert seen == [min(lim, _device_sms())], (lim, seen)
