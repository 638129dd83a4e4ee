"""-m gpu: the stem and fusion-deconv kernels held to exact references.

(a) lp_stem_fused_f16 equals the unfused chain it replaces, value for value:
      a = im2col(fp16(x))                       [M, 32], k = c*9 + ky*3 + kx, 5 zero columns (conv_ref.stem_im2col)
      e = lp_pw1x1_f16(a, W1, b1, ReLU6)        one wgmma per K=16 slice, fp32 accumulators, one rounding of acc + bias
      d = lp_dwconv_f16(e, w_dw, b_dw, k3 s1 ReLU6, precision 2)
      y = lp_pw1x1_f16(d, W3, b3)
    and the parts of that chain against references that run no kernel: e and y against fp64 (gpu_util.check_reduction,
    y over the emulated d), d equal to dw_emul.dwconv.
(b) lp_stem_fused_f16 on an fp32 image equals it on the image rounded to fp16 (RNE), bit for bit.
(c) lp_stem_conv3x3_s2 equals conv_ref.stem_conv bit for bit, on the vector and the generic load path.
(d) lp_fusion_deconv_f16, every output element against fp64 (gpu_util.check_bound, K = 4 (Cr + Cw) products per
    output; ReLU is 1-Lipschitz, so the bound holds after it), on the row kernel and on the tiled kernel."""
import numpy as np
import pytest
import torch

import conv_ref as cr
import dw_emul as de
import mma_emul as me
from litepose_b200 import _lib
from gpu_util import check_bound, check_reduction, pack_pw, stream

pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def assert_equal_values(got, want, what):
    got = np.asarray(got)
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    neq = got != want            # float compare: -0 == +0 (hmax may leave a -0)
    assert not neq.any(), "%s: %d of %d elements differ (first at %s: %r vs %r)" % (
        what, neq.sum(), neq.size, np.argwhere(neq)[0], got[neq][0], want[neq][0])


@pytest.fixture
def dw_precision():
    """sets lp_set_dw_precision for the test and always restores the per-kernel-size default"""
    lib = _lib.load()
    try:
        yield lib.lp_set_dw_precision
    finally:
        lib.lp_set_dw_precision(-1)


# ---------------------------------------------------------------- (a), (b) the fused stem
# (n, h, w, C0)
STEM_FUSED_SHAPES = [
    (2, 36, 64, 16),      # Ho = 18: a ragged tile row (Ho % 8 != 0)
    (1, 52, 36, 8),       # Ho = 26, Wo = 18 (W % 8 == 4): ragged in both; C0 = 8, a partial n_tile
    (1, 100, 100, 24),    # Ho = Wo = 50; C0 = 24, a partial n_tile
    (2, 64, 68, 32),      # Wo = 34 (W % 8 == 4)
    (3, 2, 4, 8),         # a 1 x 2 output
    (1, 32, 64, 24),      # 4 tiles: a grid below the SM count
    (4, 512, 512, 16),    # 2048 tiles: many per persistent CTA
]


def _stem_inputs(n, h, w, c0, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 3, h, w)).astype(np.float32)
    w1 = (rng.standard_normal((32, 27)) * 0.3).astype(np.float16)
    b1 = (rng.standard_normal(32) * 0.2).astype(np.float32)
    wdw = (rng.standard_normal((9, 32)) * 0.3).astype(np.float16)
    bdw = (rng.standard_normal(32) * 0.2).astype(np.float32)
    w3 = (rng.standard_normal((c0, 32)) / 32 ** 0.5).astype(np.float16)
    b3 = (rng.standard_normal(c0) * 0.1).astype(np.float32)
    return x, w1, b1, wdw, bdw, w3, b3


def _pw(a, wpk, bpk, m, k, n, act):
    lib = _lib.load()
    out = torch.full((m, n), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_pw1x1_f16(a.data_ptr(), wpk.data_ptr(), bpk.data_ptr(), None, out.data_ptr(), m, k, n, act,
                                stream()), "pw1x1")
    return out


def _check_stem_fused(n, h, w, c0, flip, seed):
    lib = _lib.load()
    assert lib.lp_stem_fused_supported(h, w, c0) == 1
    x, w1, b1, wdw, bdw, w3, b3 = _stem_inputs(n, h, w, c0, seed)
    x16 = x.astype(np.float16)
    ho, wo = h // 2, w // 2
    m = n * ho * wo
    what = "stem_fused n%d %dx%d c0 %d flip %d" % (n, h, w, c0, flip)
    w1p = np.zeros((32, 64), np.float16)
    w1p[:, :27] = w1
    w1d, b1d, wdd, bdd = _dev(w1p), _dev(b1), _dev(wdw), _dev(bdw)
    w3k, b3k = pack_pw(torch.from_numpy(w3), torch.from_numpy(b3))

    def fused(xin, fp32):
        xd = _dev(xin)
        y = torch.full((n, ho, wo, c0), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(lib.lp_stem_fused_f16(xd.data_ptr(), 1 if fp32 else 0, flip, w1d.data_ptr(), b1d.data_ptr(),
                                         wdd.data_ptr(), bdd.data_ptr(), w3k.data_ptr(), b3k.data_ptr(), y.data_ptr(),
                                         n, h, w, c0, stream()), "stem_fused")
        torch.cuda.synchronize()
        return y.cpu().numpy().reshape(m, c0)

    # the chain, through the C ABI
    a = cr.stem_im2col(x16, flip)
    w1k, b1k = pack_pw(torch.from_numpy(w1p[:, :32].copy()), torch.from_numpy(b1))
    e = _pw(_dev(a), w1k, b1k, m, 32, 32, de.ACT_RELU6)
    d = torch.full((n, ho, wo, 32), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_dwconv_f16(e.data_ptr(), wdd.data_ptr(), bdd.data_ptr(), d.data_ptr(), n, 32, ho, wo, 3, 1,
                                 de.ACT_RELU6, stream()), "dwconv")
    chain = _pw(d, w3k, b3k, m, 32, c0, de.ACT_NONE)
    torch.cuda.synchronize()
    e, d, chain = e.cpu().numpy(), d.cpu().numpy(), chain.cpu().numpy()

    got16 = fused(x16, False)
    assert_equal_values(got16, chain, what + " fp16 vs chain")
    got32 = fused(x, True)
    assert np.array_equal(got32.view(np.uint16), got16.view(np.uint16)), (
        "%s: the fp32 image does not give the result of its fp16 rounding (%d elements differ)"
        % (what, (got32.view(np.uint16) != got16.view(np.uint16)).sum()))

    # the chain's parts against references that run no kernel
    check_reduction(e, a[:, :27], w1, b1, None, 27, what + " conv1", de.ACT_RELU6)
    d_emul = de.dwconv(e.reshape(n, ho, wo, 32), wdw, bdw, 3, 1, de.ACT_RELU6, 2)
    assert_equal_values(d, d_emul, what + " dwconv vs dw_emul")
    check_reduction(chain, d_emul, w3, b3, None, 32, what + " 1x1")
    # both GEMMs against the tensor-core emulator, value for value, on the first and last 16384 pixels
    rows = np.r_[0:min(m, 16384), max(16384, m - 16384):m]
    assert_equal_values(e[rows], me.pw1x1(a[rows], w1p[:, :32], b1, None, de.ACT_RELU6), what + " conv1 vs mma_emul")
    assert_equal_values(chain[rows], me.pw1x1(d_emul.reshape(m, 32)[rows], w3, b3), what + " 1x1 vs mma_emul")


@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("n,h,w,c0", STEM_FUSED_SHAPES)
def test_stem_fused_equals_chain(n, h, w, c0, flip, dw_precision):
    dw_precision(2)
    _check_stem_fused(n, h, w, c0, flip, n * 1000 + h * 7 + w + c0 + flip)


@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("arch,size", cr.PLAN_SIZES)
def test_stem_fused_equals_chain_plan_shapes(arch, size, flip, dw_precision):
    """the stem launch the engine plans for LitePose-XS/S/M/L at their baseline input sizes"""
    dw_precision(2)
    n, h, w, c0 = cr.plan_stem_shape(arch, size)
    _check_stem_fused(n, h, w, c0, flip, size + flip)


# ---------------------------------------------------------------- (c) the fallback stem
# (n, h, w, fp32, offset, vector path)
STEM_CONV_CASES = [
    (2, 36, 128, False, 0, True),     # fp16, W % 8 == 0; Ho = 18
    (2, 36, 128, True, 0, True),      # fp32, W % 4 == 0
    (1, 20, 272, False, 0, True),     # Wo = 136 > 128: a third CTA column of 8 pixels
    (1, 20, 260, True, 0, True),      # Wo = 130: a third CTA column of 2 pixels
    (2, 52, 100, False, 0, False),    # fp16, W % 8 == 4; Ho = 26
    (1, 20, 260, False, 0, False),    # fp16, W % 8 == 4, a partial CTA column
    (2, 52, 98, True, 0, False),      # fp32, W % 4 == 2
    (1, 36, 128, False, 1, False),    # the image one element into its buffer: misaligned base
    (1, 36, 128, True, 1, False),
    (3, 2, 2, False, 0, False),       # H = W = 2
    (3, 2, 2, True, 0, False),
]


@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("n,h,w,fp32,offset,vec", STEM_CONV_CASES)
def test_stem_conv_bit_exact(n, h, w, fp32, offset, vec, flip):
    lib = _lib.load()
    rng = np.random.default_rng(n * 100 + h + w + fp32 + offset)
    x = rng.standard_normal((n, 3, h, w)).astype(np.float32 if fp32 else np.float16)
    wt = (rng.standard_normal((32, 27)) * 0.3).astype(np.float16)
    b = (rng.standard_normal(32) * 0.2).astype(np.float32)
    buf = _dev(np.concatenate([np.zeros(offset, x.dtype), x.ravel()]))
    xd = buf[offset:]
    assert ((xd.data_ptr() % 16 == 0) and w % (4 if fp32 else 8) == 0) == vec    # stem.cu's choice of load path
    y = torch.full((n, h // 2, w // 2, 32), float("nan"), dtype=torch.float16, device="cuda")
    wd, bd = _dev(wt), _dev(b)
    _lib.check(lib.lp_stem_conv3x3_s2(xd.data_ptr(), 1 if fp32 else 0, flip, wd.data_ptr(), bd.data_ptr(), y.data_ptr(),
                                      n, h, w, stream()), "stem")
    torch.cuda.synchronize()
    assert_equal_values(y.cpu().numpy(), cr.stem_conv(x, wt, b, flip),
                        "stem n%d %dx%d fp32 %d offset %d flip %d" % (n, h, w, fp32, offset, flip))


# ---------------------------------------------------------------- (d) fusion deconv against fp64
def _check_deconv(n, h, w, cr_, cw, co, rows):
    lib = _lib.load()
    assert cr.uses_rows_kernel(cr_, cw, co, w) == rows
    xr, xw, wr, ww, b = cr.deconv_inputs(n, h, w, cr_, cw, co, n + h * 3 + w * 5 + cr_ + cw + co)
    wp = np.zeros(lib.lp_deconv_packed_elems(cr_, cw, co), np.uint16)
    bp = np.zeros(lib.lp_deconv_packed_bias_elems(co), np.float32)
    _lib.check(lib.lp_deconv_pack(wr.view(np.uint16).ctypes.data, ww.view(np.uint16).ctypes.data, b.ctypes.data, cr_,
                                  cw, co, wp.ctypes.data, bp.ctypes.data), "deconv_pack")
    wd, bd, rd, rwd = _dev(wp.view(np.float16)), _dev(bp), _dev(xr), _dev(xw)
    out = torch.full((n, 2 * h, 2 * w, co), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_fusion_deconv_f16(rd.data_ptr(), rwd.data_ptr(), wd.data_ptr(), bd.data_ptr(), out.data_ptr(), n,
                                        h, w, cr_, cw, co, stream()), "deconv")
    torch.cuda.synchronize()
    ref, mag = cr.deconv_f64(xr, xw, wr, ww, b)
    check_bound(out.cpu().numpy(), ref, mag, 4 * (cr_ + cw),
                "deconv %s n%d %dx%d cr%d cw%d co%d" % ("rows" if rows else "tiled", n, h, w, cr_, cw, co))


@pytest.mark.parametrize("n,h,w,cr_,cw,co", cr.DECONV_ROWS_CASES)
def test_deconv_rows_fp64(n, h, w, cr_, cw, co):
    _check_deconv(n, h, w, cr_, cw, co, True)


@pytest.mark.parametrize("n,h,w,cr_,cw,co", cr.DECONV_TILED_CASES)
def test_deconv_tiled_fp64(n, h, w, cr_, cw, co):
    _check_deconv(n, h, w, cr_, cw, co, False)


@pytest.mark.parametrize("arch,size", cr.PLAN_SIZES)
def test_deconv_fp64_plan_shapes(arch, size):
    """the three deconv levels the engine plans for LitePose-XS/S/M/L at their baseline input sizes"""
    for n, h, w, cr_, cw, co in cr.plan_deconv_shapes(arch, size):
        _check_deconv(n, h, w, cr_, cw, co, cr.uses_rows_kernel(cr_, cw, co, w))
