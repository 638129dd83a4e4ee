"""CPU: the references of test_gpu_stem_deconv_exact.py checked on their own, and the kernel selection of the deconv.

(a) conv_ref.fma32 is fmaf, correctly rounded, against fractions.Fraction: random triples, exact ties on fp32 midpoints
    and triples whose float64 sum lands on a midpoint that the exact sum is not on.
(b) conv_ref.stem_conv equals float64 conv2d up to the fp32 accumulation and one fp16 rounding, and reads the mirror.
(c) conv_ref.deconv_f64 (torch conv_transpose2d) equals the kernels' sub-pixel form summed directly.
(d) The case lists reach the kernels they claim: lp_deconv_packed_elems carries the row-kernel weights exactly when the
    channels qualify, and the tiled cases cover every tile width of pick_spatial_tile."""
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_ref as cr
from litepose_b200 import _lib


# ---------------------------------------------------------------- (a) fma32
def _fma_exact(x, w, c):
    """fmaf(x, w, c) through exact rationals: the fp32 value nearest x*w + c, ties to the even significand"""
    v = Fraction(float(x)) * Fraction(float(w)) + Fraction(float(c))
    f = np.float32(float(v))
    while Fraction(float(f)) > v:
        f = np.nextafter(f, np.float32(-np.inf))
    while Fraction(float(np.nextafter(f, np.float32(np.inf)))) <= v:
        f = np.nextafter(f, np.float32(np.inf))
    if Fraction(float(f)) == v:
        return f
    g = np.nextafter(f, np.float32(np.inf))
    dl, dh = v - Fraction(float(f)), Fraction(float(g)) - v
    if dl != dh:
        return f if dl < dh else g
    return f if int(np.array(f).view(np.int32)) & 1 == 0 else g


def _check_fma(x, w, c):
    x, w, c = np.asarray(x, np.float32), np.asarray(w, np.float16), np.asarray(c, np.float32)
    got = cr.fma32(x, w, c)
    for i in range(x.size):
        want = _fma_exact(x.flat[i], w.flat[i], c.flat[i])
        assert got.flat[i].view(np.int32) == np.array(want).view(np.int32), (
            "fma32(%r, %r, %r) = %r, exact %r" % (x.flat[i], w.flat[i], c.flat[i], got.flat[i], want))
    return got


def test_fma32_random_triples():
    rng = np.random.default_rng(0)
    m = 4000
    x = (rng.standard_normal(m) * np.exp2(rng.integers(-8, 8, m))).astype(np.float32)
    w = (rng.standard_normal(m) * 0.3).astype(np.float16)
    c = (rng.standard_normal(m) * np.exp2(rng.integers(-8, 8, m))).astype(np.float32)
    c[:200] = -(x[:200].astype(np.float64) * w[:200]).astype(np.float32)     # near-total cancellation
    _check_fma(x, w, c)


def _power_of_two_neighbours():
    """(W, M, d): odd 11-bit W, 24-bit M with M * W = 2^34 + d, 0 < |d| < 32 -- a product within 2^-29 of a power of two
    that needs more than 29 significant bits"""
    out = []
    for wi in range(1025, 2048, 2):
        for d in range(-31, 32):
            if d and (2 ** 34 + d) % wi == 0:
                mi = (2 ** 34 + d) // wi
                if 2 ** 23 <= mi < 2 ** 24:
                    out.append((wi, mi, d))
    return out


def test_fma32_midpoint_triples():
    """c = a (fp32) and x*w = half an ulp of a: an exact tie, which goes to the even one of a and its successor; and x*w
    = half an ulp times (1 + d 2^-34): the exact sum lies just off the midpoint, but float64 rounds it onto it, so only
    the TwoSum error tells the direction"""
    rng = np.random.default_rng(1)
    xs, ws, cs = [], [], []
    near = _power_of_two_neighbours()
    assert len(near) >= 8, "no 35-bit products next to a power of two"
    for i in range(400):
        a = np.float32(rng.uniform(1.0, 2.0) * 2.0 ** int(rng.integers(-20, 20)) * (1 if i % 2 else -1))
        half_ulp = (float(np.nextafter(abs(a), np.float32(np.inf))) - float(abs(a))) / 2
        sgn = 1.0 if a > 0 else -1.0
        if i % 3 == 0:                                                   # exact tie: x = half ulp / w, w a power of two
            wv = 2.0 ** int(rng.integers(-3, 3))
            xs.append(np.float32(sgn * half_ulp / wv))
            ws.append(wv)
        else:                                                            # x*w = +-half ulp (1 + d 2^-34), d != 0
            wi, mi, d = near[i % len(near)]
            wv = wi * 2.0 ** -10                                         # fp16: 11-bit odd significand
            xv = mi * 2.0 ** -24 * half_ulp                              # fp32: 24-bit significand
            s = sgn if i % 3 == 1 else -sgn                              # toward or away from zero
            xs.append(np.float32(s * xv / 2.0 ** (34 - 24 - 10)))
            ws.append(wv)
        cs.append(a)
    x, w, c = np.array(xs, np.float32), np.array(ws, np.float16), np.array(cs, np.float32)
    assert (x.astype(np.float64) * w.astype(np.float64) != 0).all()
    got = _check_fma(x, w, c)
    naive = (x.astype(np.float64) * w.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    assert (naive != got).sum() >= 50, "the triples do not separate fma32 from a rounding through float64"


# ---------------------------------------------------------------- (b) stem reference
@pytest.mark.parametrize("fp32", [False, True])
@pytest.mark.parametrize("flip", [False, True])
def test_stem_conv_reference(fp32, flip):
    rng = np.random.default_rng(2)
    x = rng.standard_normal((2, 3, 10, 14)).astype(np.float32)
    if not fp32:
        x = x.astype(np.float16)
    w = (rng.standard_normal((32, 27)) * 0.3).astype(np.float16)
    b = (rng.standard_normal(32) * 0.2).astype(np.float32)
    got = cr.stem_conv(x, w, b, flip)
    src = torch.from_numpy(x.astype(np.float64))
    if flip:
        src = torch.flip(src, [3])
    ref = F.conv2d(src, torch.from_numpy(w.astype(np.float64)).view(32, 3, 3, 3),
                   torch.from_numpy(b.astype(np.float64)), 2, 1).clamp(0, 6).permute(0, 2, 3, 1).numpy()
    # 27 fp32 roundings of partial sums <= 27 * 2^-24 * sum |x w| + |b|, then one fp16 rounding
    mag = F.conv2d(src.abs(), torch.from_numpy(np.abs(w.astype(np.float64))).view(32, 3, 3, 3), None, 2, 1)
    mag = mag.permute(0, 2, 3, 1).numpy() + np.abs(b)
    assert got.shape == ref.shape and got.dtype == np.float16
    assert (np.abs(got.astype(np.float64) - ref) <= 2.0 ** -11 * np.abs(ref) + 27 * 2.0 ** -24 * mag + 2.0 ** -25).all()
    a = cr.stem_im2col(x.astype(np.float16), flip)
    assert a.shape == (2 * 5 * 7, 32) and not a[:, 27:].any()
    pre = a[:, :27].astype(np.float64) @ w.astype(np.float64)[:, :27].T + b
    if not fp32:
        assert np.allclose(np.clip(pre, 0, 6), ref.reshape(-1, 32), rtol=0, atol=1e-12)


def test_stem_conv_fp16_path_is_fma32():
    """for fp16 images the shortcut (fp32 product, fp32 add) and fma32 agree: an fp16 x fp16 product is exact in fp32"""
    rng = np.random.default_rng(3)
    x = rng.standard_normal(20000).astype(np.float16)
    w = (rng.standard_normal(20000) * 0.3).astype(np.float16)
    c = rng.standard_normal(20000).astype(np.float32)
    short = x.astype(np.float32) * w.astype(np.float32) + c
    assert np.array_equal(short.view(np.int32), cr.fma32(x.astype(np.float32), w, c).view(np.int32))


# ---------------------------------------------------------------- (c) deconv reference
@pytest.mark.parametrize("n,h,w,cin,co", [(1, 1, 1, 8, 8), (2, 3, 5, 8, 16), (1, 6, 4, 24, 8)])
def test_deconv_f64_equals_subpixel_sum(n, h, w, cin, co):
    xr, xw, wr, ww, b = cr.deconv_inputs(n, h, w, cin, 16, co, n + h + w + cin)
    ref, mag = cr.deconv_f64(xr, xw, wr, ww, b)
    direct = cr.deconv_subpixel(xr, wr) + cr.deconv_subpixel(xw, ww) + b.astype(np.float64)
    assert ref.shape == (n, 2 * h, 2 * w, co)
    assert np.allclose(ref, np.maximum(direct, 0), rtol=1e-12, atol=1e-12)
    dmag = (cr.deconv_subpixel(np.abs(xr), np.abs(wr)) + cr.deconv_subpixel(np.abs(xw), np.abs(ww)) +
            np.abs(b.astype(np.float64)))
    assert np.allclose(mag, dmag, rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------- (d) kernel selection
def _packed_elems_split(cr_, cw, co):
    lib = _lib.load()
    total = lib.lp_deconv_packed_elems(cr_, cw, co)
    tiled = cr.tiled_packed_elems(cr_, cw, co)
    assert total in (tiled, tiled + 16 * cr.round16(co) * 64), (cr_, cw, co, total, tiled)
    return total != tiled


def test_deconv_row_weights_packed_exactly_when_channels_qualify():
    for cr_ in range(8, 72, 8):
        for cw in range(8, 72, 8):
            for co in range(8, 72, 8):
                assert _packed_elems_split(cr_, cw, co) == cr.rows_channels_ok(cr_, cw, co), (cr_, cw, co)


def test_deconv_cases_reach_the_kernel_they_name():
    for n, h, w, cr_, cw, co in cr.DECONV_ROWS_CASES:
        assert cr.uses_rows_kernel(cr_, cw, co, w) and _packed_elems_split(cr_, cw, co)
    for n, h, w, cr_, cw, co in cr.DECONV_TILED_CASES:
        assert not cr.uses_rows_kernel(cr_, cw, co, w)
    tiled = cr.DECONV_TILED_CASES
    assert {cr.pick_spatial_tile(h, w) for n, h, w, _, _, _ in tiled} == {8, 16, 32}
    assert any(w == 63 and cr.rows_channels_ok(a, b, c) for n, h, w, a, b, c in tiled)
    assert {c for *_, c in tiled} >= {40, 48, 56, 64}
    assert max(cr.tiled_packed_elems(a, b, c) // (16 * cr.round16(c) * 64) for n, h, w, a, b, c in tiled) == 5
    rows = cr.DECONV_ROWS_CASES
    assert {c for *_, c in rows} == {8, 16, 24, 32}
    assert {(a + b) // 8 for n, h, w, a, b, c in rows} >= {3, 5, 7, 8}
    assert any(w == 64 for n, h, w, *_ in rows) and any(h == 1 for n, h, *_ in rows)
    assert any(w % 128 for n, h, w, *_ in rows if w > 128)


def test_pick_spatial_tile_rule():
    assert cr.pick_spatial_tile(4, 32) == 32 and cr.pick_spatial_tile(8, 16) == 16 and cr.pick_spatial_tile(16, 8) == 8
    assert cr.pick_spatial_tile(12, 63) == 32            # ties keep the widest tile


def test_plan_shapes():
    """the baseline sizes run the fused stem, and their deconv levels include both kernels"""
    lib = _lib.load()
    kinds = set()
    for arch, size in cr.PLAN_SIZES:
        n, h, w, c0 = cr.plan_stem_shape(arch, size)
        assert (n, h, w) == (1, size, size) and lib.lp_stem_fused_supported(h, w, c0) == 1
        for n, h, w, a, b, c in cr.plan_deconv_shapes(arch, size):
            kinds.add(cr.uses_rows_kernel(a, b, c, w))
    assert kinds == {True, False}
    assert cr.plan_deconv_shapes("L", 640)[0] == (1, 40, 40, 160, 96, 64)
