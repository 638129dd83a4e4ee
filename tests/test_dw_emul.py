"""CPU: the bit-exact depthwise emulator (dw_emul.py) checked against exact rational rounding, against a literal scalar
restatement of the dwconv.cu thread loop, and against an fp64 convolution within each mode's analytic error bound; and
the GPU exactness tests' inputs checked to be ones on which the mirror rule and the precision mode change the result."""
import math
from fractions import Fraction

import numpy as np
import pytest

import dw_emul as de


# ---------------------------------------------------------------- exact rounding of a rational
def round_frac(q, mant_bits, emin, fmax):
    """round-to-nearest-even of the rational q to a binary format with `mant_bits` fraction bits and minimum normal
    exponent emin (subnormals below); |result| > fmax -> inf"""
    if q == 0:
        return 0.0
    sign = -1 if q < 0 else 1
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    if Fraction(2) ** (e + 1) <= a:
        e += 1
    ulp = Fraction(2) ** (max(e, emin) - mant_bits)
    m = a / ulp
    fl = m.numerator // m.denominator
    rem = m - fl
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
        fl += 1
    v = fl * ulp
    if v > fmax:
        return sign * math.inf
    return sign * float(v)


def r16_exact(q):
    return round_frac(q, 10, -14, Fraction(65504) + Fraction(16))   # 65520 and above round to inf


def r32_exact(q):
    return round_frac(q, 23, -126, Fraction(2) ** 128)


def _f(v):
    return Fraction(float(v))


def _fp16_values(rng, n):
    """random finite fp16 values over the whole range: normals of every exponent, subnormals, signs"""
    bits = rng.integers(0, 0x7C00, n, dtype=np.uint16) | (rng.integers(0, 2, n, dtype=np.uint16) << 15)
    return bits.view(np.float16)


def _near_midpoint_triples(rng, n):
    """(a, b, c) with a*b + c within a few 2^-22 ulps of an fp16 rounding midpoint above c"""
    out = []
    while len(out) < n:
        c = np.float16(rng.uniform(-4, 4))
        if c == 0:
            continue
        ulp = float(np.spacing(np.abs(c)))
        target = ulp / 2 * (1 if rng.integers(2) else -1) * (1 + 2 * rng.integers(0, 3))
        a = np.float16(rng.uniform(1, 2) * (1 if rng.integers(2) else -1))
        b = np.float16(target / float(a))
        if np.isfinite(b) and b != 0:
            out.append((a, b, c))
    return out


def test_primitives_random_triples():
    rng = np.random.default_rng(1)
    a, b, c = (_fp16_values(rng, 4000) for _ in range(3))
    # keep the products finite in fp16 range for the chain ops
    ok = np.abs(a.astype(np.float64) * b.astype(np.float64)) < 60000
    a, b, c = a[ok], b[ok], c[ok]
    got_fma, got_mul, got_add = de.hfma(a, b, c), de.hmul(a, b), de.hadd(a, c)
    got_ffma = de.fhfma(a, b, c.astype(np.float32))
    for i in range(a.size):
        fa, fb, fc = _f(a[i]), _f(b[i]), _f(c[i])
        assert float(got_fma[i]) == r16_exact(fa * fb + fc), (a[i], b[i], c[i])
        assert float(got_mul[i]) == r16_exact(fa * fb), (a[i], b[i])
        assert float(got_add[i]) == r16_exact(fa + fc), (a[i], c[i])
        assert float(got_ffma[i]) == r32_exact(fa * fb + fc), (a[i], b[i], c[i])


def test_primitives_near_midpoints():
    rng = np.random.default_rng(2)
    triples = _near_midpoint_triples(rng, 3000)
    # hand-made: exact ties (to even, both directions) and one 2^-20 above / below a tie
    one, t11 = np.float16(1.0), np.float16(2.0 ** -11)
    triples += [(t11, one, one), (t11, one, np.float16(1 + 2.0 ** -10)), (t11, np.float16(-1.0), one),
                (np.float16(2.0 ** -11 * (1 + 2.0 ** -10)), one, one),
                (np.float16(2.0 ** -12 * (2 - 2.0 ** -10)), one, one)]
    a, b, c = (np.array(v, np.float16) for v in zip(*triples))
    got = de.hfma(a, b, c)
    via32 = (a.astype(np.float32) * b.astype(np.float32) + c.astype(np.float32)).astype(np.float16)
    double_rounded = 0
    for i in range(a.size):
        want = r16_exact(_f(a[i]) * _f(b[i]) + _f(c[i]))
        assert float(got[i]) == want, (a[i], b[i], c[i], got[i], want)
        double_rounded += float(via32[i]) != want
    # the cases are sharp enough that the float32 route (double rounding) gets some of them wrong
    assert double_rounded > 0
    assert de.hfma(t11, one, one) == one                                   # tie -> even (1.0)
    assert de.hfma(t11, one, np.float16(1 + 2.0 ** -10)) == np.float16(1 + 2.0 ** -9)


def test_primitives_subnormals():
    rng = np.random.default_rng(3)
    sub = (rng.integers(1, 0x400, 3000, dtype=np.uint16) | (rng.integers(0, 2, 3000, dtype=np.uint16) << 15)).view(
        np.float16)
    small = np.float16(rng.uniform(-8, 8, 3000))
    a, b, c = small, np.roll(small, 7), sub
    for x, y, z in ((a, b, c), (sub, small, np.roll(sub, 3)), (sub, np.roll(sub, 5), sub)):
        got = de.hfma(x, y, z)
        gm, ga = de.hmul(x, y), de.hadd(x, z)
        for i in range(x.size):
            fx, fy, fz = _f(x[i]), _f(y[i]), _f(z[i])
            assert float(got[i]) == r16_exact(fx * fy + fz)
            assert float(gm[i]) == r16_exact(fx * fy)
            assert float(ga[i]) == r16_exact(fx + fz)
    assert de.r16(2.0 ** -25) == 0 and de.r16(2.0 ** -25 * 1.5) == np.float16(2.0 ** -24)   # smallest subnormal


# ---------------------------------------------------------------- scalar restatement of the dwconv.cu thread loop
def kernel_loop(x, w, bias, k, s, act, prec):
    """One channel: x [H, W] fp16, w [k*k] fp16, bias float -> [H/s, W/s] fp16, computed tile by tile, micro-block by
    micro-block exactly as dwconv_kernel does (slot array in[], j, kx, mirrored weights / columns / stores)."""
    H, W = x.shape
    Ho, Wo = H // s, W // s
    TH = TW = 32 if s == 1 else 16
    IC = IR = 3 * s + k
    PAIRS_X, NPAIRS = TW // 8, (TH // 4) * (TW // 8)
    y = np.full((Ho, Wo), np.nan, np.float16)

    def tile_px(r, c, oy0, ox0):   # the TMA-staged haloed tile, zero outside the image
        gy, gx = oy0 * s - k // 2 + r, ox0 * s - k // 2 + c
        return x[gy, gx] if 0 <= gy < H and 0 <= gx < W else np.float16(0)

    for ty in range((Ho + TH - 1) // TH):
        for tx in range((Wo + TW - 1) // TW):
            oy0, ox0 = ty * TH, tx * TW
            for q in range(NPAIRS):
                for sub in (0, 1):
                    mir = s == 1 and sub == 1
                    by, bx = q // PAIRS_X, (q % PAIRS_X) * 2 + sub
                    oy, ox = by * 4, bx * 4
                    if oy0 + oy >= Ho or ox0 + ox >= Wo:
                        continue
                    wreg = [w[ky * k + (k - 1 - kx if mir else kx)] for ky in range(k) for kx in range(k)]
                    acc = [[np.float32(bias)] * 4 for _ in range(4)]
                    acch = [[np.float16(bias)] * 4 for _ in range(4)]
                    part = [[None] * 4 for _ in range(4)]
                    for r in range(IR):
                        inp = [tile_px(oy * s + r, ox * s + (IC - 1 - c if mir else c), oy0, ox0) for c in range(IC)]
                        for i in range(4):
                            ky = r - i * s
                            if not 0 <= ky < k:
                                continue
                            for j in range(4):
                                if prec == 0:
                                    for kx in range(k):
                                        acc[i][j] = de.fhfma(inp[j * s + kx], wreg[ky * k + kx], acc[i][j])
                                elif prec == 1:
                                    sacc = de.hmul(inp[j * s], wreg[ky * k])
                                    for kx in range(1, k):
                                        sacc = de.hfma(inp[j * s + kx], wreg[ky * k + kx], sacc)
                                    acc[i][j] = de.fhadd(sacc, acc[i][j])
                                else:
                                    for kx in range(k):
                                        if ky % 2 == 0 and kx == 0:
                                            part[i][j] = de.hmul(inp[j * s + kx], wreg[ky * k + kx])
                                        else:
                                            part[i][j] = de.hfma(inp[j * s + kx], wreg[ky * k + kx], part[i][j])
                                    if ky % 2 == 1 or ky == k - 1:
                                        acch[i][j] = de.hadd(acch[i][j], part[i][j])
                    for i in range(4):
                        for j in range(4):
                            jj = 3 - j if mir else j
                            if oy0 + oy + i < Ho and ox0 + ox + jj < Wo:
                                if prec == 2:
                                    v = de.act_f16(np.float16(acch[i][j]), act)
                                else:
                                    v = np.float16(de.act_f32(np.float32(acc[i][j]), act))
                                y[oy0 + oy + i, ox0 + ox + jj] = v
    return y


@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("s", [1, 2])
@pytest.mark.parametrize("prec", [0, 1, 2])
def test_emulator_matches_scalar_kernel_loop(k, s, prec):
    """maps with W in {5, 6, 9, 12}: partial mirrored micro-blocks (mirrored stores clipped at W); two channels"""
    for idx, (h, w) in enumerate([(6, 5), (4, 6), (7, 9), (10, 12)]):
        if s == 2:
            h, w = 2 * h, 2 * w
        x, wt, b = de.make_inputs(1, 2, h, w, k, ("signed", "relu6", "tiny", "signed")[idx], 100 * k + 10 * s + idx)
        act = idx % 3
        got = de.dwconv(x, wt, b, k, s, act, prec)
        for ch in range(2):
            want = kernel_loop(x[0, :, :, ch], wt[:, ch], b[ch], k, s, act, prec)
            assert not np.isnan(want).any()
            np.testing.assert_array_equal(got[0, :, :, ch], want, err_msg="k%d s%d prec%d %dx%d" % (k, s, prec, h, w))


@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("s", [1, 2])
@pytest.mark.parametrize("prec", [0, 1, 2])
def test_emulator_within_analytic_bound(k, s, prec):
    """every mode against the fp64 convolution: |err| <= 2^-11 |ref| + n_r u S + k^2 2^-24, where S = sum |x w| + |b|
    and n_r u bounds the accumulated rounding (fp32: k^2 + 1 roundings of u = 2^-24; fp16: k^2 taps + row folds + the
    fp16 bias, u = 2^-11)"""
    x, wt, b = de.make_inputs(2, 48, 20, 28, k, "signed", k + s + prec)
    got = de.dwconv(x, wt, b, k, s, de.ACT_NONE, prec).astype(np.float64)
    ref, mag = de.conv_f64(x, wt, b, k, s)
    n_r, u = (k * k + 1, 2.0 ** -24) if prec == 0 else (k * k + k + 2, 2.0 ** -11)
    bound = 2.0 ** -11 * np.abs(ref) + n_r * u * mag + k * k * 2.0 ** -24
    ratio = (np.abs(got - ref) / bound).max()
    assert ratio <= 1.0, ratio


def test_mirror_and_precision_change_the_gpu_test_inputs():
    """on the inputs of tests/test_gpu_dw_exact.py, the mirror rule changes the result of every stride-1 mode and the
    three precision modes differ pairwise: a kernel that ignored either would fail those exactness tests"""
    from test_gpu_dw_exact import prec_switch_case, dw_cases

    for k in (3, 5, 7):
        n, c, h, w, kind, seed = prec_switch_case(k)
        x, wt, b = de.make_inputs(n, c, h, w, k, kind, seed)
        outs = [de.dwconv(x, wt, b, k, 1, de.ACT_RELU6, p) for p in (0, 1, 2)]
        for p, q in ((0, 1), (0, 2), (1, 2)):
            assert (outs[p] != outs[q]).any(), "k%d: prec %d and %d agree" % (k, p, q)
        for p in (1, 2):
            flat = de.dwconv(x, wt, b, k, 1, de.ACT_RELU6, p, mirror=False)
            assert (flat != outs[p]).any(), "k%d prec %d: the mirror rule changes nothing" % (k, p)
    # and in the per-(k, s, prec, act) cases: every stride-1 case with an fp16 mode sees the mirror rule
    for k in (3, 5, 7):
        for prec in (1, 2):
            n, c, h, w, kind, seed = dw_cases(k, 1, prec, de.ACT_RELU6)[0]
            x, wt, b = de.make_inputs(n, c, h, w, k, kind, seed)
            a = de.dwconv(x, wt, b, k, 1, de.ACT_RELU6, prec)
            assert (a != de.dwconv(x, wt, b, k, 1, de.ACT_RELU6, prec, mirror=False)).any()
            assert (a != de.dwconv(x, wt, b, k, 1, de.ACT_RELU6, 0)).any()
