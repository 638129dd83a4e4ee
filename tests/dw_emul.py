"""Bit-exact CPU emulation of the depthwise arithmetic of every kernel (test infrastructure, numpy only).  It lives in one
place on the device, dw_inner.cuh: dwconv(..., prec) restates its dw_ffma (prec 0), dw_rowsum (prec 1) and dw_hfma2
(prec 2), which lp_dwconv_f16 (dwconv.cu), the fused block kernels (dwpw.cu, dwblock.cu), the fused stem and the heads call.

Every step of the kernels' arithmetic has a unique correctly rounded result, so it can be restated exactly:
  - an fp16 x fp16 product is exact in fp32 (22 significant bits), so fp32 `x*w + acc` in numpy is the kernels' fmaf;
  - an HFMA2 / HMUL2 / HADD2 lane is one correctly rounded fp16 value.  It is computed here in float64 and rounded once
    with numpy's float64 -> float16 conversion (round to nearest even).  With fp16 operands a*b + c is exact in float64
    for every finite fp16 result (|a*b| < 2^16, lowest bit >= 2^-48), so that single rounding is the hardware's.
    Rounding through float32 instead (or torch's CPU double -> half, which goes through float) would double-round
    results that sit just above an fp16 midpoint.

Precision modes (lp_set_dw_precision):
  0  acc = bias (fp32); every tap in kernel-row order acc = fmaf(x, w, acc); activation in fp32, then -> fp16
  1  per kernel row an fp16 chain (hmul on the first tap, hfma on the rest), each row sum added to the fp32 accumulator
  2  running fp16 total seeded with fp16(bias); kernel rows {0,1}, {2,3}, {4,5}, {6} form one chain each (hmul at even
     ky, kx = 0, then hfma), folded into the total with hadd after an odd ky or the last ky; hmax / hmin activation
Mirrored lanes: at stride 1 the half-warp with sub = 1 takes the x-odd 4x4 micro-block and walks the kx taps of every
kernel row from k-1 down to 0.  Every kernel tiles x in multiples of 16 pixels, so an output pixel with (x // 4) % 2 == 1
accumulates each row in reverse kx order (mirror=False drops the rule, for tests that must see it matter)."""
import numpy as np

ACT_NONE, ACT_RELU, ACT_RELU6 = 0, 1, 2
_F64, _F32, _F16 = np.float64, np.float32, np.float16


def r16(v):
    """float64 -> fp16, one round-to-nearest-even rounding (overflow -> inf, as on the GPU)"""
    with np.errstate(over="ignore"):
        return np.asarray(v, _F64).astype(_F16)


def hmul(a, b):
    return r16(np.asarray(a, _F64) * np.asarray(b, _F64))


def hfma(a, b, c):
    return r16(np.asarray(a, _F64) * np.asarray(b, _F64) + np.asarray(c, _F64))


def hadd(a, b):
    return r16(np.asarray(a, _F64) + np.asarray(b, _F64))


def fhfma(a, b, c):
    """fmaf(fp16 a, fp16 b, fp32 c): the product is exact in fp32, so the fp32 add is the only rounding"""
    return np.asarray(a, _F16).astype(_F32) * np.asarray(b, _F16).astype(_F32) + np.asarray(c, _F32)


def fhadd(a, c):
    return np.asarray(a, _F16).astype(_F32) + np.asarray(c, _F32)


def act_f32(v, act):
    if act == ACT_RELU:
        return np.maximum(v, _F32(0))
    if act == ACT_RELU6:
        return np.minimum(np.maximum(v, _F32(0)), _F32(6))
    return v


def act_f16(v, act):
    if act != ACT_NONE:
        v = np.maximum(v, _F16(0))
    if act == ACT_RELU6:
        v = np.minimum(v, _F16(6))
    return v


def mirrored_columns(wout, stride, mirror=True):
    """bool [Wout]: output columns whose kernel rows are accumulated from kx = k-1 down to 0"""
    x = np.arange(wout)
    if not mirror or stride != 1:
        return np.zeros(wout, bool)
    return (x // 4) % 2 == 1


def dwconv(x, w, bias, k, stride, act, prec, mirror=True):
    """x [N,H,W,C] fp16 (NHWC), w [k*k, C] fp16 (tap-major), bias [C] fp32 or None -> [N,H/s,W/s,C] fp16, bit-exact
    with lp_dwconv_f16 at precision `prec` (and, for k = 7, stride 1, ReLU6, prec 2, with the fused kernels' depthwise)."""
    x = np.asarray(x, _F16)
    w = np.asarray(w, _F16)
    n, h, wd, c = x.shape
    assert w.shape == (k * k, c) and k in (3, 5, 7) and stride in (1, 2) and prec in (0, 1, 2)
    ho, wo = h // stride, wd // stride
    p = k // 2
    xp = np.zeros((n, h + 2 * p + stride, wd + 2 * p + stride, c), _F16)
    xp[:, p:p + h, p:p + wd] = x
    b32 = np.zeros(c, _F32) if bias is None else np.asarray(bias, _F32)
    mir = mirrored_columns(wo, stride, mirror)
    ox = np.arange(wo) * stride
    rows = np.arange(ho) * stride

    def tap(ky, t):
        """input and weight of kx step t of kernel row ky, per output column ([N,Ho,Wo,C], [Wo,C])"""
        if not mir.any():
            return xp[:, ky:ky + stride * ho:stride, t:t + stride * wo:stride], w[ky * k + t]
        kx = np.where(mir, k - 1 - t, t)
        xs = xp[:, rows + ky][:, :, ox + kx]
        return xs, w[ky * k + kx]

    if prec == 0:
        acc = np.broadcast_to(b32, (n, ho, wo, c)).copy()
        for ky in range(k):
            for t in range(k):
                xs, ws = tap(ky, t)
                acc = fhfma(xs, ws, acc)
        return act_f32(acc, act).astype(_F16)
    if prec == 1:
        acc = np.broadcast_to(b32, (n, ho, wo, c)).copy()
        for ky in range(k):
            xs, ws = tap(ky, 0)
            s = hmul(xs, ws)
            for t in range(1, k):
                xs, ws = tap(ky, t)
                s = hfma(xs, ws, s)
            acc = fhadd(s, acc)
        return act_f32(acc, act).astype(_F16)
    acch = np.broadcast_to(b32.astype(_F16), (n, ho, wo, c)).copy()
    part = None
    for ky in range(k):
        for t in range(k):
            xs, ws = tap(ky, t)
            part = hmul(xs, ws) if (ky % 2 == 0 and t == 0) else hfma(xs, ws, part)
        if ky % 2 == 1 or ky == k - 1:
            acch = hadd(acch, part)
    return act_f16(acch, act)


def default_prec(k):
    """lp_set_dw_precision(-1): packed fp16 for the backbone / stem kernel sizes, fp32 for the k = 5 heads"""
    return 0 if k == 5 else 2


# ---------------------------------------------------------------- seeded inputs shared by the CPU and GPU tests
def make_inputs(n, c, h, w, k, kind, seed):
    """x [N,H,W,C] fp16, tap-major weights [k*k, C] fp16, bias [C] fp32.

    kind 'relu6':  ReLU6-range activations (what the 1x1 expansions feed the depthwise), BN-folded weight scales
    kind 'signed': signed randn activations
    kind 'tiny':   signed randn with the first 32-channel slab scaled to ~1e-4, so that its products and partial sums
                   are fp16 subnormals
    BN folding multiplies each channel's kernel by gamma / sqrt(var + eps): the weights get a log-normal per-channel
    scale on top of a 1/k fan-in scale, and the bias a spread comparable to the activations."""
    rng = np.random.default_rng(seed)
    if kind == "relu6":
        x = np.clip(rng.standard_normal((n, h, w, c)) * 2.0 + 1.0, 0.0, 6.0)
    else:
        x = rng.standard_normal((n, h, w, c))
    if kind == "tiny":
        x[..., :32] *= 1e-4
    scale = np.exp(rng.standard_normal(c) * 0.5) / k
    wt = rng.standard_normal((k * k, c)) * scale
    bias = rng.standard_normal(c) * 0.5
    if kind == "tiny":
        wt[:, :32] = np.clip(wt[:, :32], -0.5, 0.5)
        bias[:32] *= 1e-4
    return x.astype(_F16), wt.astype(_F16), bias.astype(_F32)


def conv_f64(x, w, bias, k, stride):
    """plain fp64 depthwise convolution (no activation), [N,Ho,Wo,C] float64, plus sum |x*w| + |bias| per output"""
    x = np.asarray(x, _F64)
    w = np.asarray(w, _F64)
    n, h, wd, c = x.shape
    ho, wo = h // stride, wd // stride
    p = k // 2
    xp = np.zeros((n, h + 2 * p + stride, wd + 2 * p + stride, c))
    xp[:, p:p + h, p:p + wd] = x
    b = np.zeros(c) if bias is None else np.asarray(bias, _F64)
    out = np.broadcast_to(b, (n, ho, wo, c)).copy()
    mag = np.broadcast_to(np.abs(b), (n, ho, wo, c)).copy()
    for ky in range(k):
        for kx in range(k):
            prod = xp[:, ky:ky + stride * ho:stride, kx:kx + stride * wo:stride] * w[ky * k + kx]
            out += prod
            mag += np.abs(prod)
    return out, mag
