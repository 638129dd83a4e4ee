"""The NCHW train-mode BatchNorm kernels (litepose_b200/csrc/bn_nchw_train.cu) restated on the CPU, bit for bit (test
infrastructure, numpy only).

fwd(x, gamma, beta, rmean, rvar, momentum, eps, act) -> (y, saved [4, C], new running mean, new running var) and
bwd(x, dy, gamma, saved, act) -> (dx, dgamma, dbeta) take NCHW x / dy [N,C,H,W] (fp32 or fp16) and fp32 [C] parameters,
and return what lp_bn_nchw_fwd / lp_bn_nchw_bwd write:
  - channel c's M = N*H*W values are numbered j = n * H*W + p; range r holds j in [r * RANGE, (r + 1) * RANGE); thread t
    of its CTA adds j = r * RANGE + t + 256 i in i order, in fp64 from +0; each warp's lanes are folded by the shfl_xor
    butterfly 16, 8, 4, 2, 1 (lane 0's value), the eight warps added in order, and the ranges added in order (sums()).
    A value past M is emulated as an added +0: a sum that starts at +0 never holds -0, so this is the kernel's skip;
  - forward: the pair (x, x*x); the merge is bn_train_emul.stats's fp64 derivation (the kernels share it), plus
    mean = fp32(S1 / M) and invstd = fp32(1 / sqrt(var + eps)), invstd / scale / shift / the new running variance NaN
    where fp32(mean) is not finite; y = act(fmaf(x, scale, shift)), ReLU (v <= 0 ? +0 : v),
    ReLU6 then (v >= 6 ? 6 : v), rounded once to x's dtype;
  - backward: v = fmaf(x, scale, shift), mask ReLU !(v <= 0), ReLU6 !(v <= 0) and !(v >= 6); g = mask ? dy : +0;
    xhat = fp32(fp32(x - mean) * invstd); the pair (g, g * xhat); dbeta = fp32(Sg), dgamma = fp32(Sgx),
    k = fp32(gamma * invstd), mg = fp32(Sg / M), mgx = fp32(Sgx / M); dx = fp32(k * fmaf(-xhat, mgx, fp32(g - mg))),
    rounded once more to dy's dtype.

BOUND against fp64 (u = 2^-24, fp32 inputs; exact_fwd / exact_bwd evaluate the formulas in fp64 from the same inputs,
the backward with the kernels' own activation mask, since a pre-activation within rounding of 0 or 6 may fall on
either side), elementwise:
  y      |got - exact| <= 4u (|x s| + |mean s| + |beta|) (+ half an fp16 ulp of the result for fp16), s = gamma * invstd:
         scale and shift are rounded once each and the fmaf once; the fp64 statistics add far less.
  dx     |got - exact| <= 8u |k| (|g| + |mg| + (|xhat| + |mean invstd|) |mgx|) (+ half an fp16 ulp): xhat carries three
         roundings and the saved mean one, mg / mgx / k one each, the subtraction, fmaf and product one each.
  dgamma |got - exact| <= 4u sum |g| (|xhat| + |mean invstd|) + u |exact|;  dbeta |got - exact| <= u |exact| + 2^-45 sum |g|.
bound_fwd / bound_bwd give these limits."""
import numpy as np

from conv_ref import fma32

_F64, _F32, _F16 = np.float64, np.float32, np.float16
RANGE, THREADS = 8192, 256
ACT_NONE, ACT_RELU, ACT_RELU6 = 0, 1, 2
U32 = 2.0 ** -24


def nparts(n, h, w):
    return (n * h * w + RANGE - 1) // RANGE


def workspace_bytes(n, c, h, w):
    return nparts(n, h, w) * c * 2 * 8 + 3 * c * 4


def _per_channel(a):
    """[N,C,H,W] -> [C, M] in j order"""
    a = np.asarray(a)
    n, c = a.shape[:2]
    return np.ascontiguousarray(a.reshape(n, c, -1).transpose(1, 0, 2).reshape(c, -1))


def sums(v1, v2):
    """v1, v2 [C, M] float64 -> (S1, S2) [C] in the kernels' order"""
    c, m = v1.shape
    parts = (m + RANGE - 1) // RANGE
    out = []
    for v in (v1, v2):
        p = np.zeros((c, parts * RANGE), _F64)
        p[:, :m] = v
        p = p.reshape(c, parts, RANGE // THREADS, THREADS)
        acc = np.zeros((c, parts, THREADS), _F64)
        for i in range(RANGE // THREADS):                 # each thread's values in i order
            acc = acc + p[:, :, i]
        lanes = acc.reshape(c, parts, THREADS // 32, 32)
        idx = np.arange(32)
        for o in (16, 8, 4, 2, 1):                        # the butterfly
            lanes = lanes + lanes[..., idx ^ o]
        w = lanes[..., 0]
        t = w[..., 0].copy()
        for k in range(1, THREADS // 32):                 # warps in order
            t = t + w[..., k]
        s = t[:, 0].copy()
        for r in range(1, parts):                         # ranges in order
            s = s + t[:, r]
        out.append(s)
    return out[0], out[1]


def _bcast(a, shape):
    return np.broadcast_to(np.asarray(a, _F32)[None, :, None, None], shape)


def act_fn(v, act):
    v = np.asarray(v, _F32)
    if act != ACT_NONE:
        v = np.where(v <= 0, _F32(0), v).astype(_F32)
    if act == ACT_RELU6:
        v = np.where(v >= 6, _F32(6), v).astype(_F32)
    return v


def mask_fn(v, act):
    if act == ACT_RELU:
        return ~(v <= 0)
    if act == ACT_RELU6:
        return ~(v <= 0) & ~(v >= 6)
    return np.ones(v.shape, bool)


def fwd(x, gamma, beta, rmean, rvar, momentum, eps, act):
    x = np.asarray(x)
    dt = x.dtype
    n, c, h, w = x.shape
    m = n * h * w
    xc = _per_channel(x).astype(_F64)
    s1, s2 = sums(xc, xc * xc)
    mf = _F64(m)
    mean = s1 / mf
    var = s2 / mf - mean * mean
    var = np.where(var > 0, var, _F64(0))
    var_u = var * mf / (mf - _F64(1))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        sd = np.sqrt(var + _F64(eps))
        s = np.asarray(gamma, _F32).astype(_F64) / sd
        scale = s.astype(_F32)
        shift = (np.asarray(beta, _F32).astype(_F64) - mean * s).astype(_F32)
        keep = _F64(1.0) - _F64(momentum)
        nm = (keep * np.asarray(rmean, _F32).astype(_F64) + _F64(momentum) * mean).astype(_F32)
        nv = (keep * np.asarray(rvar, _F32).astype(_F64) + _F64(momentum) * var_u).astype(_F32)
        mean32, invstd = mean.astype(_F32), (_F64(1) / sd).astype(_F32)
        bad = ~np.isfinite(mean32)                        # an inf or NaN in the channel: NaN variance
        invstd, scale, shift, nv = [np.where(bad, _F32(np.nan), a).astype(_F32) for a in (invstd, scale, shift, nv)]
        saved = np.stack([mean32, invstd, scale, shift])
        y = act_fn(fma32(x.astype(_F32), _bcast(scale, x.shape), _bcast(shift, x.shape)), act).astype(dt)
    return y, saved, nm, nv


def _xhat(x, saved):
    with np.errstate(over="ignore", invalid="ignore"):
        return ((np.asarray(x, _F32) - _bcast(saved[0], x.shape)).astype(_F32) *
                _bcast(saved[1], x.shape)).astype(_F32)


def grad_in(x, dy, saved, act):
    """g = mask ? dy : +0 (fp32)"""
    x = np.asarray(x)
    with np.errstate(over="ignore", invalid="ignore"):
        v = fma32(x.astype(_F32), _bcast(saved[2], x.shape), _bcast(saved[3], x.shape))
    return np.where(mask_fn(v, act), np.asarray(dy).astype(_F32), _F32(0)).astype(_F32)


def bwd(x, dy, gamma, saved, act):
    x, dy = np.asarray(x), np.asarray(dy)
    dt = dy.dtype
    n, c, h, w = x.shape
    m = n * h * w
    g = grad_in(x, dy, saved, act)
    xh = _xhat(x, saved)
    gc = _per_channel(g).astype(_F64)
    with np.errstate(over="ignore", invalid="ignore"):
        sg, sgx = sums(gc, gc * _per_channel(xh).astype(_F64))
        dbeta, dgamma = sg.astype(_F32), sgx.astype(_F32)
        k = (np.asarray(gamma, _F32).astype(_F64) * saved[1].astype(_F64)).astype(_F32)
        mg, mgx = (sg / _F64(m)).astype(_F32), (sgx / _F64(m)).astype(_F32)
        d = (g - _bcast(mg, x.shape)).astype(_F32)
        d = fma32(-xh, _bcast(mgx, x.shape), d)
        dx = (_bcast(k, x.shape) * d).astype(_F32).astype(dt)
    return dx, dgamma, dbeta


# ---------------------------------------------------------------- fp64 references and bounds
def exact_fwd(x, gamma, beta, eps, act):
    xd = np.asarray(x).astype(_F64)
    mean = xd.mean(axis=(0, 2, 3))
    var = ((xd - mean[None, :, None, None]) ** 2).mean(axis=(0, 2, 3))
    s = np.asarray(gamma, _F64) / np.sqrt(var + eps)
    v = (xd - mean[None, :, None, None]) * s[None, :, None, None] + np.asarray(beta, _F64)[None, :, None, None]
    if act != ACT_NONE:
        v = np.maximum(v, 0)
    if act == ACT_RELU6:
        v = np.minimum(v, 6)
    n, _, h, w = xd.shape
    return v, mean, var * (n * h * w) / (n * h * w - 1.0), s


def bound_fwd(x, gamma, beta, eps, fp16=False):
    _, mean, _, s = exact_fwd(x, gamma, beta, eps, ACT_NONE)
    b = lambda a: np.asarray(a, _F64)[None, :, None, None]
    lim = 4 * U32 * (np.abs(np.asarray(x, _F64) * b(s)) + np.abs(b(mean * s)) + np.abs(b(beta)))
    if fp16:
        ex, _, _, _ = exact_fwd(x, gamma, beta, eps, ACT_NONE)
        lim = lim + 2.0 ** -11 * np.abs(ex) + 2.0 ** -25
    return lim


def exact_bwd(x, dy, gamma, eps, saved, act):
    """fp64 dx, dgamma, dbeta with the kernels' activation mask"""
    xd = np.asarray(x).astype(_F64)
    g = grad_in(x, dy, saved, act).astype(_F64)
    mean = xd.mean(axis=(0, 2, 3))[None, :, None, None]
    var = ((xd - mean) ** 2).mean(axis=(0, 2, 3))[None, :, None, None]
    inv = 1.0 / np.sqrt(var + eps)
    xh = (xd - mean) * inv
    mg = g.mean(axis=(0, 2, 3), keepdims=True)
    mgx = (g * xh).mean(axis=(0, 2, 3), keepdims=True)
    dx = np.asarray(gamma, _F64)[None, :, None, None] * inv * (g - mg - xh * mgx)
    return dx, (g * xh).sum(axis=(0, 2, 3)), g.sum(axis=(0, 2, 3))


def bound_bwd(x, dy, gamma, eps, saved, act, fp16=False):
    xd = np.asarray(x).astype(_F64)
    g = np.abs(grad_in(x, dy, saved, act).astype(_F64))
    inv = saved[1].astype(_F64)[None, :, None, None]
    mi = np.abs(saved[0].astype(_F64)[None, :, None, None] * inv)
    xh = np.abs(xd - saved[0].astype(_F64)[None, :, None, None]) * inv
    dx64, dg64, db64 = exact_bwd(x, dy, gamma, eps, saved, act)
    mg = np.abs(g.mean(axis=(0, 2, 3), keepdims=True))
    mgx = np.abs((g * xh).mean(axis=(0, 2, 3), keepdims=True))
    k = np.abs(np.asarray(gamma, _F64)[None, :, None, None] * inv)
    ldx = 8 * U32 * k * (g + mg + (xh + mi) * mgx)
    if fp16:
        ldx = ldx + 2.0 ** -11 * np.abs(dx64) + 2.0 ** -25
    ldg = 4 * U32 * (g * (xh + mi)).sum(axis=(0, 2, 3)) + U32 * np.abs(dg64)
    ldb = U32 * np.abs(db64) + 2.0 ** -45 * g.sum(axis=(0, 2, 3))
    return ldx, ldg, ldb

