"""The NCHW depthwise training kernels (litepose_b200/csrc/dw_train.cu) restated on the CPU, bit for bit (test
infrastructure, numpy only).

fwd(x, w, s), dgrad(dy, w, s, h, w_), wgrad(x, dy, s) take NCHW arrays x [N,C,H,W], dy [N,C,Ho,Wo] and w [C,k,k]
(or [C,1,k,k]), all fp32 or all fp16, and return what lp_dw_nchw_fwd / _dgrad / _wgrad write, in the same dtype:
  - operands are converted exactly to fp32; every sum is an fp32 fmaf chain from +0 (conv_ref.fma32: the product of two
    fp32 values is exact in fp64, so its TwoSum rounding is fmaf's), an fp16 result that fp32 value rounded once;
  - forward: taps ky = 0..k-1 (outer), kx = 0..k-1 (inner), inputs outside the plane +0;
  - dgrad: taps ky = k-1..0, kx = k-1..0 with (i + p - k_) a multiple of s in both axes, dy outside its plane +0;
  - wgrad: per range (128 output rows x 32 columns of one image) and thread (lane tx, warp ty) an fmaf chain over the
    thread's pixels (oy0 + 32q + 4ty + r, ox0 + tx), q then r, those inside the plane only; the lanes folded by the
    shfl_xor butterfly 16, 8, 4, 2, 1 and the warps added in order, in fp32; the range partials added in fp64 in range
    order, rounded to fp32 (then fp16).
A pixel outside the plane is emulated as a product of +0 * +0: an fmaf chain that starts at +0 never holds -0, so
adding +0 leaves it unchanged, exactly as the kernel's skip does.

BOUND (fp64 reference, fp32 operands, u = 2^-24), elementwise over the outputs:
  forward / dgrad  |got - exact| <= k^2 u * sum |x * w| over the taps (+ half an fp16 ulp of the result for fp16);
  wgrad            |got - exact| <= (4 * DWT_PASSES + 5 + 7 + 2) u * sum |x * dy| (+ half an fp16 ulp for fp16):
                   at most 16 fmaf roundings per thread chain, 5 butterfly and 7 warp additions, the fp64 merge and the
                   final rounding each below u of the sum of magnitudes.
bound_fwd / bound_dgrad / bound_wgrad give these limits from fp64 arithmetic."""
import numpy as np

from conv_ref import fma32

_F64, _F32, _F16 = np.float64, np.float32, np.float16
TILE, ROWS, PASSES, WARPS = 32, 4, 4, 8
U32 = 2.0 ** -24


def _w(w):
    w = np.asarray(w)
    return w.reshape(w.shape[0], w.shape[-2], w.shape[-1])


def out_size(h, s):
    return (h - 1) // s + 1


def _pad(a, p):
    return np.pad(np.asarray(a, _F32), ((0, 0), (0, 0), (p, p + 1), (p, p + 1)))


def fwd(x, w, s):
    x = np.asarray(x)
    dt = x.dtype
    w = _w(w).astype(_F32)
    n, c, h, wd = x.shape
    k = w.shape[-1]
    p = k // 2
    ho, wo = out_size(h, s), out_size(wd, s)
    xp = _pad(x, p)
    acc = np.zeros((n, c, ho, wo), _F32)
    for ky in range(k):
        for kx in range(k):
            xs = xp[:, :, ky:ky + (ho - 1) * s + 1:s, kx:kx + (wo - 1) * s + 1:s]
            acc = fma32(xs, w[None, :, ky, kx, None, None], acc)
    return acc.astype(dt)


def dgrad(dy, w, s, h, wd):
    """dx [N,C,h,wd] of dy [N,C,Ho,Wo]"""
    dy = np.asarray(dy)
    dt = dy.dtype
    w = _w(w).astype(_F32)
    n, c, ho, wo = dy.shape
    k = w.shape[-1]
    p = k // 2
    # dy padded so that every (i + p - k_) // s in [-k, out) indexes it: rows shifted by k
    dp = np.zeros((n, c, ho + 2 * k + 2, wo + 2 * k + 2), _F32)
    dp[:, :, k:k + ho, k:k + wo] = dy.astype(_F32)
    iy, ix = np.arange(h), np.arange(wd)
    acc = np.zeros((n, c, h, wd), _F32)
    for ky in range(k - 1, -1, -1):
        ry = iy + p - ky
        my = (ry % s) == 0
        for kx in range(k - 1, -1, -1):
            rx = ix + p - kx
            mx = (rx % s) == 0
            v = dp[:, :, (ry // s + k)[:, None], (rx // s + k)[None, :]]
            new = fma32(v, w[None, :, ky, kx, None, None], acc)
            m = (my[:, None] & mx[None, :])[None, None]
            acc = np.where(m, new, acc).astype(_F32)
    return acc.astype(dt)


def wgrad_partials(x, dy, k, s):
    """fp32 partials [ranges, C, k*k] in the kernel's range order"""
    x, dy = np.asarray(x), np.asarray(dy)
    n, c, h, wd = x.shape
    ho, wo = dy.shape[2:]
    p = k // 2
    ry = -(-ho // (TILE * PASSES))
    rx = -(-wo // TILE)
    hp, wp = ry * TILE * PASSES, rx * TILE
    # dy, and per tap the x value each output pixel multiplies, on the padded range grid (+0 outside the planes)
    d = np.zeros((n, c, hp, wp), _F32)
    d[:, :, :ho, :wo] = dy.astype(_F32)
    xp = np.zeros((n, c, hp * s + k, wp * s + k), _F32)
    xp[:, :, p:p + h, p:p + wd] = x.astype(_F32)
    valid = np.zeros((hp, wp), bool)
    valid[:ho, :wo] = True
    out = np.empty((n * ry * rx, c, k * k), _F32)
    for ky in range(k):
        for kx in range(k):
            xs = xp[:, :, ky:ky + (hp - 1) * s + 1:s, kx:kx + (wp - 1) * s + 1:s]
            xs = np.where(valid, xs, _F32(0))
            dv = np.where(valid, d, _F32(0))
            # [n, c, ry, q, ty, r, rx, tx]
            xs = xs.reshape(n, c, ry, PASSES, WARPS, ROWS, rx, TILE)
            dv = dv.reshape(n, c, ry, PASSES, WARPS, ROWS, rx, TILE)
            acc = np.zeros((n, c, ry, WARPS, rx, TILE), _F32)
            for q in range(PASSES):
                for r in range(ROWS):
                    acc = fma32(xs[:, :, :, q, :, r], dv[:, :, :, q, :, r], acc)
            v = acc
            for half in (16, 8, 4, 2, 1):          # lane 0 of the shfl_xor butterfly
                v = (v[..., :half] + v[..., half:2 * half]).astype(_F32)
            v = v[..., 0]                          # [n, c, ry, ty, rx]
            t = v[:, :, :, 0]
            for wq in range(1, WARPS):
                t = (t + v[:, :, :, wq]).astype(_F32)
            out[:, :, ky * k + kx] = t.transpose(0, 2, 3, 1).reshape(n * ry * rx, c)
    return out


def wgrad(x, dy, k, s):
    """dw [C, k, k] in x's dtype"""
    x = np.asarray(x)
    c = x.shape[1]
    if x.shape[0] == 0:
        return np.zeros((c, k, k), x.dtype)
    part = wgrad_partials(x, dy, k, s).astype(_F64)
    tot = part[0].copy()
    for i in range(1, part.shape[0]):
        tot = tot + part[i]
    return tot.astype(_F32).astype(x.dtype).reshape(c, k, k)


# ---------------------------------------------------------------- fp64 references and the stated bounds
def _conv64(x, w, s, absval=False):
    import torch
    import torch.nn.functional as F
    x = torch.from_numpy(np.asarray(x, _F64))
    w = torch.from_numpy(_w(w).astype(_F64)[:, None])
    if absval:
        x, w = x.abs(), w.abs()
    k = w.shape[-1]
    return F.conv2d(x, w, None, s, k // 2, 1, x.shape[1]).numpy()


def _grads64(x, w, dy, s, absval=False):
    import torch
    import torch.nn.functional as F
    xt = torch.from_numpy(np.asarray(x, _F64)).requires_grad_(True)
    wt = torch.from_numpy(_w(w).astype(_F64)[:, None]).requires_grad_(True)
    g = torch.from_numpy(np.asarray(dy, _F64))
    if absval:
        with torch.no_grad():
            xt.abs_()
            wt.abs_()
        g = g.abs()
    k = wt.shape[-1]
    y = F.conv2d(xt, wt, None, s, k // 2, 1, xt.shape[1])
    dx, dw = torch.autograd.grad(y, (xt, wt), g)
    return dx.numpy(), dw.numpy()[:, 0]


def _half_ulp16(v):
    a = np.abs(np.asarray(v, _F64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 11)


def exact_fwd(x, w, s):
    return _conv64(x, w, s)


def exact_grads(x, w, dy, s):
    """fp64 (dx, dw [C,k,k])"""
    return _grads64(x, w, dy, s)


def bound_fwd(x, w, s, fp16=False):
    k = _w(w).shape[-1]
    ex = _conv64(x, w, s)
    b = k * k * U32 * _conv64(x, w, s, absval=True)
    return b + (_half_ulp16(ex) * 1.01 if fp16 else 0)


def bound_dgrad(x, w, dy, s, fp16=False):
    k = _w(w).shape[-1]
    ex = _grads64(x, w, dy, s)[0]
    b = k * k * U32 * _grads64(x, w, dy, s, absval=True)[0]
    return b + (_half_ulp16(ex) * 1.01 if fp16 else 0)


def bound_wgrad(x, w, dy, s, fp16=False):
    ex = _grads64(x, w, dy, s)[1]
    b = (4 * PASSES + 5 + 7 + 2) * U32 * _grads64(x, w, dy, s, absval=True)[1]
    return b + (_half_ulp16(ex) * 1.01 if fp16 else 0)
