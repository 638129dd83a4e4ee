"""SuperLitePose.lp_recalibrate_bn (litepose_b200/bn_train.py) restated on the CPU, bit for bit (test infrastructure,
numpy only).

forward(sub, x, running, bn_params) -> (outputs, {BatchNorm name: (new running mean, new running var)}, non-finite
names) for the SupernetSub that litepose_b200.subnet.derive_supernet_subnet gives, the running statistics of the
sub-network's slices and {name: (momentum, eps)}.  The raw producers are the kernels' arithmetic as tests/net_emul.py's
helpers pin it, with zero bias and no activation:
  - stem: conv_ref's fmaf chain over the 27 taps (lp_stem_conv3x3_s2_act), no clamp, one rounding to fp16;
  - depthwise: dw_emul.dwconv at the kernel's default precision; 1x1: mma_emul.pw1x1; deconv: mma_emul's slice order of
    the kernel lp_fusion_deconv_act_f16 picks, fp32(acc + 0) rounded to fp16; heads: mma_emul.head_dual.
stats() restates lp_bn_stats_f16 (the pixel ranges, lanes and merge order bn_train.cu states, fp64, every operation
rounded once) and apply() lp_bn_apply_f16 (fmaf, the kernel's ReLU / ReLU6, + residual in fp32, one rounding)."""
import numpy as np

import conv_ref as cr
import dw_emul as de
import mma_emul as me
import net_emul as ne

_F64, _F32, _F16 = np.float64, np.float32, np.float16
BN_ROWS, BN_THREADS, BN_MAX_VT = 2048, 256, 32


def stats_sums(x):
    """x [M, C] fp16 -> (sum, sum of squares) [C] float64 in lp_bn_stats_f16's order"""
    x = np.asarray(x, _F16)
    m, c = x.shape
    vt = min(c // 8, BN_MAX_VT)
    rl = BN_THREADS // vt
    parts = (m + BN_ROWS - 1) // BN_ROWS
    k = (BN_ROWS + rl - 1) // rl
    xr = np.zeros((parts, k * rl, c), _F64)     # zero padding: adding +0 to a sum that started at +0 changes nothing
    flat = np.zeros((parts * BN_ROWS, c), _F64)
    flat[:m] = x
    xr[:, :BN_ROWS] = flat.reshape(parts, BN_ROWS, c)
    xr = xr.reshape(parts, k, rl, c)
    s1 = np.zeros((parts, rl, c), _F64)
    s2 = np.zeros((parts, rl, c), _F64)
    for i in range(k):                          # lane l: pixels l, l + rl, l + 2 rl, ... of its range
        s1 = s1 + xr[:, i]
        s2 = s2 + xr[:, i] * xr[:, i]
    t1, t2 = s1[:, 0].copy(), s2[:, 0].copy()
    for lane in range(1, rl):                   # lanes in order
        t1 = t1 + s1[:, lane]
        t2 = t2 + s2[:, lane]
    a1, a2 = t1[0].copy(), t2[0].copy()
    for p in range(1, parts):                   # pixel ranges in order
        a1 = a1 + t1[p]
        a2 = a2 + t2[p]
    return a1, a2


def stats(x, gamma, beta, rmean, rvar, momentum, eps):
    """lp_bn_stats_f16: x [M, C] fp16 -> scale, shift, new mean, new var ([C] fp32), nonfinite"""
    m = x.shape[0]
    s1, s2 = stats_sums(x)
    mf = _F64(m)
    mean = s1 / mf
    var = s2 / mf - mean * mean
    var = np.where(var > 0, var, _F64(0))
    var_u = var * mf / (mf - _F64(1))
    s = np.asarray(gamma, _F32).astype(_F64) / np.sqrt(var + _F64(eps))
    with np.errstate(over="ignore", invalid="ignore"):
        scale = s.astype(_F32)
        shift = (np.asarray(beta, _F32).astype(_F64) - mean * s).astype(_F32)
        keep = _F64(1.0) - _F64(momentum)
        nm = (keep * np.asarray(rmean, _F32).astype(_F64) + _F64(momentum) * mean).astype(_F32)
        nv = (keep * np.asarray(rvar, _F32).astype(_F64) + _F64(momentum) * var_u).astype(_F32)
    bad = not (np.isfinite(scale).all() and np.isfinite(shift).all() and np.isfinite(nm).all() and
               np.isfinite(nv).all())
    return scale, shift, nm, nv, bad


def apply(x, scale, shift, act, res=None):
    """lp_bn_apply_f16: x [..., C] fp16 -> fp16"""
    x = np.asarray(x, _F16)
    v = cr.fma32(np.broadcast_to(np.asarray(scale, _F32), x.shape), x, np.broadcast_to(np.asarray(shift, _F32), x.shape))
    if act != de.ACT_NONE:
        v = np.where(v > 0, v, _F32(0)).astype(_F32)
    if act == de.ACT_RELU6:
        v = np.where(v < 6, v, _F32(6)).astype(_F32)
    if res is not None:
        v = (v + np.asarray(res, _F16).astype(_F32)).astype(_F32)
    return v.astype(_F16)


def stem_raw(x, w, flip=False):
    """lp_stem_conv3x3_s2_act, act none, bias NULL: x [N,3,H,W] fp32 / fp16, w [32, 27] fp16 -> [N,Ho,Wo,32] fp16"""
    fp32 = np.asarray(x).dtype == _F32
    taps = cr._taps(x, flip)
    w = np.asarray(w, _F16)
    n, ho, wo = taps[0].shape
    acc = np.zeros((n, ho, wo, 32), _F32)
    for t, xs in enumerate(taps):
        xs = xs[..., None]
        if fp32:
            acc = cr.fma32(xs, w[:, t], acc)
        else:
            acc = xs.astype(_F32) * w[:, t].astype(_F32) + acc
    return acc.astype(_F16)


def deconv_raw(xr, xw, wr, ww, bias=None):
    """lp_fusion_deconv_act_f16, act none: fp32(acc + bias (default zero)) -> [N,2H,2W,Co] fp16"""
    n, h, w, _ = np.shape(xr)
    co = np.shape(wr)[1]
    bias = np.zeros(co, _F32) if bias is None else np.asarray(bias, _F32)
    rows = cr.uses_rows_kernel(np.shape(wr)[0], np.shape(ww)[0], co, w)
    out = np.empty((n, 2 * h, 2 * w, co), _F16)
    for a in (0, 1):
        for b in (0, 1):
            acc = me.gemm(me.deconv_slices(xr, xw, wr, ww, a, b, rows), "zero")
            out[:, a::2, b::2] = (np.asarray(acc, _F32) + bias).astype(_F32).astype(_F16).reshape(n, h, w, co)
    return out


def _w16(sd, name):
    return ne._np(sd[name]).astype(_F16)


def _dw_raw(x, sd, name, stride):
    w = _w16(sd, name)
    c, k = w.shape[0], w.shape[-1]
    return de.dwconv(x, np.ascontiguousarray(w.reshape(c, k * k).T), np.zeros(c, _F32), k, stride, de.ACT_NONE,
                     de.default_prec(k))


def _pw_raw(x, sd, name):
    w = _w16(sd, name)
    co = w.shape[0]
    return ne._pw(x, w.reshape(co, -1), np.zeros(co, _F32), de.ACT_NONE)


def forward(sub, x, running, bn_params):
    """sub: SupernetSub; x [N,3,H,W] numpy fp32 / fp16; running {name: (mean [c], var [c])} -> (outs [out0, out1]
    (fp32 for fp32 x, else fp16), {name: (new mean, new var)}, [names with non-finite statistics])"""
    sd, arch = sub.state_dict, sub.arch
    x = np.asarray(x)
    out_fp32 = x.dtype == _F32
    new, bad = {}, []

    def bn(t, name, act, res=None):
        c = t.shape[-1]
        mom, eps = bn_params[name]
        rm, rv = running[name]
        sc, sh, nm, nv, nf = stats(t.reshape(-1, c), ne._np(sd[name + ".weight"]), ne._np(sd[name + ".bias"]),
                                   rm, rv, mom, eps)
        new[name] = (nm, nv)
        if nf:
            bad.append(name)
        return apply(t, sc, sh, act, res)

    cur = bn(stem_raw(x, _w16(sd, "first.0.0.weight").reshape(32, 27)), "first.0.1", de.ACT_RELU6)
    cur = bn(_dw_raw(cur, sd, "first.1.0.weight", 1), "first.1.1", de.ACT_RELU6)
    cur = bn(_pw_raw(cur, sd, "first.2.weight"), "first.3", de.ACT_NONE)
    feats = [cur]
    nb = 0
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            p = "stage.%d.%d." % (si, bi)
            t = bn(_pw_raw(cur, sd, p + "inv.0.weight"), p + "inv.1", de.ACT_RELU6)
            t = bn(_dw_raw(t, sd, p + "depth_conv.0.weight", sub.strides[nb]), p + "depth_conv.1", de.ACT_RELU6)
            cur = bn(_pw_raw(t, sd, p + "point_conv.0.weight"), p + "point_conv.1", de.ACT_NONE,
                     cur if sub.residual[nb] else None)
            nb += 1
        feats.append(cur)
    refined = feats[-1]
    outs = []
    for i in range(len(arch["deconv_setting"])):
        raw = feats[-i - 2]
        refined = bn(deconv_raw(refined, raw, _w16(sd, "deconv_refined.%d.weight" % i),
                                _w16(sd, "deconv_raw.%d.weight" % i)), "deconv_bnrelu.%d.0" % i, de.ACT_RELU)
        if i > 0:
            t = []
            for nm, src in (("final_refined", refined), ("final_raw", feats[-i - 3])):
                pre = "%s.%d.conv." % (nm, i - 1)
                t.append(bn(_dw_raw(src, sd, pre + "0.weight", 1), pre + "1", de.ACT_RELU))
            w1 = _w16(sd, "final_refined.%d.conv.3.weight" % (i - 1))
            w2 = _w16(sd, "final_raw.%d.conv.3.weight" % (i - 1))
            co = w1.shape[0]
            n, hh, ww, c1 = t[0].shape
            o = me.head_dual(t[0].reshape(-1, c1), t[1].reshape(-1, t[1].shape[3]), w1.reshape(co, c1),
                             w2.reshape(co, -1), out_fp32)
            outs.append(o.reshape(n, hh, ww, co).transpose(0, 3, 1, 2))
    return outs, new, bad
