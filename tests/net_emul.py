"""The LitePose forward of LitePoseEngine restated on the CPU, bit for bit (test infrastructure, numpy only).

forward(state_dict, arch, x, flip, out_fp32) -> [out0 [N,2J,H/4,W/4], out1 [N,J,H/2,W/2]] as LitePoseEngine.run
returns them.  The restatement shares no code with engine.py:
  - BN fold in numpy float32 from the state dict: s = gamma / sqrt(var + eps), weight * s rounded once (RNE) to fp16,
    bias = beta - mean * s in fp32; the deconv pair's scale goes into both branches and its shift is applied once; the
    heads' 1x1 weights are not folded.
  - The stem: the fused stem's chain where lp_stem_fused_supported (conv_ref.stem_im2col of the fp16 image -> the 1x1
    GEMM of mma_emul -> ReLU6 -> dw_emul k3 -> GEMM), else conv_ref.stem_conv -> dw_emul k3 -> GEMM.
  - Every inverted-residual block as pw (ReLU6) -> dwconv (ReLU6, dw_emul.default_prec) -> pw (+ identity), which the
    fused block kernels equal by their own tests.
  - The deconv levels in the slice order of the kernel lp_fusion_deconv_f16 picks for the level's shape.
  - The heads: dw_emul k5 (prec 0, ReLU) on both branches, then the C1-then-C2 GEMM, raw fp32 or fp16."""
import numpy as np

import conv_ref as cr
import dw_emul as de
import mma_emul as me

EPS = 1e-5
_F16, _F32 = np.float16, np.float32


def _np(t):
    return t.detach().cpu().float().numpy()


def fold(sd, bn, eps=EPS):
    """(scale, shift) fp32 of BatchNorm `bn`"""
    s = _np(sd[bn + ".weight"]) / np.sqrt(_np(sd[bn + ".running_var"]) + _F32(eps))
    return s.astype(_F32), (_np(sd[bn + ".bias"]) - _np(sd[bn + ".running_mean"]) * s).astype(_F32)


def _conv_fold(sd, conv, bn):
    """fp16 folded weight [Co, ...] and fp32 bias"""
    s, b = fold(sd, bn)
    w = _np(sd[conv + ".weight"])
    return (w * s.reshape((-1,) + (1,) * (w.ndim - 1))).astype(_F16), b


def _dw(sd, conv, bn):
    """depthwise weights tap-major [k*k, C] fp16, bias fp32, k"""
    w, b = _conv_fold(sd, conv, bn)
    c, k = w.shape[0], w.shape[-1]
    return np.ascontiguousarray(w.reshape(c, k * k).T), b, k


def _pw(x, w, b, act, res=None):
    """NHWC x through the 1x1 GEMM of lp_pw1x1_f16"""
    n, h, wd, c = x.shape
    co = w.shape[0]
    r = None if res is None else res.reshape(-1, co)
    return me.pw1x1(x.reshape(-1, c), w.reshape(co, c), b, r, act).reshape(n, h, wd, co)


def stem_fused_supported(h, w, c0):
    from litepose_b200 import _lib
    return bool(_lib.load().lp_stem_fused_supported(h, w, c0))


def forward(sd, arch, x, flip=False, out_fp32=True, trace=None):
    """x: [N,3,H,W] fp32 or fp16 numpy (or CPU tensor).  trace: a list that receives (name, NHWC fp16) of the stem
    output, every block output and every deconv level, in the order the engine's plan allocates them"""
    trace = [] if trace is None else trace
    x = np.asarray(x.numpy() if hasattr(x, "numpy") else x)
    n, _, h, w = x.shape
    h2, w2 = h // 2, w // 2
    ws, bs = _conv_fold(sd, "first.0.0", "first.0.1")
    wdw, bdw, _ = _dw(sd, "first.1.0", "first.1.1")
    wpw, bpw = _conv_fold(sd, "first.2", "first.3")
    c0 = wpw.shape[0]
    if stem_fused_supported(h, w, c0):
        a = cr.stem_im2col(x.astype(_F16), flip)
        w1p = np.zeros((32, 32), _F16)
        w1p[:, :27] = ws.reshape(32, 27)
        e = me.pw1x1(a, w1p, bs, None, de.ACT_RELU6).reshape(n, h2, w2, 32)
    else:
        e = cr.stem_conv(x, ws.reshape(32, 27), bs, flip)
    d = de.dwconv(e, wdw, bdw, 3, 1, de.ACT_RELU6, de.default_prec(3))
    cur = _pw(d, wpw, bpw, de.ACT_NONE)
    trace.append(("stem", cur))
    feats = [cur]
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            p = "stage.%d.%d." % (si, bi)
            stride = st["stride"] if bi == 0 else 1
            wi, bi_ = _conv_fold(sd, p + "inv.0", p + "inv.1")
            wd, bd, k = _dw(sd, p + "depth_conv.0", p + "depth_conv.1")
            wc, bc = _conv_fold(sd, p + "point_conv.0", p + "point_conv.1")
            t = _pw(cur, wi, bi_, de.ACT_RELU6)
            t = de.dwconv(t, wd, bd, k, stride, de.ACT_RELU6, de.default_prec(k))
            res = cur if (stride == 1 and cur.shape[3] == wc.shape[0]) else None
            cur = _pw(t, wc, bc, de.ACT_NONE, res)
            trace.append(("stage %d block %d" % (si, bi), cur))
        feats.append(cur)
    refined, raw = feats[-1], feats[-2]
    outs = []
    for i in range(3):
        s, b = fold(sd, "deconv_bnrelu.%d.0" % i)
        wr = (_np(sd["deconv_refined.%d.weight" % i]) * s.reshape(1, -1, 1, 1)).astype(_F16)
        ww = (_np(sd["deconv_raw.%d.weight" % i]) * s.reshape(1, -1, 1, 1)).astype(_F16)
        rows = cr.uses_rows_kernel(wr.shape[0], ww.shape[0], wr.shape[1], refined.shape[2])
        refined = me.deconv(refined, raw, wr, ww, b, rows)
        trace.append(("deconv %d (%s kernel)" % (i, "row" if rows else "tiled"), refined))
        raw = feats[-i - 3]
        if i > 0:
            t = []
            for nm, src in (("final_refined", refined), ("final_raw", raw)):
                pre = "%s.%d.conv." % (nm, i - 1)
                wdh, bdh, k = _dw(sd, pre + "0", pre + "1")
                t.append(de.dwconv(src, wdh, bdh, k, 1, de.ACT_RELU, de.default_prec(k)))
            w1 = _np(sd["final_refined.%d.conv.3.weight" % (i - 1)]).astype(_F16)
            w2 = _np(sd["final_raw.%d.conv.3.weight" % (i - 1)]).astype(_F16)
            co = w1.shape[0]
            nn, hh, ww_, c1 = t[0].shape
            o = me.head_dual(t[0].reshape(-1, c1), t[1].reshape(-1, t[1].shape[3]), w1.reshape(co, c1),
                             w2.reshape(co, -1), out_fp32)
            outs.append(o.reshape(nn, hh, ww_, co).transpose(0, 3, 1, 2))
    return outs
