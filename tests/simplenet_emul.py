"""The pose_simplenet forward of LitePoseEngine restated on the CPU, bit for bit (test infrastructure, numpy only).

The single-branch forms of the deconv and head calls (Cw = C2 = 0, no raw tensor), in the slice orders of mma_emul:
  - deconv_single: lp_fusion_deconv_f16 with no raw branch.  Row kernel: every tap group over the k16 slices of
    [refined | 0] (K = Cr rounded up to 16); tiled kernel: the 64-channel K blocks of the refined branch only.
  - head_single: lp_head_pw_dual_f16 with C2 = 0 - the K blocks of the one source, ceil(valid / 16) slices each.
forward(state_dict, arch, x, flip, out_fp32, trace) mirrors net_emul.forward for a state dict without deconv_raw.* /
final_raw.*: the same stem and blocks (through net_emul's fold and GEMM helpers), then each deconv level on the refined
tensor alone and each output head as dw_emul k5 (prec 0, ReLU) followed by head_single."""
import numpy as np

import conv_ref as cr
import dw_emul as de
import mma_emul as me
import net_emul as ne

_F16 = np.float16


def deconv_single(xr, wr, bias, rows, m=me.MODEL):
    """xr [N,H,W,Cr] fp16, wr [Cr,Co,4,4] fp16, bias [Co] fp32 -> [N,2H,2W,Co] fp16"""
    n, h, w, _ = np.shape(xr)
    co = np.shape(wr)[1]
    return me.deconv(xr, np.zeros((n, h, w, 0), _F16), wr, np.zeros((0, co, 4, 4), _F16), bias, rows, m)


def head_single(a1, w1, fp32, m=me.MODEL):
    """a1 [M, C1], w1 [Co, C1] fp16 -> [M, Co] raw fp32 accumulators or one RNE rounding to fp16"""
    return me.head_store(me.gemm(me.k_slices(a1, w1), "zero", m), fp32)


def forward(sd, arch, x, flip=False, out_fp32=True, trace=None):
    """x: [N,3,H,W] fp32 or fp16 numpy.  trace: a list that receives (name, NHWC fp16) of the stem output, every block
    output and every deconv level, in the order the engine's plan allocates them"""
    trace = [] if trace is None else trace
    x = np.asarray(x)
    n, _, h, w = x.shape
    h2, w2 = h // 2, w // 2
    ws, bs = ne._conv_fold(sd, "first.0.0", "first.0.1")
    wdw, bdw, _ = ne._dw(sd, "first.1.0", "first.1.1")
    wpw, bpw = ne._conv_fold(sd, "first.2", "first.3")
    if ne.stem_fused_supported(h, w, wpw.shape[0]):
        a = cr.stem_im2col(x.astype(_F16), flip)
        w1p = np.zeros((32, 32), _F16)
        w1p[:, :27] = ws.reshape(32, 27)
        e = me.pw1x1(a, w1p, bs, None, de.ACT_RELU6).reshape(n, h2, w2, 32)
    else:
        e = cr.stem_conv(x, ws.reshape(32, 27), bs, flip)
    d = de.dwconv(e, wdw, bdw, 3, 1, de.ACT_RELU6, de.default_prec(3))
    cur = ne._pw(d, wpw, bpw, de.ACT_NONE)
    trace.append(("stem", cur))
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            p = "stage.%d.%d." % (si, bi)
            stride = st["stride"] if bi == 0 else 1
            wi, bi_ = ne._conv_fold(sd, p + "inv.0", p + "inv.1")
            wd, bd, k = ne._dw(sd, p + "depth_conv.0", p + "depth_conv.1")
            wc, bc = ne._conv_fold(sd, p + "point_conv.0", p + "point_conv.1")
            t = ne._pw(cur, wi, bi_, de.ACT_RELU6)
            t = de.dwconv(t, wd, bd, k, stride, de.ACT_RELU6, de.default_prec(k))
            res = cur if (stride == 1 and cur.shape[3] == wc.shape[0]) else None
            cur = ne._pw(t, wc, bc, de.ACT_NONE, res)
            trace.append(("stage %d block %d" % (si, bi), cur))
    refined = cur
    outs = []
    for i in range(3):
        s, b = ne.fold(sd, "deconv_bnrelu.%d.0" % i)
        wr = (ne._np(sd["deconv_refined.%d.weight" % i]) * s.reshape(1, -1, 1, 1)).astype(_F16)
        rows = cr.uses_rows_kernel(wr.shape[0], 0, wr.shape[1], refined.shape[2])
        refined = deconv_single(refined, wr, b, rows)
        trace.append(("deconv %d (%s kernel)" % (i, "row" if rows else "tiled"), refined))
        if i > 0:
            pre = "final_refined.%d.conv." % (i - 1)
            wdh, bdh, k = ne._dw(sd, pre + "0", pre + "1")
            t = de.dwconv(refined, wdh, bdh, k, 1, de.ACT_RELU, de.default_prec(k))
            w1 = ne._np(sd[pre + "3.weight"]).astype(_F16)
            co = w1.shape[0]
            nn, hh, ww, c1 = t.shape
            o = head_single(t.reshape(-1, c1), w1.reshape(co, c1), out_fp32)
            outs.append(o.reshape(nn, hh, ww, co).transpose(0, 3, 1, 2))
    return outs
