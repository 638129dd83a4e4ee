"""The engine's forward of a super-network sub-network restated on the CPU, bit for bit (test infrastructure, numpy only).

forward(state_dict, arch, x, flip, out_fp32, residual, strides) -> [out0, out1] as
LitePoseEngine(state_dict, arch, device, residual=residual, strides=strides).run(x, flip, out_fp32) returns them, for
the LitePose-named state dict, arch and per-block lists that litepose_b200.subnet.derive_supernet_subnet gives.  It is
tests/net_emul.py's forward with the block stride and identity add read from the two lists instead of LitePose's rule
(stage stride on block 0, identity at stride 1 between equal widths): the super-network fixes both by its own
structure.  Every step uses net_emul's helpers (BN fold, stem, 1x1 GEMM, depthwise, deconv, heads), so the arithmetic
is the one net_emul pins; tests/test_supernet_emul.py checks that with LitePose's lists it equals net_emul.forward."""
import numpy as np

import conv_ref as cr
import dw_emul as de
import mma_emul as me
import net_emul as ne

_F16 = np.float16


def forward(sd, arch, x, flip=False, out_fp32=True, residual=None, strides=None):
    """x: [N,3,H,W] fp32 or fp16 numpy (or CPU tensor); residual / strides: one entry per block, stage-major"""
    x = np.asarray(x.numpy() if hasattr(x, "numpy") else x)
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
    feats = [cur]
    nb = 0
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            p = "stage.%d.%d." % (si, bi)
            wi, bi_ = ne._conv_fold(sd, p + "inv.0", p + "inv.1")
            wd, bd, k = ne._dw(sd, p + "depth_conv.0", p + "depth_conv.1")
            wc, bc = ne._conv_fold(sd, p + "point_conv.0", p + "point_conv.1")
            t = ne._pw(cur, wi, bi_, de.ACT_RELU6)
            t = de.dwconv(t, wd, bd, k, strides[nb], de.ACT_RELU6, de.default_prec(k))
            cur = ne._pw(t, wc, bc, de.ACT_NONE, cur if residual[nb] else None)
            nb += 1
        feats.append(cur)
    refined, raw = feats[-1], feats[-2]
    outs = []
    for i in range(3):
        s, b = ne.fold(sd, "deconv_bnrelu.%d.0" % i)
        wr = (ne._np(sd["deconv_refined.%d.weight" % i]) * s.reshape(1, -1, 1, 1)).astype(_F16)
        ww = (ne._np(sd["deconv_raw.%d.weight" % i]) * s.reshape(1, -1, 1, 1)).astype(_F16)
        rows = cr.uses_rows_kernel(wr.shape[0], ww.shape[0], wr.shape[1], refined.shape[2])
        refined = me.deconv(refined, raw, wr, ww, b, rows)
        raw = feats[-i - 3]
        if i > 0:
            t = []
            for nm, src in (("final_refined", refined), ("final_raw", raw)):
                pre = "%s.%d.conv." % (nm, i - 1)
                wdh, bdh, k = ne._dw(sd, pre + "0", pre + "1")
                t.append(de.dwconv(src, wdh, bdh, k, 1, de.ACT_RELU, de.default_prec(k)))
            w1 = ne._np(sd["final_refined.%d.conv.3.weight" % (i - 1)]).astype(_F16)
            w2 = ne._np(sd["final_raw.%d.conv.3.weight" % (i - 1)]).astype(_F16)
            co = w1.shape[0]
            nn_, hh, ww_, c1 = t[0].shape
            o = me.head_dual(t[0].reshape(-1, c1), t[1].reshape(-1, t[1].shape[3]), w1.reshape(co, c1),
                             w2.reshape(co, -1), out_fp32)
            outs.append(o.reshape(nn_, hh, ww_, co).transpose(0, 3, 1, 2))
    return outs
