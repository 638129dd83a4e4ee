"""Training-mode forward of a super-network sub-network on the sm_90a kernels: the BatchNorm recalibration pass of the
architecture search (reference calibrate_test.py:58-61, ``model.train(); model(images)``).

``BNTrainPlan`` is built from ``litepose_b200.subnet.derive_supernet_subnet``'s unfolded sub-network (its slices, the
k = 5 / 3 depthwise transform and the supernet's strides and identity adds).  Every BatchNorm becomes three launches:
the raw convolution without BN fold or bias (rounded once to fp16), ``lp_bn_stats_f16`` (batch statistics, the
normalisation's scale / shift and the updated running statistics, staged on the device) and ``lp_bn_apply_f16``
(normalise + activation (+ identity), in place).  The fused stem, block and head kernels fold BN into their weights and
never expose the pre-BN values, so the plan runs the unfused ones:

    first.0 conv3x3 s2     lp_stem_conv3x3_s2_act, no activation       -> ReLU6
    first.1 dw3x3          lp_dwconv_f16, no activation               -> ReLU6
    first.2 1x1            lp_pw1x1_f16, no activation                -> none
    block inv / depth_conv lp_pw1x1_f16 / lp_dwconv_f16 (k 7/5/3)      -> ReLU6
    block point_conv       lp_pw1x1_f16                               -> none, + identity where the supernet adds it
    deconv level           lp_fusion_deconv_act_f16, both branches    -> ReLU
    head branch            lp_dwconv_f16 dw5x5                        -> ReLU, then lp_head_pw_dual_f16 (NCHW out)

``run`` returns the outputs and the staged statistics; it writes nothing into a module (the caller checks the non-finite
flags once and copies the staged values in).  The activations of a plan are carved out of one arena (engine._Bump); the
staging buffers are tensors of their own."""
import ctypes

import numpy as np
import torch

from . import _lib
from .engine import LitePoseEngine, _Bump, _np16, _Op


def bn_names(arch):
    """The BatchNorm modules a sub-network ``arch`` (supernet names) runs, in the plan's order"""
    names = ["first.0.1", "first.1.1", "first.3"]
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            p = "stage.%d.%d." % (si, bi)
            names += [p + "inv.1", p + "depth_conv.1", p + "point_conv.1"]
    for i in range(len(arch["deconv_setting"])):
        names.append("deconv_bnrelu.%d.0" % i)
        if i > 0:
            names += ["final_refined.%d.conv.1" % (i - 1), "final_raw.%d.conv.1" % (i - 1)]
    return names


class BNTrainPlan(LitePoseEngine):
    """The train-mode forward of one sub-network at one input shape (n, h, w, dtype) on one device.

    ``sub``: a SupernetSub; ``bn_params``: {BatchNorm name: (momentum, eps)} for every name of ``bn_names(sub.arch)``.
    The packed weights and the BatchNorm affine parameters are taken once, from ``sub``; the running statistics are
    read at every ``run`` from the tensors passed there."""

    def __init__(self, sub, bn_params, device, n, h, w, in_dtype):
        self._init_common(sub.arch, device)
        if h % 16 or w % 16:
            raise ValueError("LitePose input height/width must be multiples of 16, got %dx%d" % (h, w))
        if not 1 <= n <= 65535:
            raise ValueError("batch of %d images: the stem takes 1 to 65535" % n)
        if in_dtype not in (torch.float16, torch.float32):
            raise ValueError("input dtype %s: fp32, or fp16 under network_to_half" % in_dtype)
        self.n, self.h, self.w, self.in_dtype = n, h, w, in_dtype
        sd = sub.state_dict
        self.names = bn_names(sub.arch)
        self.channels = [int(sd[b + ".weight"].shape[0]) for b in self.names]
        bad = [(b, c) for b, c in zip(self.names, self.channels) if c % 8]
        if bad:
            raise ValueError("the kernels take channel counts that are multiples of 8: %s" % bad)
        # per BatchNorm i, 8-aligned float offsets: gamma / beta in `affine`, running mean / var in `running_in`,
        # scale / shift / new mean / new var in `staged`
        self.offs = np.concatenate([[0], np.cumsum(self.channels)]).astype(np.int64)
        total = int(self.offs[-1])
        affine = torch.cat([torch.cat([sd[b + ".weight"].float(), sd[b + ".bias"].float()]) for b in self.names])
        self.affine = affine.to(self.device)
        self.momentum_eps = [bn_params[b] for b in self.names]
        self.running_in = torch.empty(2 * total, dtype=torch.float32, device=self.device)
        self.staged = torch.empty(4 * total, dtype=torch.float32, device=self.device)
        self.flags = torch.zeros(len(self.names), dtype=torch.int32, device=self.device)
        self._pack(sd, sub)
        m = _Bump()
        self._plan(m)
        self.arena = torch.empty(m.used, dtype=torch.uint8, device=self.device)
        self._plan(_Bump(self.arena))

    # ------------------------------------------------------------------ weights (no BN fold, no bias)
    def _pack(self, sd, sub):
        P = {"stem": sd["first.0.0.weight"].float().reshape(32, 27).half().contiguous().to(self.device)}

        def dw(name):
            wt = sd[name].float()
            return self._pack_dw(wt, torch.zeros(wt.shape[0]))

        P["stem_dw"] = dw("first.1.0.weight")
        P["stem_pw"] = self._pack_pw(sd["first.2.weight"].float(), None)
        blocks = []
        for si, st in enumerate(sub.arch["backbone_setting"]):
            for bi in range(st["num_blocks"]):
                p = "stage.%d.%d." % (si, bi)
                nb = len(blocks)
                blocks.append({"inv": self._pack_pw(sd[p + "inv.0.weight"].float(), None),
                               "dw": dw(p + "depth_conv.0.weight"),
                               "pc": self._pack_pw(sd[p + "point_conv.0.weight"].float(), None),
                               "stride": int(sub.strides[nb]), "res": bool(sub.residual[nb]),
                               "last": bi == st["num_blocks"] - 1})
        P["blocks"] = blocks
        P["deconv"], P["heads"] = [], []
        for i in range(len(sub.arch["deconv_setting"])):
            wr, ww = sd["deconv_refined.%d.weight" % i].float(), sd["deconv_raw.%d.weight" % i].float()
            cr, cw, co = wr.shape[0], ww.shape[0], wr.shape[1]
            if co > 64:
                raise ValueError("deconv level %d: %d output channels, the deconv kernels take at most 64" % (i, co))
            wp = np.zeros(self.lib.lp_deconv_packed_elems(cr, cw, co), np.uint16)
            bp = np.zeros(self.lib.lp_deconv_packed_bias_elems(co), np.float32)
            a, c = _np16(wr), _np16(ww)
            _lib.check(self.lib.lp_deconv_pack(a.ctypes.data, c.ctypes.data, None, cr, cw, co, wp.ctypes.data,
                                               bp.ctypes.data), "lp_deconv_pack")
            P["deconv"].append({"w": self._dev(wp, torch.float16), "b": self._dev(bp, torch.float32),
                                "Cr": cr, "Cw": cw, "Co": co})
            if i > 0:
                hd = {nm: dw("%s.%d.conv.0.weight" % (nm, i - 1)) for nm in ("final_refined", "final_raw")}
                w1 = sd["final_refined.%d.conv.3.weight" % (i - 1)].float()
                w2 = sd["final_raw.%d.conv.3.weight" % (i - 1)].float()
                co, c1, c2 = w1.shape[0], w1.shape[1], w2.shape[1]
                a, c = _np16(w1.reshape(co, c1)), _np16(w2.reshape(co, c2))
                hp = np.zeros(self.lib.lp_head_packed_elems(c1, c2, co), np.uint16)
                _lib.check(self.lib.lp_head_pack(a.ctypes.data, c.ctypes.data, c1, c2, co, hp.ctypes.data),
                           "lp_head_pack")
                hd.update({"pw": self._dev(hp, torch.float16), "C1": c1, "C2": c2, "Co": co})
                P["heads"].append(hd)
        self.P = P

    # ------------------------------------------------------------------ plan
    def _plan(self, alloc):
        lib, P, n, h, w = self.lib, self.P, self.n, self.h, self.w
        f16 = torch.float16
        ops, outs = [], []
        self.in_ptr = ctypes.c_void_p(0)
        total = int(self.offs[-1])
        ws_bytes = 0
        ws_ops = []

        def buf(*shape):
            return alloc(shape, f16)

        def fptr(t, off):
            return t.data_ptr() + 4 * int(off)

        def bn(x, m, act, res=None):
            """batch statistics of x [m, C], then normalise + act (+ res) in place"""
            nonlocal ws_bytes
            i = len([op for op in ops if op.name.startswith("bn_stats")])
            c, o = self.channels[i], int(self.offs[i])
            if m < 2:
                raise ValueError("%s: %d value per channel; train-mode BatchNorm needs more than 1 (N*H*W > 1)"
                                 % (self.names[i], m))
            mom, eps = self.momentum_eps[i]
            ws_bytes = max(ws_bytes, lib.lp_bn_stats_workspace_bytes(m, c))
            scale, shift = fptr(self.staged, o), fptr(self.staged, total + o)
            args = [x.data_ptr(), m, c, self.affine.data_ptr() + 8 * o, self.affine.data_ptr() + 8 * o + 4 * c,
                    fptr(self.running_in, o), fptr(self.running_in, total + o), float(mom), float(eps), scale, shift,
                    fptr(self.staged, 2 * total + o), fptr(self.staged, 3 * total + o), fptr(self.flags, i), None, 0]
            ws_ops.append(args)
            ops.append(_Op("bn_stats " + self.names[i], lib.lp_bn_stats_f16, args))
            ops.append(_Op("bn_apply " + self.names[i], lib.lp_bn_apply_f16,
                           [x.data_ptr(), scale, shift, None if res is None else res.data_ptr(), x.data_ptr(), m, c,
                            act]))

        h2, w2 = h // 2, w // 2
        m0 = n * h2 * w2
        y0, y1 = buf(n, h2, w2, 32), buf(n, h2, w2, 32)
        ops.append(_Op("stem_raw", lib.lp_stem_conv3x3_s2_act,
                       [self.in_ptr, 1 if self.in_dtype == torch.float32 else 0, 0, P["stem"].data_ptr(), None,
                        y0.data_ptr(), n, h, w, _lib.ACT_NONE]))
        bn(y0, m0, _lib.ACT_RELU6)
        d = P["stem_dw"]
        ops.append(_Op("stem_dw_raw", lib.lp_dwconv_f16, [y0.data_ptr(), d["w"].data_ptr(), d["b"].data_ptr(),
                                                           y1.data_ptr(), n, 32, h2, w2, 3, 1, _lib.ACT_NONE]))
        bn(y1, m0, _lib.ACT_RELU6)
        q = P["stem_pw"]
        cur = buf(n, h2, w2, q["N"])
        ops.append(_Op("stem_pw_raw", lib.lp_pw1x1_f16, [y1.data_ptr(), q["w"].data_ptr(), q["b"].data_ptr(), None,
                                                          cur.data_ptr(), m0, q["K"], q["N"], _lib.ACT_NONE]))
        bn(cur, m0, _lib.ACT_NONE)
        ch, cw_ = h2, w2
        feats = [(cur, ch, cw_)]
        max_e = max_d = 0
        th, tw = h2, w2
        for blk in P["blocks"]:
            max_e = max(max_e, n * th * tw * blk["inv"]["N"])
            th, tw = th // blk["stride"], tw // blk["stride"]
            max_d = max(max_d, n * th * tw * blk["dw"]["C"])
        e_buf, d_buf = alloc((max_e,), f16), alloc((max_d,), f16)
        for blk in P["blocks"]:
            inv, dw, pc = blk["inv"], blk["dw"], blk["pc"]
            oh, ow = ch // blk["stride"], cw_ // blk["stride"]
            ops.append(_Op("inv_raw", lib.lp_pw1x1_f16, [cur.data_ptr(), inv["w"].data_ptr(), inv["b"].data_ptr(),
                                                          None, e_buf.data_ptr(), n * ch * cw_, inv["K"], inv["N"],
                                                          _lib.ACT_NONE]))
            bn(e_buf, n * ch * cw_, _lib.ACT_RELU6)
            ops.append(_Op("dw_raw", lib.lp_dwconv_f16, [e_buf.data_ptr(), dw["w"].data_ptr(), dw["b"].data_ptr(),
                                                          d_buf.data_ptr(), n, dw["C"], ch, cw_, dw["k"],
                                                          blk["stride"], _lib.ACT_NONE]))
            bn(d_buf, n * oh * ow, _lib.ACT_RELU6)
            out = buf(n, oh, ow, pc["N"])
            ops.append(_Op("pc_raw", lib.lp_pw1x1_f16, [d_buf.data_ptr(), pc["w"].data_ptr(), pc["b"].data_ptr(),
                                                         None, out.data_ptr(), n * oh * ow, pc["K"], pc["N"],
                                                         _lib.ACT_NONE]))
            bn(out, n * oh * ow, _lib.ACT_NONE, cur if blk["res"] else None)
            cur, ch, cw_ = out, oh, ow
            if blk["last"]:
                feats.append((cur, ch, cw_))
        refined, rh, rw = feats[-1]
        out_fp32 = self.in_dtype == torch.float32
        for i, dc in enumerate(P["deconv"]):
            raw = feats[-i - 2][0]
            nxt = buf(n, rh * 2, rw * 2, dc["Co"])
            ops.append(_Op("deconv_raw", lib.lp_fusion_deconv_act_f16,
                           [refined.data_ptr(), raw.data_ptr(), dc["w"].data_ptr(), dc["b"].data_ptr(), nxt.data_ptr(),
                            n, rh, rw, dc["Cr"], dc["Cw"], dc["Co"], _lib.ACT_NONE]))
            refined, rh, rw = nxt, rh * 2, rw * 2
            bn(refined, n * rh * rw, _lib.ACT_RELU)
            if i > 0:
                hd = P["heads"][i - 1]
                t = []
                for nm, src in (("final_refined", refined), ("final_raw", feats[-i - 3][0])):
                    d = hd[nm]
                    tb = buf(n, rh, rw, d["C"])
                    ops.append(_Op("head_dw_raw", lib.lp_dwconv_f16,
                                   [src.data_ptr(), d["w"].data_ptr(), d["b"].data_ptr(), tb.data_ptr(), n, d["C"], rh,
                                    rw, d["k"], 1, _lib.ACT_NONE]))
                    bn(tb, n * rh * rw, _lib.ACT_RELU)
                    t.append(tb)
                o = alloc((n, hd["Co"], rh, rw), torch.float32 if out_fp32 else f16)
                outs.append(o)
                ops.append(_Op("head_pw", lib.lp_head_pw_dual_f16,
                               [t[0].data_ptr(), t[1].data_ptr(), hd["pw"].data_ptr(), o.data_ptr(),
                                1 if out_fp32 else 0, n, rh, rw, hd["C1"], hd["C2"], hd["Co"]]))
        ws = alloc((max(ws_bytes, 16),), torch.uint8)
        for args in ws_ops:
            args[-2:] = [ws.data_ptr(), ws_bytes]
        self.ops, self.outs = ops, outs

    # ------------------------------------------------------------------ run
    def run(self, x, running):
        """x: NCHW CUDA tensor of the plan's shape and dtype; running: [(running_mean[:c], running_var[:c])] per
        BatchNorm in ``names`` order.  Returns (outputs (clones), staged): staged [4, sum C] fp32 rows scale, shift,
        new running mean, new running var (a view of the plan's buffer, valid until the next run), and the per-layer
        non-finite flags stay in ``flags``."""
        x = x.contiguous()
        assert tuple(x.shape) == (self.n, 3, self.h, self.w) and x.dtype == self.in_dtype and x.device == self.device
        total = int(self.offs[-1])
        with torch.cuda.device(self.device):
            torch.cat([t.float() for t, _ in running] + [t.float() for _, t in running],
                      out=self.running_in.view(2 * total))
            self.flags.zero_()
            self.in_ptr.value = x.data_ptr()
            self._launch_all({"ops": self.ops}, torch.cuda.current_stream().cuda_stream)
        return [o.clone() for o in self.outs], self.staged.view(4, total)
