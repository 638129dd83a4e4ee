"""Host-side executor of the LitePose forward on the sm_90a kernels.

``LitePoseEngine`` turns a reference-compatible state_dict (names/shapes of
reference lib/models/pose_mobilenet.py:21-156) into BN-folded, kernel-packed fp16
weights (fold recipe: reference fuse_bn.py:81-137,147-162; shared-BN deconv pair:
scale into both branches, shift once) and runs the network as a fixed sequence of
C-ABI calls (include/litepose_b200.h) on NHWC fp16 activations.  The state_dict of reference
lib/models/pose_simplenet.py (no deconv_raw.* / final_raw.*: the head without the fusion branch)
runs the same plan with the single-branch forms of the deconv and head calls.  A plan (buffers +
call list) is built per (N, H, W, dtype) and can be captured into a CUDA graph.
PyTorch is used for device memory and streams only.
"""
import collections
import ctypes

import numpy as np
import torch

from . import _lib

EPS = 1e-5


def _fold(sd, bn):
    """BN (scale, shift) in fp32, every step correctly rounded: the square root is taken in fp64 and rounded once
    to fp32, which is the correctly rounded fp32 square root.  torch's vectorised fp32 sqrt on the CPU is not always
    (it can be one ulp off), so folding in fp32 directly would give weights that depend on the device the state_dict
    lives on."""
    s = sd[bn + ".weight"].float() / torch.sqrt((sd[bn + ".running_var"].float() + EPS).double()).float()
    b = sd[bn + ".bias"].float() - sd[bn + ".running_mean"].float() * s
    return s, b


def _np16(t):
    """fp32 tensor -> contiguous uint16 view of its fp16 rounding (host)."""
    return np.ascontiguousarray(t.detach().float().cpu().half().numpy()).view(np.uint16)


class _Bump(object):
    """Allocator of _build_plan that carves every buffer of a plan out of one byte arena (256-byte aligned).  Without an
    arena it only measures: the placeholders it returns have a null data pointer and the plan is thrown away."""

    class _Null(object):
        def __init__(self, shape):
            self.shape = tuple(shape)

        def data_ptr(self):
            return 0

    def __init__(self, arena=None):
        self.arena, self.used = arena, 0

    def __call__(self, shape, dtype):
        nbytes = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        off = (self.used + 255) // 256 * 256
        self.used = off + nbytes
        if self.arena is None:
            return self._Null(shape)
        return self.arena[off:off + nbytes].view(dtype).view(shape)


# most arena-backed plans (mixed batches) kept at once; they own no device memory of their own
ARENA_PLANS = 16


class _Op(object):
    __slots__ = ("fn", "args", "name")

    def __init__(self, name, fn, args):
        self.name, self.fn, self.args = name, fn, args


FOLDED_FORMAT = "litepose_b200-folded-1"

# The two LitePose heads of the reference (named after the modules that build them): pose_mobilenet's Fusion Deconv
# Head adds a raw branch from the backbone to every deconv level and output head; pose_simplenet, the paper's ablation
# without it, has the same names minus deconv_raw.* / final_raw.*.
FUSION, SIMPLE = "pose_mobilenet", "pose_simplenet"


def _topology(sd):
    """FUSION or SIMPLE from the state_dict's keys; a dict with the raw branch on some levels only is refused"""
    raw = ["deconv_raw.%d.weight" % i for i in range(3)] + ["final_raw.%d.conv.3.weight" % i for i in range(2)]
    have = [k for k in raw if k in sd]
    if len(have) == len(raw):
        return FUSION
    if not have and not any(k.startswith(("deconv_raw.", "final_raw.")) for k in sd):
        return SIMPLE
    raise ValueError("LitePoseEngine runs the fusion head (the raw branch on all 3 deconv levels and both output heads, "
                     "pose_mobilenet) or no raw branch at all (pose_simplenet); this state_dict has it on some levels "
                     "only: %s present, %s missing" % (have or "no raw weights", [k for k in raw if k not in sd]))


class LitePoseEngine(object):
    def __init__(self, state_dict, arch, device, num_joints_out=None, residual=None, strides=None):
        """``residual`` / ``strides``: per inverted-residual block, stage-major, whether it adds its input and its
        stride.  By default a block's stride is its stage's on block 0 and 1 after, and it adds its input when the
        stride is 1 and its widths are equal (LitePose's rule); the super-network fixes both by its own structure
        (litepose_b200.subnet.derive_supernet_subnet)."""
        self._init_common(arch, device)
        sd = {k: v.detach() for k, v in state_dict.items()}
        self._prep(sd, residual, strides)

    def _init_common(self, arch, device):
        """device 'cpu' is accepted for weight preparation / folded-checkpoint conversion only: run() needs CUDA."""
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type == "cuda":
            with torch.cuda.device(self.device):
                _lib.check(self.lib.lp_device_check(), "lp_device_check")
        self.arch = arch
        self.plans = {}
        self.arena_plans = collections.OrderedDict()    # LRU of plans whose buffers live in self.arenas
        self.arenas = {}                                # pass -> uint8 arena shared by every arena plan of that pass

    # ------------------------------------------------------------------ folded checkpoint ("next" row 4)
    # BN fold (reference fuse_bn.py:81-162) and kernel packing become a load-time no-op: the file holds exactly the
    # arrays the kernels read (fp16 packed weights, fp32 biases) plus the shape metadata of the plan builder.
    def export_folded(self, path):
        import json
        arrays, meta = {}, {}

        def walk(node, prefix):
            if isinstance(node, dict):
                for k, v in node.items():
                    walk(v, prefix + [str(k)])
            elif isinstance(node, list):
                meta["/".join(prefix) + "#len"] = len(node)
                for i, v in enumerate(node):
                    walk(v, prefix + [str(i)])
            elif torch.is_tensor(node):
                arrays["/".join(prefix)] = node.detach().cpu().numpy()
            else:
                meta["/".join(prefix)] = node

        walk(self.P, [])
        header = {"format": FOLDED_FORMAT, "arch": self.arch, "channels": self.channels, "meta": meta,
                  "lib_version": int(self.lib.lp_version()), "topology": self.topology}
        np.savez(path, __header__=np.frombuffer(json.dumps(header).encode(), dtype=np.uint8), **arrays)

    @classmethod
    def from_folded(cls, path, device):
        import json
        z = np.load(path)
        header = json.loads(bytes(z["__header__"]).decode())
        if header.get("format") != FOLDED_FORMAT:
            raise ValueError("not a %s file: %r" % (FOLDED_FORMAT, header.get("format")))
        eng = cls.__new__(cls)
        eng._init_common(header["arch"], device)
        if header["lib_version"] != int(eng.lib.lp_version()):
            raise ValueError("folded checkpoint was packed for library version %d, this is %d (re-export it)"
                             % (header["lib_version"], int(eng.lib.lp_version())))
        eng.channels = list(header["channels"])
        eng.topology = header.get("topology", FUSION)     # files written before the single-branch head: fusion
        if eng.topology not in (FUSION, SIMPLE):
            raise ValueError("folded checkpoint has an unknown head topology %r" % (eng.topology,))
        meta = header["meta"]
        root = {}

        def put(keys, value):
            node = root
            for k in keys[:-1]:
                node = node.setdefault(k, {})
            node[keys[-1]] = value

        for k in z.files:
            if k != "__header__":
                put(k.split("/"), torch.from_numpy(np.ascontiguousarray(z[k])).to(eng.device))
        lists = set()
        for k, v in meta.items():
            if k.endswith("#len"):
                lists.add(k[:-4])
            else:
                put(k.split("/"), v)

        def fix(node, prefix):
            if isinstance(node, dict):
                for k in list(node.keys()):
                    node[k] = fix(node[k], prefix + [k])
                if "/".join(prefix) in lists:
                    return [node[str(i)] for i in range(meta["/".join(prefix) + "#len"])]
            return node

        eng.P = fix(root, [])
        for name in ("deconv", "heads", "blocks"):
            eng.P.setdefault(name, [])
        return eng

    # ------------------------------------------------------------------ weights
    def _dev(self, arr, dtype):
        return torch.from_numpy(np.ascontiguousarray(arr)).view(dtype).to(self.device)

    def _pack_pw(self, w, bias):
        n, k = w.shape[0], w.shape[1]
        w16 = _np16(w.reshape(n, k))
        wp = np.zeros(self.lib.lp_pw1x1_packed_elems(k, n), np.uint16)
        bp = np.zeros(self.lib.lp_pw1x1_packed_bias_elems(n), np.float32)
        b = None if bias is None else np.ascontiguousarray(bias.detach().float().cpu().numpy())
        _lib.check(self.lib.lp_pw1x1_pack(w16.ctypes.data, None if b is None else b.ctypes.data, k, n,
                                          wp.ctypes.data, bp.ctypes.data), "lp_pw1x1_pack")
        return {"w": self._dev(wp, torch.float16), "b": self._dev(bp, torch.float32), "K": k, "N": n}

    def _pack_dw(self, w, bias):
        c, k = w.shape[0], w.shape[-1]
        wt = w.reshape(c, k * k).t().contiguous()   # tap-major [k*k][C]
        return {"w": wt.half().to(self.device), "b": bias.float().contiguous().to(self.device), "C": c, "k": k}

    def _prep(self, sd, residual=None, strides=None):
        arch = self.arch
        total = sum(st["num_blocks"] for st in arch["backbone_setting"])
        for name, per_block in (("residual", residual), ("strides", strides)):
            if per_block is not None and len(per_block) != total:
                raise ValueError("%s lists %d blocks, the architecture has %d" % (name, len(per_block), total))
        P = {}
        n_dec = len([k for k in sd if k.startswith("deconv_refined.") and k.endswith(".weight")])
        if n_dec != 3 or tuple(sd["first.0.0.weight"].shape) != (32, 3, 3, 3):
            raise ValueError("LitePoseEngine implements the shipped LitePose topology (32-channel 3x3 stem, "
                             "MODEL.EXTRA.NUM_DECONV_LAYERS == 3, 4x4 stride-2 deconvs; reference "
                             "lib/models/pose_mobilenet.py:36-135); this state_dict has %d deconv levels and a %s stem"
                             % (n_dec, tuple(sd["first.0.0.weight"].shape)))
        s, b = _fold(sd, "first.0.1")
        w = sd["first.0.0.weight"].float() * s.view(-1, 1, 1, 1)
        w1p = torch.zeros((32, 64), dtype=torch.float16)
        w1p[:, :27] = w.reshape(32, 27).half()
        P["stem"] = {"w": w.reshape(32, 27).half().contiguous().to(self.device),
                     "b": b.contiguous().to(self.device),
                     "w1p": w1p.contiguous().to(self.device)}      # fused stem: [32][64] K-major rows (27 taps, zero padded)
        s, b = _fold(sd, "first.1.1")
        P["stem_dw"] = self._pack_dw(sd["first.1.0.weight"].float() * s.view(-1, 1, 1, 1), b)
        s, b = _fold(sd, "first.3")
        P["stem_pw"] = self._pack_pw(sd["first.2.weight"].float() * s.view(-1, 1, 1, 1), b)
        self.channels = [sd["first.2.weight"].shape[0]]
        blocks = []
        for si, st in enumerate(arch["backbone_setting"]):
            for bi in range(st["num_blocks"]):
                p = "stage.%d.%d." % (si, bi)
                stride = int(strides[len(blocks)]) if strides is not None else st["stride"] if bi == 0 else 1
                s, b = _fold(sd, p + "inv.1")
                inv = self._pack_pw(sd[p + "inv.0.weight"].float() * s.view(-1, 1, 1, 1), b)
                s, b = _fold(sd, p + "depth_conv.1")
                dw = self._pack_dw(sd[p + "depth_conv.0.weight"].float() * s.view(-1, 1, 1, 1), b)
                s, b = _fold(sd, p + "point_conv.1")
                pc = self._pack_pw(sd[p + "point_conv.0.weight"].float() * s.view(-1, 1, 1, 1), b)
                cin, cout = inv["K"], pc["N"]
                res = stride == 1 and cin == cout if residual is None else bool(residual[len(blocks)])
                if res and (stride != 1 or cin != cout):
                    raise ValueError("%s: an identity add needs stride 1 and equal widths, the block has stride %d "
                                     "and %d -> %d channels" % (p[:-1], stride, cin, cout))
                if dw["k"] == 7 and ((stride == 1 and self.lib.lp_block_s1_supported(cin, inv["N"], cout)) or
                                     (stride == 2 and self.lib.lp_block_s2_supported(cin, inv["N"], cout))):
                    # block-fused kernel (lp_block_s1_f16 / lp_block_s2_f16): expansion weights as [Ce][Cin padded to
                    # 64] K-major rows, fp32 bias
                    wfold = sd[p + "inv.0.weight"].float() * _fold(sd, p + "inv.1")[0].view(-1, 1, 1, 1)
                    w16 = _np16(wfold.reshape(inv["N"], cin))
                    wk = np.zeros(self.lib.lp_block_s1_wexp_elems(cin, inv["N"]), np.uint16)
                    _lib.check(self.lib.lp_block_s1_pack_wexp(w16.ctypes.data, cin, inv["N"], wk.ctypes.data),
                               "lp_block_s1_pack_wexp")
                    inv["wblk"] = self._dev(wk, torch.float16)
                    inv["bblk"] = _fold(sd, p + "inv.1")[1].float().contiguous().to(self.device)
                blocks.append({"inv": inv, "dw": dw, "pc": pc, "stride": stride, "stage": si,
                               "res": res, "last": bi == st["num_blocks"] - 1})
            self.channels.append(blocks[-1]["pc"]["N"])
        P["blocks"] = blocks
        P["deconv"] = []
        P["heads"] = []
        self.topology = _topology(sd)
        # single-branch head (pose_simplenet): no raw weights, Cw = C2 = 0 and NULL raw pointers in the C ABI
        fusion = self.topology == FUSION

        def addr(arr):
            return None if arr is None else arr.ctypes.data

        for i in range(3):
            s, b = _fold(sd, "deconv_bnrelu.%d.0" % i)
            wr = sd["deconv_refined.%d.weight" % i].float() * s.view(1, -1, 1, 1)
            ww = sd["deconv_raw.%d.weight" % i].float() * s.view(1, -1, 1, 1) if fusion else None
            cr, cw, co = wr.shape[0], ww.shape[0] if fusion else 0, wr.shape[1]
            wp = np.zeros(self.lib.lp_deconv_packed_elems(cr, cw, co), np.uint16)
            bp = np.zeros(self.lib.lp_deconv_packed_bias_elems(co), np.float32)
            bb = np.ascontiguousarray(b.cpu().numpy())
            a, c = _np16(wr), _np16(ww) if fusion else None
            _lib.check(self.lib.lp_deconv_pack(a.ctypes.data, addr(c), bb.ctypes.data, cr, cw, co,
                                               wp.ctypes.data, bp.ctypes.data), "lp_deconv_pack")
            P["deconv"].append({"w": self._dev(wp, torch.float16), "b": self._dev(bp, torch.float32),
                                "Cr": cr, "Cw": cw, "Co": co})
            if i > 0:
                hd = {}
                for nm in ("final_refined", "final_raw") if fusion else ("final_refined",):
                    p = "%s.%d.conv." % (nm, i - 1)
                    s, b = _fold(sd, p + "1")
                    hd[nm + "_dw"] = self._pack_dw(sd[p + "0.weight"].float() * s.view(-1, 1, 1, 1), b)
                w1 = sd["final_refined.%d.conv.3.weight" % (i - 1)].float()
                w2 = sd["final_raw.%d.conv.3.weight" % (i - 1)].float() if fusion else None
                co, c1, c2 = w1.shape[0], w1.shape[1], w2.shape[1] if fusion else 0
                a, c = _np16(w1.reshape(co, c1)), _np16(w2.reshape(co, c2)) if fusion else None
                hd.update({"C1": c1, "C2": c2, "Co": co})
                # fused head: concatenated depthwise slabs + slab-ordered 1x1 weights
                d1, d2 = hd["final_refined_dw"], hd.get("final_raw_dw")
                dwc = np.zeros(self.lib.lp_head_fused_dw_elems(c1, c2), np.uint16)
                bdc = np.zeros(dwc.size // 25, np.float32)
                pwc = np.zeros(self.lib.lp_head_fused_pw_elems(c1, c2, co), np.uint16)
                x1, x2 = _np16(d1["w"].float()), _np16(d2["w"].float()) if fusion else None
                y1 = np.ascontiguousarray(d1["b"].cpu().numpy())
                y2 = np.ascontiguousarray(d2["b"].cpu().numpy()) if fusion else None
                _lib.check(self.lib.lp_head_fused_pack(x1.ctypes.data, y1.ctypes.data, addr(x2), addr(y2),
                                                       a.ctypes.data, addr(c), c1, c2, co, dwc.ctypes.data,
                                                       bdc.ctypes.data, pwc.ctypes.data), "lp_head_fused_pack")
                hd.update({"dw_cat": self._dev(dwc, torch.float16), "bdw_cat": self._dev(bdc, torch.float32),
                           "pw_cat": self._dev(pwc, torch.float16)})
                P["heads"].append(hd)
        self.P = P

    # ------------------------------------------------------------------ plan
    def _build_plan(self, n, h, w, in_dtype, out_fp32, alloc=None):
        """alloc(shape, dtype) provides every buffer of the plan (default: a tensor of its own)."""
        if h % 16 or w % 16:
            raise ValueError("LitePose input height/width must be multiples of 16, got %dx%d" % (h, w))
        lib, P, dev = self.lib, self.P, self.device
        f16 = torch.float16
        ops = []
        if alloc is None:
            def alloc(shape, dtype):
                return torch.empty(shape, dtype=dtype, device=dev)

        def buf(*shape):
            return alloc(shape, f16)

        plan = {"in_ptr": ctypes.c_void_p(0), "flip": ctypes.c_int(0)}
        h2, w2 = h // 2, w // 2
        x0 = buf(n, h2, w2, P["stem_pw"]["N"])
        st, d, q = P["stem"], P["stem_dw"], P["stem_pw"]
        keep = [x0]
        if "w1p" in st and lib.lp_stem_fused_supported(h, w, q["N"]):
            # conv3x3 s2 -> dw3x3 -> 1x1 in one kernel: the two 32-channel half-resolution tensors never reach HBM
            ops.append(_Op("stem_fused", lib.lp_stem_fused_f16,
                           [plan["in_ptr"], 1 if in_dtype == torch.float32 else 0, plan["flip"], st["w1p"].data_ptr(),
                            st["b"].data_ptr(), d["w"].data_ptr(), d["b"].data_ptr(), q["w"].data_ptr(), q["b"].data_ptr(),
                            x0.data_ptr(), n, h, w, q["N"]]))
        else:
            a0 = buf(n, h2, w2, 32)
            a1 = buf(n, h2, w2, 32)
            keep += [a0, a1]
            ops.append(_Op("stem", lib.lp_stem_conv3x3_s2,
                           [plan["in_ptr"], 1 if in_dtype == torch.float32 else 0, plan["flip"], st["w"].data_ptr(),
                            st["b"].data_ptr(), a0.data_ptr(), n, h, w]))
            ops.append(_Op("stem_dw", lib.lp_dwconv_f16, [a0.data_ptr(), d["w"].data_ptr(), d["b"].data_ptr(),
                                                           a1.data_ptr(), n, 32, h2, w2, 3, 1, _lib.ACT_RELU6]))
            ops.append(_Op("stem_pw", lib.lp_pw1x1_f16, [a1.data_ptr(), q["w"].data_ptr(), q["b"].data_ptr(), None,
                                                          x0.data_ptr(), n * h2 * w2, q["K"], q["N"], _lib.ACT_NONE]))
        x_list = [(x0, h2, w2)]
        cur, ch, cw_ = x0, h2, w2
        # scratch for the expanded tensors, sized for the largest block that does not run as one kernel
        max_e = max_d = 0
        th, tw = h2, w2
        for blk in P["blocks"]:
            th2, tw2 = th // blk["stride"], tw // blk["stride"]
            if "wblk" not in blk["inv"]:
                max_e = max(max_e, n * th * tw * blk["inv"]["N"])
                max_d = max(max_d, n * th2 * tw2 * blk["dw"]["C"])
            th, tw = th2, tw2
        e_buf = alloc((max(max_e, 1),), f16)
        d_buf = alloc((max(max_d, 1),), f16)
        keep += [e_buf, d_buf]
        for blk in P["blocks"]:
            inv, dw, pc = blk["inv"], blk["dw"], blk["pc"]
            oh, ow = ch // blk["stride"], cw_ // blk["stride"]
            out = buf(n, oh, ow, pc["N"])
            keep.append(out)
            if "wblk" in inv:
                # the whole block in one kernel: the 6x-expanded tensor never reaches HBM
                if blk["stride"] == 1:
                    ops.append(_Op("block_s1", lib.lp_block_s1_f16,
                                   [cur.data_ptr(), inv["wblk"].data_ptr(), inv["bblk"].data_ptr(), dw["w"].data_ptr(),
                                    dw["b"].data_ptr(), pc["w"].data_ptr(), pc["b"].data_ptr(), 1 if blk["res"] else 0,
                                    out.data_ptr(), n, ch, cw_, inv["K"], dw["C"], pc["N"]]))
                else:
                    ops.append(_Op("block_s2", lib.lp_block_s2_f16,
                                   [cur.data_ptr(), inv["wblk"].data_ptr(), inv["bblk"].data_ptr(), dw["w"].data_ptr(),
                                    dw["b"].data_ptr(), pc["w"].data_ptr(), pc["b"].data_ptr(), out.data_ptr(), n, ch,
                                    cw_, inv["K"], dw["C"], pc["N"]]))
                cur, ch, cw_ = out, oh, ow
                if blk["last"]:
                    x_list.append((cur, ch, cw_))
                continue
            ops.append(_Op("inv", lib.lp_pw1x1_f16, [cur.data_ptr(), inv["w"].data_ptr(), inv["b"].data_ptr(), None,
                                                      e_buf.data_ptr(), n * ch * cw_, inv["K"], inv["N"],
                                                      _lib.ACT_RELU6]))
            if blk["stride"] == 1 and dw["k"] == 7 and pc["N"] <= 160 and dw["C"] <= 992:
                # depthwise + projection (+ identity) in one kernel: the expanded dw output never reaches HBM
                ops.append(_Op("dw7_project", lib.lp_dw7_project_f16,
                               [e_buf.data_ptr(), dw["w"].data_ptr(), dw["b"].data_ptr(), pc["w"].data_ptr(),
                                pc["b"].data_ptr(), cur.data_ptr() if blk["res"] else None, out.data_ptr(), n, ch,
                                cw_, dw["C"], pc["N"]]))
            else:
                ops.append(_Op("dw7", lib.lp_dwconv_f16, [e_buf.data_ptr(), dw["w"].data_ptr(), dw["b"].data_ptr(),
                                                           d_buf.data_ptr(), n, dw["C"], ch, cw_, dw["k"],
                                                           blk["stride"], _lib.ACT_RELU6]))
                ops.append(_Op("pc", lib.lp_pw1x1_f16, [d_buf.data_ptr(), pc["w"].data_ptr(), pc["b"].data_ptr(),
                                                         cur.data_ptr() if blk["res"] else None, out.data_ptr(),
                                                         n * oh * ow, pc["K"], pc["N"], _lib.ACT_NONE]))
            cur, ch, cw_ = out, oh, ow
            if blk["last"]:
                x_list.append((cur, ch, cw_))
        refined, rh, rw = x_list[-1]
        outs = []

        def raw_ptr(level, channels):
            # the backbone output a raw branch reads (pose_simplenet: none, a NULL pointer with 0 channels)
            return x_list[level][0].data_ptr() if channels else None

        for i in range(3):
            dc = P["deconv"][i]
            nxt = buf(n, rh * 2, rw * 2, dc["Co"])
            keep.append(nxt)
            ops.append(_Op("deconv", lib.lp_fusion_deconv_f16,
                           [refined.data_ptr(), raw_ptr(-i - 2, dc["Cw"]), dc["w"].data_ptr(), dc["b"].data_ptr(),
                            nxt.data_ptr(), n, rh, rw, dc["Cr"], dc["Cw"], dc["Co"]]))
            refined, rh, rw = nxt, rh * 2, rw * 2
            if i > 0:
                hd = P["heads"][i - 1]
                o = alloc((n, hd["Co"], rh, rw), torch.float32 if out_fp32 else f16)
                outs.append(o)
                ops.append(_Op("head_fused", lib.lp_head_fused_f16,
                               [refined.data_ptr(), raw_ptr(-i - 3, hd["C2"]), hd["dw_cat"].data_ptr(),
                                hd["bdw_cat"].data_ptr(), hd["pw_cat"].data_ptr(), o.data_ptr(),
                                1 if out_fp32 else 0, n, rh, rw, hd["C1"], hd["C2"], hd["Co"]]))
        plan.update({"ops": ops, "outs": outs, "keep": keep})
        return plan

    def plan_for(self, n, h, w, in_dtype, out_fp32, flip=False, slot=0):
        # the flip pass owns its own buffers so that both passes can be in flight at once; ``slot`` selects one of
        # several buffer sets (the pipeline alternates two so that step i+1's passes never touch the outputs step i's
        # glue is still reading)
        key = (n, h, w, in_dtype, out_fp32, bool(flip), slot)
        pl = self.plans.get(key)
        if pl is None:
            pl = self._build_plan(n, h, w, in_dtype, out_fp32)
            self.plans[key] = pl
        return pl

    def reserve_arena(self, specs):
        """Size the arenas for the plans ``specs`` = [(n, h, w, in_dtype, out_fp32, flip)] before any of them runs.
        An arena only grows (to the largest plan it has served); growing it drops the arena plans built on the old one.
        Call it when nothing that reads an arena plan's buffers is still queued on another stream."""
        need = {}
        for n, h, w, in_dtype, out_fp32, flip in specs:
            m = _Bump()
            self._build_plan(n, h, w, in_dtype, out_fp32, alloc=m)
            key = bool(flip)
            need[key] = max(need.get(key, 0), m.used)
        for key, nbytes in need.items():
            ar = self.arenas.get(key)
            if ar is None or ar.numel() < nbytes:
                for k in [k for k in self.arena_plans if k[5] == key]:
                    del self.arena_plans[k]
                self.arenas[key] = None
                self.arenas[key] = torch.empty(nbytes, dtype=torch.uint8, device=self.device)

    def arena_plan_for(self, n, h, w, in_dtype, out_fp32, flip=False):
        """A plan whose buffers are carved out of the arena of its pass (plain / mirrored): plans of every size share
        that memory, so device memory does not grow with the number of distinct (n, h, w) served.  Arena plans of one
        pass must run in stream order (the pipeline's mixed batches do); at most ARENA_PLANS are kept."""
        key = (n, h, w, in_dtype, out_fp32, bool(flip))
        pl = self.arena_plans.get(key)
        if pl is not None:
            self.arena_plans.move_to_end(key)
            return pl
        self.reserve_arena([(n, h, w, in_dtype, out_fp32, flip)])
        pl = self._build_plan(n, h, w, in_dtype, out_fp32, alloc=_Bump(self.arenas[key[5]]))
        self.arena_plans[key] = pl
        while len(self.arena_plans) > ARENA_PLANS:
            self.arena_plans.popitem(last=False)
        return pl

    # ------------------------------------------------------------------ run
    def _launch_all(self, plan, stream_ptr):
        for op in plan["ops"]:
            rc = op.fn(*op.args, stream_ptr)
            if rc:
                _lib.check(rc, op.name)

    def run(self, x, flip=False, out_fp32=True, clone=True, slot=0, arena=False):
        """x: NCHW fp16/fp32 CUDA tensor.  Returns [out0 [N,2J,H/4,W/4], out1 [N,J,H/2,W/2]]
        (fp32 when out_fp32 else fp16).  ``flip`` computes the forward of torch.flip(x,[3]).  ``arena``: run on an arena
        plan (arena_plan_for; eager launches only) - its outputs are overwritten by the next arena run of the same pass."""
        if self.device.type != "cuda":
            raise RuntimeError("LitePoseEngine.run needs a CUDA device (this engine was prepared on %s)" % self.device)
        assert x.is_cuda and x.dim() == 4 and x.shape[1] == 3
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        x = x.contiguous()
        n, _, h, w = x.shape
        if arena:
            plan = self.arena_plan_for(n, h, w, x.dtype, out_fp32, flip)
        else:
            plan = self.plan_for(n, h, w, x.dtype, out_fp32, flip, slot)
        with torch.cuda.device(self.device):
            plan["in_ptr"].value = x.data_ptr()
            plan["flip"].value = 1 if flip else 0
            self._launch_all(plan, torch.cuda.current_stream().cuda_stream)
        outs = plan["outs"]
        return [o.clone() for o in outs] if clone else list(outs)
