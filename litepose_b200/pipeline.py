"""End-to-end batched inference: frames -> keypoints, mirroring the reference's
per-image loop (reference valid.py:195-233) for a whole batch on one GPU:

    image.cuda()                          -> pinned H2D copy (side stream, double buffered)
    get_multi_stage_outputs(flip=True)    -> two engine passes (the flip pass mirrors inside the stem)
    aggregate_results                     -> one fused glue kernel (lp_glue_f32)
    parser.parse(final_heatmaps, tags)    -> device parser (NMS/top-K, match, adjust, refine)
    get_final_preds                       -> left to the caller (CPU, tiny; "next" row 3)

Deviations from valid.py, all forced by the synthetic setting (SURVEY.md §8b last row):
frames are synthetic tensors instead of dataloader images; weights are random-init; the
optional ``plant`` hook adds planted person patches between glue and parser (a random-weight
network detects nobody); no dataset.evaluate.  One process drives one GPU; ranks shard the
batch and a single NCCL gather of the packed keypoints follows (litepose_b200/dist.py).
"""
import torch

from . import _lib
from .config import flip_index_for
from .parser import DeviceParser, check_max_people


class PlantedCrowd(object):
    """Sparse planted persons for the synthetic benchmark: Gaussian det patches are
    max-composited into the heat-maps and 9x9 tag patches overwrite the tag maps (all T).
    Index/value lists are built once on the host (litepose_b200.synth conventions) and applied by ONE kernel of the
    library on the device (lp_plant_crowd_f32); host tensors (the CPU baseline arm, the oracle side of the tests) take
    the equivalent torch index ops."""

    def __init__(self, n, num_joints, h, w, t, num_people=5, seed=0, device="cuda", presence=0.9, sigma=2.0):
        import numpy as np
        rng = np.random.RandomState(seed)
        r = int(3 * sigma)
        yy, xx = np.mgrid[-r:r + 1, -r:r + 1]
        gauss = np.exp(-(xx ** 2 + yy ** 2) / (2.0 * sigma * sigma)).astype(np.float32)
        didx, dval, tidx, tval = [], [], [], []
        m = min(20, h // 4, w // 4)
        for i in range(n):
            for p in range(num_people):
                cy, cx = rng.randint(m, h - m), rng.randint(m, w - m)
                for j in range(num_joints):
                    present = rng.rand() < presence
                    dy, dx = rng.randint(-15, 16), rng.randint(-15, 16)
                    amp = np.float32(rng.uniform(0.5, 1.0))
                    if not present:
                        continue
                    y = int(np.clip(cy + dy, r, h - r - 1))
                    x = int(np.clip(cx + dx, r, w - r - 1))
                    base = (i * num_joints + j) * h * w
                    ys, xs = np.mgrid[y - r:y + r + 1, x - r:x + r + 1]
                    didx.append((base + ys * w + xs).ravel())
                    dval.append((amp * gauss).ravel())
                    ys, xs = np.mgrid[y - 4:y + 5, x - 4:x + 5]
                    flat = (base + ys * w + xs).ravel()
                    tv = (2.0 * p + rng.randn(81, t) * 0.05).astype(np.float32)
                    tidx.append((flat[:, None] * t + np.arange(t)[None, :]).ravel())
                    tval.append(tv.ravel())
        if didx:
            di, dv = np.concatenate(didx).astype(np.int64), np.concatenate(dval).astype(np.float32)
            ti, tv = np.concatenate(tidx).astype(np.int64), np.concatenate(tval).astype(np.float32)
            # overlapping tag patches: the LAST writer wins (what a sequential index_copy_ does); de-duplicated here so
            # that the device kernel's plain stores are race free and every device sees the same maps
            _, first_rev = np.unique(ti[::-1], return_index=True)
            last = np.sort(ti.size - 1 - first_rev)
            ti, tv = ti[last], tv[last]
        else:
            di = ti = np.zeros(0, np.int64)
            dv = tv = np.zeros(0, np.float32)
        self.didx, self.dval = torch.from_numpy(di).to(device), torch.from_numpy(dv).to(device)
        self.tidx, self.tval = torch.from_numpy(ti).to(device), torch.from_numpy(tv).to(device)

    def apply(self, det, tag):
        if not self.didx.numel():
            return det, tag
        if det.is_cuda:
            if not (det.is_contiguous() and tag.is_contiguous() and det.dtype == torch.float32 and tag.dtype == torch.float32):
                raise ValueError("PlantedCrowd.apply: contiguous float32 det / tag expected")
            # one launch of the library's kernel (overlapping det patches: atomic max, order independent)
            _lib.check(_lib.load().lp_plant_crowd_f32(det.data_ptr(), self.didx.data_ptr(), self.dval.data_ptr(),
                                                      self.didx.numel(), tag.data_ptr(), self.tidx.data_ptr(),
                                                      self.tval.data_ptr(), self.tidx.numel(),
                                                      torch.cuda.current_stream().cuda_stream), "lp_plant_crowd_f32")
            return det, tag
        # host tensors: the same workload for the CPU baseline arm and the oracle side of the tests
        det.view(-1).scatter_reduce_(0, self.didx, self.dval, reduce="amax", include_self=True)
        tag.view(-1).index_copy_(0, self.tidx, self.tval)
        return det, tag


def unpack_fast_payload(host, M, J):
    """Rows of lp_pack_fast_payload_f32 ([N, M*J*4 + 2] float32 host tensor or array: M persons x J joints x (x, y,
    val, tag) | person count | KM status) -> list over images of (ans ndarray [P,J,4], P).  Raises LitePoseError on an
    image whose KM assignment hit its round cap (status 1): such a result is never returned."""
    import numpy as np
    a = host.numpy() if torch.is_tensor(host) else np.asarray(host, np.float32)
    kp = M * J * 4
    if a.ndim != 2 or a.shape[1] != kp + 2:
        raise ValueError("fast payload: rows of %d floats expected, got shape %r" % (kp + 2, a.shape))
    out = []
    for i in range(a.shape[0]):
        if int(a[i, kp + 1]) != 0:
            raise _lib.LitePoseError("image %d: the KM assignment hit its round cap (status %d); no result"
                                     % (i, int(a[i, kp + 1])))
        p = int(a[i, kp])
        out.append((a[i, :kp].reshape(M, J, 4)[:p].copy(), p))
    return out


class ImagesTicket(object):
    """Ticket of LitePosePipeline.submit_images: which list slot holds the list, and the submission it belongs to.  Only
    collect_images takes it (the tickets of submit() are slot numbers)."""
    __slots__ = ("owner", "slot", "serial")

    def __init__(self, owner, slot, serial):
        self.owner, self.slot, self.serial = owner, slot, serial

    def __repr__(self):
        return "ImagesTicket(slot=%d, serial=%d)" % (self.slot, self.serial)


class LitePosePipeline(object):
    def __init__(self, model, cfg, use_graphs=True, keep=64, grouping="ae"):
        """model: litepose_b200 drop-in LitePose on a CUDA device (eval).

        grouping: "ae" - the evaluation parser (lib/core/group.py: NMS/top-K, tag matching, adjust, refine, scores);
        "fast" - the demo's parser (nano_demo/fast_utils/group.py:38-47: peak finder + KM assignment, no adjust /
        refine, at most 32 persons).  Every entry point then returns, per image, (ans [P,J,4] float32 = x, y, val, tag
        in person-creation order, P) instead of (ans [P,J,3+T], scores, P)."""
        if grouping not in ("ae", "fast"):
            raise ValueError("grouping=%r: 'ae' or 'fast' expected" % (grouping,))
        self.cfg = cfg
        self._validate_cfg(cfg)
        self.grouping = grouping
        if grouping == "fast":
            self._validate_fast_cfg(cfg)
        self.lib = _lib.load()
        self.device = next(model.parameters()).device
        self.engine = model.lp_engine(self.device)
        from .lib.core.group import Params
        p = Params(cfg)
        self.params = p
        self.parser = DeviceParser(p.num_joints, p.max_num_people, p.detection_threshold, p.tag_threshold,
                                   p.use_detection_val, p.ignore_too_much, p.joint_order, cfg.TEST.NMS_KERNEL,
                                   cfg.TEST.NMS_PADDING)
        self.flip = bool(cfg.TEST.FLIP_TEST)
        self.scales = sorted((float(v) for v in cfg.TEST.SCALE_FACTOR), reverse=True)    # valid.py:205: largest first
        self.project = bool(cfg.TEST.PROJECT2IMAGE)
        self.adjust, self.refine = bool(cfg.TEST.ADJUST), bool(cfg.TEST.REFINE)
        self.fidx = torch.tensor(flip_index_for(cfg), dtype=torch.int32, device=self.device)
        # model channel layout (pose_mobilenet.py:86-100, lib/config/default.py:175-177): DATASET.NUM_JOINTS counts the
        # centre joint when WITH_CENTER is on (the parser drops it with IGNORE_CENTER: Params.num_joints);
        # TAG_PER_JOINT off = ONE tag map after the heat-maps
        self.model_joints = int(cfg.DATASET.NUM_JOINTS)
        self.tag_shared = not bool(cfg.MODEL.TAG_PER_JOINT)
        self.canonical = self.model_joints == p.num_joints and not self.tag_shared
        self.use_graphs = use_graphs
        # persons per image in the fixed-size packed payload (the D2H copy / NCCL gather of every step).  The reference
        # returns every person it finds (lib/core/group.py:96,269-291); an image with more than ``keep`` persons is
        # never clipped: step() fetches the full result from the parser's buffers (capacity J*K persons) in a second
        # copy, and unpack() raises if it is handed an overflowing payload without that second copy.
        self.keep = min(int(keep), self.parser.pcap)
        J = p.num_joints
        if grouping == "fast":
            from .fast_utils.group import Params as FastParams
            fp = FastParams(cfg)
            # the demo's parser hands joint_order to assign(), which reads the first C entries: the entries that name no
            # plane are dropped, as fast_utils.group.HeatmapParser._joint_order does
            self.fast = {"M": int(fp.max_num_people), "thr": float(fp.detection_threshold), "win": int(fp.window_size),
                         "tag_thr": float(fp.tag_threshold),
                         "jo": torch.tensor([j for j in fp.joint_order if j < J][:J], dtype=torch.int32,
                                            device=self.device)}
        # packed payload per image: ae = ``keep`` persons x J x (x, y, val, T tags) | their scores | person count;
        # fast = every person (M <= 32) x J x (x, y, val, tag) | person count | KM status
        self.T = 2 if self.flip else 1
        self.row = J * (3 + self.T)
        self.width = self.fast["M"] * J * 4 + 2 if grouping == "fast" else self.keep * self.row + self.keep + 1
        self._state = {}
        self._async = None                # submit()/collect() slots
        self._final = None                # per-image inverse affines of get_final_preds (host, [N,6] float64)

    @staticmethod
    def _validate_cfg(cfg):
        """The fused glue kernels cover the cfg keys that lib/core/inference.py:75-208 branches on for the LitePose head
        layout (two stages: heat + tags at 1/4, heat at 1/2): flip test, PROJECT2IMAGE, multi-scale, WITH_CENTER /
        IGNORE_CENTER, TAG_PER_JOINT.  Other stage selections (WITH_HEATMAPS / WITH_AE other than the shipped
        (True, True) / (True, False)) are rejected here instead of being silently ignored."""
        def bad(what):
            raise NotImplementedError("LitePosePipeline: %s is not supported by the fused glue kernel "
                                      "(use the reference's core.inference on the drop-in module instead)" % what)
        if cfg.DATASET.WITH_CENTER and cfg.TEST.IGNORE_CENTER and not cfg.MODEL.TAG_PER_JOINT:
            # the reference slices the last channel off the tags as well (inference.py:147-150): with ONE shared tag map
            # nothing is left and its parser fails on the empty tensor - no behaviour to reproduce
            bad("WITH_CENTER + IGNORE_CENTER with TAG_PER_JOINT=False (the reference drops the only tag map there)")
        scales = [float(v) for v in cfg.TEST.SCALE_FACTOR]
        if len(scales) != len(set(scales)) or 1.0 not in scales or min(scales) <= 0:
            # the reference takes the tags from the scale-1 pass only (inference.py:179-190): without it torch.cat of an
            # empty list fails at valid.py:224
            raise ValueError("TEST.SCALE_FACTOR=%r: distinct positive scales including 1 expected" % (scales,))
        if tuple(cfg.LOSS.WITH_HEATMAPS_LOSS) != (True, True) or tuple(cfg.TEST.WITH_HEATMAPS) != (True, True):
            bad("WITH_HEATMAPS_LOSS / TEST.WITH_HEATMAPS other than (True, True)")
        if tuple(cfg.LOSS.WITH_AE_LOSS) != (True, False) or tuple(cfg.TEST.WITH_AE) != (True, False):
            bad("WITH_AE_LOSS / TEST.WITH_AE other than (True, False)")
        if int(cfg.LOSS.NUM_STAGES) != 2:
            bad("LOSS.NUM_STAGES=%r" % (cfg.LOSS.NUM_STAGES,))
        check_max_people(cfg.DATASET.MAX_NUM_PEOPLE)

    @staticmethod
    def _validate_fast_cfg(cfg):
        """grouping="fast" runs the demo's parser as it is (nano_demo/fast_utils/group.py:38-47): peaks + KM assignment,
        nothing else.  Settings it cannot honour are refused, not ignored: adjust / refine (the demo's cfg turns both
        off, nano_demo/core/__init__.py:106-116) and more than 32 persons (the KM kernel holds 32 per joint)."""
        why = []
        if int(cfg.DATASET.MAX_NUM_PEOPLE) > 32:
            why.append("DATASET.MAX_NUM_PEOPLE=%d exceeds the 32 persons the KM assignment holds"
                       % int(cfg.DATASET.MAX_NUM_PEOPLE))
        if cfg.TEST.ADJUST:
            why.append("TEST.ADJUST is on (the fast parser has no adjust step)")
        if cfg.TEST.REFINE:
            why.append("TEST.REFINE is on (the fast parser has no refine step)")
        if why:
            raise ValueError("LitePosePipeline(grouping='fast'): " + "; ".join(why))

    def set_final_preds(self, centers=None, scales=None):
        """valid.py:230-233 on the device: after this call every step maps the keypoints of image i back to its original
        image with get_affine_transform(centers[i], scales[i], 0, [Wd, Hd], inv=1) (reference lib/utils/transforms.py
        :50-57,195-202) before they are packed for the host.  The 2x3 matrices are computed here, once, on the host
        (they depend on the image sizes only); call again when the batch composition changes, or with None to get
        heat-map coordinates back."""
        if centers is None:
            self._final = None
            return
        import numpy as np
        from .lib.utils.transforms import get_affine_transform
        self._final = (np.asarray(centers, np.float64), np.asarray(scales, np.float64))
        self._final_ver = getattr(self, "_final_ver", 0) + 1
        self._final_trans = {}
        self._get_trans = lambda hm: self._final_trans.setdefault(tuple(hm), np.stack([
            get_affine_transform(np.asarray(c), np.asarray(s), 0, list(hm), inv=1)
            for c, s in zip(*self._final)]).reshape(-1, 6))

    # -- device step (everything between the H2D copy and the D2H copy) -------------
    def _network_part(self, side, x, slot=0, arena=False):
        """Both network passes -> ([o0, o1], [f0, f1]) in the engine's buffer set ``slot`` (``arena``: in the engine's
        shared arena plans, see LitePoseEngine.arena_plan_for); the mirrored pass runs on the stream ``side``."""
        eng = self.engine
        if not self.flip:
            return eng.run(x, flip=False, out_fp32=True, clone=False, slot=slot, arena=arena), None
        # the plain and the mirrored pass are independent until the glue: fork onto a side stream so that one pass'
        # kernels fill the launch gaps and tails of the other (each pass has its own plan buffers)
        main = torch.cuda.current_stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            f = eng.run(x, flip=True, out_fp32=True, clone=False, slot=slot, arena=arena)
        o = eng.run(x, flip=False, out_fp32=True, clone=False, slot=slot, arena=arena)
        main.wait_stream(side)
        return o, f

    def _glue(self, o, f, det, tag, plant, i=0):
        """Glue launch of scale ``i`` of self.scales (largest first) on that scale's model outputs, into det / tag:
        lp_glue_f32 for the canonical single-scale layout, else lp_glue_scale_f32 (see step_device_multiscale).  After
        the last scale, the benchmark's planted persons: ``plant`` is one PlantedCrowd, a list with one (or None) per
        image, or None."""
        n, J, Hd, Wd = det.shape[0], self.params.num_joints, det.shape[2], det.shape[3]
        h, w = o[0].shape[2], o[0].shape[3]
        fl = 1 if self.flip else 0
        f0, f1 = (f[0].data_ptr(), f[1].data_ptr()) if self.flip else (None, None)
        last = i == len(self.scales) - 1
        stream = torch.cuda.current_stream().cuda_stream
        if self.canonical and len(self.scales) == 1:
            _lib.check(self.lib.lp_glue_f32(o[0].data_ptr(), o[1].data_ptr(), f0, f1, self.fidx.data_ptr(), n, J, h, w,
                                            fl, Hd, Wd, det.data_ptr(), tag.data_ptr(), stream), "lp_glue_f32")
        else:
            _lib.check(self.lib.lp_glue_scale_f32(
                o[0].data_ptr(), o[1].data_ptr(), f0, f1, self.fidx.data_ptr(), n, J, self.model_joints,
                1 if self.tag_shared else 0, h, w, fl, Hd, Wd, 1 if i > 0 else 0,
                float(len(self.scales)) if last else 1.0, det.data_ptr(),
                tag.data_ptr() if self.scales[i] == 1.0 else None, stream), "lp_glue_scale_f32")
        if not last:
            return
        if isinstance(plant, list):
            for k, p in enumerate(plant):
                if p is not None:
                    p.apply(det[k:k + 1], tag[k:k + 1])
        elif plant is not None:
            plant.apply(det, tag)

    def _forward(self, xs, det, tag, side, plant, arena=False):
        """``xs``: {scale: frames [N,3,Hs,Ws] on the device}, or the frames alone for a single-scale cfg.  Per scale,
        largest first: both network passes and the glue launch into det / tag (+ the planted persons, see _glue)."""
        if not isinstance(xs, dict):
            xs = {1.0: xs}
        for i, s in enumerate(self.scales):
            o, f = self._network_part(side, xs[s], arena=arena)
            self._glue(o, f, det, tag, plant, i)

    def _parse(self, det, tag, packed, trans, fb=None, ragged=None, outs=None):
        """The grouping mode's device parser, get_final_preds (``trans``: device pointer to [N,6] float64 matrices, or
        None) and payload pack on det / tag -> ``packed``.  Uniform maps: det [N,J,H,W], tag [N,1|J,H,W,T]; ragged
        arena: ``ragged`` = (hw [N,2] host int32, device pointer to the lp_map_desc_t of the maps), ``outs`` the dict
        that owns the ragged parser's results (DeviceParser.run_ragged).  ``fb``: the fast grouping's buffers
        (_fast_buffers).  Returns the ae parser's own buffers (ans, num, scores; capacity J*K persons, valid until its
        next run) for fetch_overflow; None with grouping="fast"."""
        J, T = self.params.num_joints, self.T
        hw, desc = ragged if ragged is not None else (None, None)
        n = det.shape[0] if ragged is None else len(hw)
        s = torch.cuda.current_stream().cuda_stream
        full = None
        if self.grouping == "fast":
            # the demo's parser where the glue left the maps: zero ans, find peaks (tag channel 0 read in place), KM
            # assignment
            f, M = self.fast, self.fast["M"]
            ans, num = fb["ans"], fb["num"]
            # lp_assign_f32 writes only the entries it assigns: without this the rows of the previous step would remain
            ans.zero_()
            H, W = (det.shape[2], det.shape[3]) if ragged is None else (0, 0)
            _lib.check(self.lib.lp_find_peaks_maps_f32(
                det.data_ptr(), tag.data_ptr(), n, H, W, None if hw is None else hw.ctypes.data, desc, J, T,
                1 if self.tag_shared else J, M, f["thr"], f["win"], fb["count"].data_ptr(), fb["val"].data_ptr(),
                fb["tag"].data_ptr(), fb["ind"].data_ptr(), s), "lp_find_peaks_maps_f32")
            _lib.check(self.lib.lp_assign_f32(fb["count"].data_ptr(), fb["val"].data_ptr(), fb["tag"].data_ptr(),
                                              fb["ind"].data_ptr(), f["jo"].data_ptr(), n, J, M, f["tag_thr"],
                                              num.data_ptr(), ans.data_ptr(), fb["status"].data_ptr(), s), "lp_assign_f32")
        elif ragged is not None:
            ans, num, scores = full = self.parser.run_ragged(det, tag, hw, desc, T, self.adjust, self.refine, outs)
        else:
            if self.tag_shared:
                # MODEL.TAG_PER_JOINT off: the one tag map serves every joint (group.py:150-152); the parser kernels
                # index [N,J,H,W,T], so the map is tiled here (one strided copy; not the shipped configuration)
                tag = tag.expand(-1, J, -1, -1, -1).contiguous()
            ans, num, scores = full = self.parser.run(det, tag, self.adjust, self.refine)
        if trans is not None:
            _lib.check(self.lib.lp_transform_preds_f32(ans.data_ptr(), num.data_ptr(), trans, n, ans.shape[1],
                                                       ans.shape[2], ans.shape[3], s), "lp_transform_preds_f32")
        if self.grouping == "fast":
            _lib.check(self.lib.lp_pack_fast_payload_f32(ans.data_ptr(), num.data_ptr(), fb["status"].data_ptr(), n, M,
                                                         J, packed.data_ptr(), s), "lp_pack_fast_payload_f32")
        else:
            _lib.check(self.lib.lp_pack_payload_f32(ans.data_ptr(), num.data_ptr(), scores.data_ptr(), n, ans.shape[1],
                                                    self.row, self.keep, packed.data_ptr(), s), "lp_pack_payload_f32")
        return full

    def _parser_part(self, st, det, tag, packed):
        """_parse on maps of the uniform-size state ``st`` -> ``packed``; the ae parser's buffers stay in st["full"]."""
        st["full"] = self._parse(det, tag, packed, None if st["trans"] is None else st["trans"].data_ptr(), st["fast"])

    def _fast_buffers(self, n, J, alloc=None):
        """Peaks, persons and status of the fast grouping for n images; ``alloc(name, shape, dtype)`` (default: new
        device tensors) lets the mixed path serve them from its grow-only buffers."""
        if alloc is None:
            alloc = lambda name, shape, dt: torch.empty(shape, dtype=dt, device=self.device)
        f32, i32, M = torch.float32, torch.int32, self.fast["M"]
        spec = {"count": ((n, J), i32), "val": ((n, J, M), f32), "tag": ((n, J, M), f32), "ind": ((n, J, M, 2), i32),
                "ans": ((n, M, J, 4), f32), "num": ((n,), i32), "status": ((n,), i32)}
        return {k: alloc(k, shape, dt) for k, (shape, dt) in spec.items()}

    def unpack_fast(self, host):
        """Fast-grouping payload (host) -> list over images of (ans ndarray [P,J,4], P); see unpack_fast_payload."""
        return unpack_fast_payload(host, self.fast["M"], self.params.num_joints)

    def _decode(self, host, st=None):
        """Host payload -> per-image results of the pipeline's grouping mode.  fast: raises on a KM status 1; ae: the
        images past ``keep`` are read from the parser's buffers of the step ``st`` that produced ``host``
        (fetch_overflow), and raise without it."""
        if self.grouping == "fast":
            return self.unpack_fast(host)
        return self.unpack(host, self.row, self.T, None if st is None else self.fetch_overflow(st, host))

    def _fetch(self, st):
        """Blocking result of a step: D2H copy of st["packed"] into the pinned st["host"], synchronise, _decode."""
        st["host"].copy_(st["packed"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self._decode(st["host"], st)

    def _forward_part(self, st, xs, det, tag):
        """_forward on the side stream and plant hook of the uniform-size state ``st``."""
        self._forward(xs, det, tag, st["side"], st["plant"])

    def _device_step(self, st, xs):
        """Network passes, glue and parser of one step on ``xs`` (see _forward) into the buffers of ``st``."""
        self._forward_part(st, xs, st["det"], st["tag"])
        self._parser_part(st, st["det"], st["tag"], st["packed"])

    @staticmethod
    def _capture(*parts):
        """One CUDA graph per callable of ``parts``, captured in order after an eager run of them all (which builds the
        engine's plans and sets the kernels' function attributes) and a synchronise."""
        for part in parts:
            part()
        torch.cuda.synchronize()
        graphs = []
        for part in parts:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                part()
            graphs.append(g)
        return graphs

    def step_device_overlapped(self, x_dev, plant=None):
        """Throughput form of step_device: the network passes of this step run on the current stream while the glue and
        the parser of the PREVIOUS step are still running on a second stream (the glue is bound by HBM writes, the parser
        is a chain of short, latency-bound kernels - both leave the FMA pipes to the network; the engine's buffers and
        det / tag / packed are double buffered).  Returns (packed, event): ``packed`` is valid once ``event`` has completed, and stays valid until the
        second next call.  CUDA graphs only."""
        if not self.use_graphs:
            raise RuntimeError("step_device_overlapped needs use_graphs=True")
        n, _, s_h, s_w = x_dev.shape
        st = self._get_state(n, s_h, s_w, x_dev.dtype, plant)
        ov = st.get("ov")
        if ov is None:
            ov = st["ov"] = {"det": [st["det"], torch.empty_like(st["det"])], "tag": [st["tag"], torch.empty_like(st["tag"])],
                             "packed": [st["packed"], torch.zeros_like(st["packed"])], "gF": [None, None], "gP": [None, None],
                             "pstream": torch.cuda.Stream(device=self.device), "P_done": [None, None],
                             "consumer_done": [None, None], "idx": 0}
        b = ov["idx"]
        ov["idx"] = b ^ 1
        main = torch.cuda.current_stream()
        ps = ov["pstream"]
        if ov["P_done"][b] is not None:
            main.wait_event(ov["P_done"][b])      # the parser that last read det/tag[b] has finished
        st["x"].copy_(x_dev, non_blocking=True)
        if ov["gF"][b] is None:
            # the eager warm-up below writes the parser's buffers, which the other slot's parser graph (still running
            # on the parser stream) shares
            for ev in ov["P_done"]:
                if ev is not None:
                    main.wait_event(ev)
            det, tag, packed = ov["det"][b], ov["tag"][b], ov["packed"][b]
            of = []

            def network():
                of[:] = self._network_part(st["side"], st["x"], slot=b)

            def glue_parse():
                # the glue writes 1.4 GB at the HBM write roofline: on the second stream it overlaps the FMA-bound network
                # passes of the next step (which write the other buffer set of the engine)
                self._glue(of[0], of[1], det, tag, st["plant"])
                self._parser_part(st, det, tag, packed)

            ov["gF"][b], ov["gP"][b] = self._capture(network, glue_parse)
        ov["gF"][b].replay()
        f_done = torch.cuda.Event()
        f_done.record(main)
        with torch.cuda.stream(ps):
            ps.wait_event(f_done)
            if ov["consumer_done"][b] is not None:
                ps.wait_event(ov["consumer_done"][b])     # the previous payload of this slot has been copied out
            ov["gP"][b].replay()
            ev = torch.cuda.Event()
            ev.record(ps)
        ov["P_done"][b] = ev
        st["ov_last"] = b
        return ov["packed"][b], ev

    def _get_state(self, n, s_h, s_w, dtype, plant, det_hw=None):
        if len(self.scales) > 1 and det_hw is None:
            raise RuntimeError("TEST.SCALE_FACTOR=%r: the multi-scale test runs through step_multiscale() / "
                               "step_device_multiscale()" % (self.scales,))
        key = (n, s_h, s_w, dtype, self._final is not None, det_hw)
        st = self._state.get(key)
        if st is None:
            J = self.params.num_joints
            Hd, Wd = det_hw if det_hw is not None else ((s_h, s_w) if self.project else (s_h // 2, s_w // 2))
            dev = self.device
            st = {
                "x": torch.empty((n, 3, s_h, s_w), dtype=dtype, device=dev),
                "side": torch.cuda.Stream(device=dev),
                "det": torch.empty((n, J, Hd, Wd), dtype=torch.float32, device=dev),
                "tag": torch.empty((n, 1 if self.tag_shared else J, Hd, Wd, self.T), dtype=torch.float32, device=dev),
                "packed": torch.zeros((n, self.width), dtype=torch.float32, device=dev),
                "host": torch.empty((n, self.width), dtype=torch.float32).pin_memory(),
                "row": self.row, "T": self.T, "graph": None, "plant": plant, "trans": None, "full": None, "ov": None,
                "fast": self._fast_buffers(n, J) if self.grouping == "fast" else None,
            }
            if self._final is not None:
                st["trans"] = torch.zeros((n, 6), dtype=torch.float64, device=dev)
            self._state[key] = st
        if st["plant"] is not plant:
            # a captured graph bakes the plant hook's index tensors in: a different hook (or none) needs a new capture
            st["graph"] = None
            st["plant"] = plant
            if st.get("ov") is not None:
                st["ov"]["gF"] = [None, None]
        if st["trans"] is not None and st.get("trans_ver") != self._final_ver:
            if len(self._final[0]) != n:
                raise ValueError("set_final_preds: %d centers for a batch of %d" % (len(self._final[0]), n))
            tr = self._get_trans((st["det"].shape[3], st["det"].shape[2]))
            st["trans"].copy_(torch.from_numpy(tr))          # read by the (captured) kernel at replay time
            st["trans_ver"] = self._final_ver
        return st

    def step_device(self, x_dev, plant=None):
        """Frames already resident on the device (NCHW fp16/fp32).  Returns the packed device result
        [N, keep*J*(3+T) + keep + 1] (keypoints, scores, person count); with grouping="fast" [N, M*J*4 + 2] (every
        person's keypoints, person count, KM status: unpack_fast_payload)."""
        n, _, s_h, s_w = x_dev.shape
        # the state of the last step_device / step_device_multiscale call: its det / tag / packed stay readable there
        # until the next call
        st = self._last_state = self._get_state(n, s_h, s_w, x_dev.dtype, plant)
        main = torch.cuda.current_stream()
        for other in self._state.values():
            ov = other.get("ov")
            if ov is None:
                continue
            # an overlapped step still queued on a parser stream reads buffers this step overwrites: the engine's
            # buffer set 0 and the parser's buffers (shared by every state of the same shapes), and this state's det /
            # tag (its buffer set 0)
            for ev in ov["P_done"]:
                if ev is not None:
                    main.wait_event(ev)
            if other is st and ov["consumer_done"][0] is not None:
                # st["packed"] is buffer set 0's payload: submit() may not have copied it out on its result stream yet
                main.wait_event(ov["consumer_done"][0])
        if not self.use_graphs:
            self._device_step(st, x_dev)
            return st["packed"]
        st["x"].copy_(x_dev, non_blocking=True)
        if st["graph"] is None:
            st["graph"], = self._capture(lambda: self._device_step(st, st["x"]))
        st["graph"].replay()
        return st["packed"]

    def step(self, frames_pinned, plant=None):
        """Public end-to-end call: pinned host frames in, host result out (blocking)."""
        self.step_device(frames_pinned.to(self.device, non_blocking=True), plant)
        return self._fetch(self._last_state)

    # -- multi-scale test (TEST.SCALE_FACTOR with several entries; reference valid.py:198-229) ----------------------------
    def step_device_multiscale(self, xs, plant=None):
        """``xs``: {scale: frames [N,3,Hs,Ws] on the device} - for every scale of TEST.SCALE_FACTOR the batch resized
        as resize_align_multi_scale does (litepose_b200.lib.utils.transforms.resize_align_normalize_device produces
        it on the device).  Per scale, largest first: both network passes, then ONE glue launch (lp_glue_scale_f32)
        that resamples the scale's flip-averaged heat-maps to the common size and accumulates them
        (aggregate_results, lib/core/inference.py:176-208); the tags come from the scale-1 pass; the sum is divided by
        the number of scales by the last launch (valid.py:223).  Common size = base_size (the scale-1 frames) with
        PROJECT2IMAGE, else the first scale's heat-map size.  Then the device parser, as in step_device.
        Launches run eagerly (no CUDA graph: one plan per scale).  Returns the packed device result."""
        scales = self.scales
        missing = [s for s in scales if s not in xs]
        if missing:
            raise ValueError("step_device_multiscale: no frames for scale(s) %r" % (missing,))
        x1, big = xs[1.0], xs[scales[0]]
        n = x1.shape[0]
        for s in scales:
            x = xs[s]
            if x.shape[0] != n or x.shape[2] % 64 or x.shape[3] % 64:
                raise ValueError("step_device_multiscale: scale %r frames %r (batch %d, sides multiples of 64 expected)"
                                 % (s, tuple(x.shape), n))
        det_hw = (x1.shape[2], x1.shape[3]) if self.project else (big.shape[2] // 2, big.shape[3] // 2)
        st = self._last_state = self._get_state(n, x1.shape[2], x1.shape[3], x1.dtype, plant, det_hw=det_hw)
        self._device_step(st, xs)
        return st["packed"]

    def step_multiscale(self, frames, plant=None):
        """Public blocking call of the multi-scale test: {scale: pinned host frames} in, host result out (the list
        over images of (ans [P,J,3+T], scores, P), as step())."""
        self.step_device_multiscale({float(s): f.to(self.device, non_blocking=True) for s, f in frames.items()}, plant)
        return self._fetch(self._last_state)

    def infer_images(self, images, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), half=True, plant=None):
        """The body of the reference's evaluation loop (valid.py:198-233) for a batch of equally sized uint8 images
        [N,H,W,3] (host, ideally pinned, or device): get_multi_scale_size -> per scale of TEST.SCALE_FACTOR
        resize_align_multi_scale + ToTensor + Normalize on the device (lp_warp_affine_normalize_u8) -> the network
        passes, glue and parser of step() / step_multiscale() -> get_final_preds on the device.  Returns the list over
        images of (final_results [P,J,3+T] in the coordinates of the original image, scores, P) - per image what
        valid.py:227-233 holds in ``final_results`` and ``scores``.

        ``images`` may also be a LIST of uint8 [H_i,W_i,3] images (numpy arrays or tensors) of any sizes - a real
        evaluation set, where every image has its own network size (infer_mixed); ``plant`` is then a list with one
        batch-1 PlantedCrowd or None per image."""
        if isinstance(images, (list, tuple)):
            return self.infer_mixed(images, mean, std, half, plant)
        import numpy as np
        from .lib.utils import transforms as T
        if images.dim() != 4 or images.shape[3] != 3 or images.dtype != torch.uint8:
            raise TypeError("infer_images: uint8 [N,H,W,3] expected")
        n, h, w, _ = images.shape
        size = int(self.cfg.DATASET.INPUT_SIZE)
        smin = min(self.scales)
        d = images.to(self.device, non_blocking=True)
        xs, center, scale = {}, None, None
        for s in self.scales:                     # the centre / scale valid.py hands to get_final_preds are the last scale's
            xs[s], center, scale = T.resize_align_normalize_device(d, size, s, smin, list(mean), list(std), half=half)
        prev = self._final                     # a caller's own set_final_preds() setting is put back afterwards
        self.set_final_preds([center] * n, [scale] * n)
        try:
            if len(self.scales) == 1:
                self.step_device(xs[1.0], plant)
            else:
                self.step_device_multiscale(xs, plant)
            return self._fetch(self._last_state)
        finally:
            if prev is None:
                self.set_final_preds(None)
            else:
                self.set_final_preds(prev[0], prev[1])

    # -- mixed batches: differently sized images in one call --------------------------------------------------------
    def _grow(self, name, numel, dtype, pinned=False, bufs=None):
        """Grow-only buffer of the mixed path (``numel`` elements at least): its size follows the largest batch served,
        not the number of batch compositions.  ``bufs``: the dict it lives in, a list slot's own buffers (_mixed_init),
        or by default the buffers every list shares."""
        bufs = self._mixed_bufs if bufs is None else bufs
        buf = bufs.get(name)
        if buf is None or buf.numel() < numel or buf.dtype != dtype:
            if pinned:
                buf = torch.empty(max(int(numel), 1), dtype=dtype).pin_memory()
            else:
                buf = torch.empty(max(int(numel), 1), dtype=dtype, device=self.device)
            bufs[name] = buf
        return buf[:numel]

    def _mixed_init(self):
        """State of the list form, made on first use.  Every list shares, in stream order (each list's device work waits
        for the previous list's, ``_mixed_tail``, whatever stream that ran on): the input, det / tag and fast-grouping
        arenas (``_mixed_bufs``), the engine's arena plans and the ragged parser's top-K lists and workspaces - only
        device work reads them.  A list SLOT owns what is read after the list's device work has been queued, until its
        result is on the host: the pinned and device staging (images, descriptors, final-pred matrices), the payload
        rows, the pinned host rows and the ragged parser's results (read by fetch_overflow).  The blocking list form has
        one slot, submit_images two."""
        if hasattr(self, "_mixed_bufs"):
            return
        dev = self.device
        self._mixed_bufs = {}
        self._mixed_side = torch.cuda.Stream(device=dev)
        self._mixed_tail = None
        self._mixed_sync = self._list_slot()
        self._lists = {"slots": [self._list_slot(), self._list_slot()], "serial": 0,
                       "copy": torch.cuda.Stream(device=dev), "res": torch.cuda.Stream(device=dev)}

    @staticmethod
    def _list_slot():
        return {"bufs": {}, "parser": {}, "done": None, "busy": False, "serial": None}

    def _mixed_enqueue(self, images, mean, std, half, plant, slot, copy=None, rows=None):
        """The device work of one mixed list, queued on the current stream without synchronising the host.  Once per
        list: the images (arena order), descriptors and final-pred matrices are packed into ``slot``'s pinned staging
        buffer and leave in ONE H2D copy (on the stream ``copy`` when given, so that it overlaps device work already
        queued); per scale ONE ragged warp launch (lp_warp_affine_normalize_ragged_u8) into the input arena of that
        scale; per size group the network passes and the glue on the existing kernels (arena plans of the engine: their
        activation memory is shared by every group size), writing the group's slice of the det / tag arena; then ONE
        ragged parser chain over the whole arena into ``slot``'s result buffers, one get_final_preds launch with
        per-image matrices and one payload pack into the first N of ``slot``'s ``rows`` (default N) payload rows, in
        arena order.  Returns the list's record (plan, payload, parser results) for _fetch / collect_images."""
        import numpy as np
        from .mixed import MixedPlan, image_shapes
        shapes = image_shapes(images)
        n = len(shapes)
        if plant is not None and len(plant) != n:
            raise ValueError("infer_images: %d plant entries for %d images" % (len(plant), n))
        J, T = self.params.num_joints, self.T
        mp = MixedPlan(shapes, self.scales, int(self.cfg.DATASET.INPUT_SIZE), self.project, J, T)
        self._mixed_init()
        own = slot["bufs"]
        in_dtype = torch.float16 if half else torch.float32
        # (1) one pinned staging buffer: the images (arena order) followed by the descriptors and final-pred matrices
        descs = [mp.warp_desc(s).view(np.uint8) for s in self.scales]
        mdesc = mp.map_desc().view(np.uint8)
        trans = np.ascontiguousarray(mp.final_trans()).reshape(-1).view(np.uint8)
        blobs = descs + [mdesc, trans]
        img_bytes = int(mp.src_off[-1])
        offs, o = [], (img_bytes + 255) // 256 * 256
        for b in blobs:
            offs.append(o)
            o = (o + b.size + 255) // 256 * 256
        host = self._grow("stage", o, torch.uint8, pinned=True, bufs=own)
        hnp = host.numpy()
        dev_imgs = []
        for p, i in enumerate(mp.order):
            im = images[i]
            a, b = int(mp.src_off[p]), int(mp.src_off[p + 1])
            if torch.is_tensor(im) and im.is_cuda:
                dev_imgs.append((a, b, im))
            else:
                hnp[a:b] = (im.contiguous().numpy() if torch.is_tensor(im) else np.ascontiguousarray(im)).reshape(-1)
        for b, off in zip(blobs, offs):
            hnp[off:off + b.size] = b
        main = torch.cuda.current_stream()
        if self._mixed_tail is not None:
            main.wait_event(self._mixed_tail)
        if copy is None:
            d = self._grow("stage_dev", o, torch.uint8, bufs=own)
            d.copy_(host, non_blocking=True)
        else:
            with torch.cuda.stream(copy):
                # allocated from the copy stream's pool: a block the current stream has just freed may still be read by
                # work queued there, which this copy does not wait for
                d = self._grow("stage_dev", o, torch.uint8, bufs=own)
                if slot["done"] is not None:
                    copy.wait_event(slot["done"])        # this slot's previous list has read its staging
                d.copy_(host, non_blocking=True)
                h2d = torch.cuda.Event()
                h2d.record(copy)
            main.wait_event(h2d)
        for a, b, im in dev_imgs:                    # images already on the device: one device copy each
            d[a:b].copy_(im.reshape(-1))
        # (2) per scale one ragged warp + ToTensor + Normalize into the scale's input arena
        mean_a, std_a = np.asarray(mean, np.float32), np.asarray(std, np.float32)
        xs_arena = {}
        stream = main.cuda_stream
        for k, s in enumerate(self.scales):
            xa = self._grow("x%d" % k, int(mp.in_off[s][-1]), in_dtype)
            mh, mw = mp.max_in_hw(s)
            _lib.check(self.lib.lp_warp_affine_normalize_ragged_u8(
                d.data_ptr(), n, d.data_ptr() + offs[k], mw, mh, mean_a.ctypes.data, std_a.ctypes.data, xa.data_ptr(),
                2 if half else 1, stream), "lp_warp_affine_normalize_ragged_u8")
            xs_arena[s] = xa
        # (3) per size group: the network passes + glue on the existing kernels, into the group's arena slice
        det_a = self._grow("det", int(mp.det_off[-1]), torch.float32)
        tag_a = self._grow("tag", int(mp.tag_off[-1]), torch.float32)
        specs = []
        for g in mp.groups:
            for s in self.scales:
                hs, ws = g.in_hw[s]
                specs.append((g.n, hs, ws, in_dtype, True, False))
                if self.flip:
                    specs.append((g.n, hs, ws, in_dtype, True, True))
        self.engine.reserve_arena(specs)
        for g in mp.groups:
            p0, p1 = g.start, g.start + g.n
            hd, wd = g.det_hw
            det = det_a[int(mp.det_off[p0]):int(mp.det_off[p1])].view(g.n, J, hd, wd)
            tag_full = tag_a[int(mp.tag_off[p0]):int(mp.tag_off[p1])].view(g.n, J, hd, wd, T)
            tag = self._grow("tag_shared", g.n * hd * wd * T, torch.float32).view(g.n, 1, hd, wd, T) \
                if self.tag_shared else tag_full
            xs = {s: xs_arena[s][int(mp.in_off[s][p0]):int(mp.in_off[s][p1])].view(g.n, 3, *g.in_hw[s])
                  for s in self.scales}
            self._forward(xs, det, tag, self._mixed_side, None if plant is None else [plant[i] for i in g.images],
                          arena=True)
            if self.tag_shared and self.grouping == "fast":
                tag_full[:, :1].copy_(tag)          # the peak finder reads the shared map as plane 0 of the image's block
            elif self.tag_shared:
                tag_full.copy_(tag.expand(-1, J, -1, -1, -1))
        # (4) once per list: ragged parser, get_final_preds, payload
        hw = np.ascontiguousarray(mp.det_hw, np.int32)
        fb = None
        if self.grouping == "fast":
            fb = self._fast_buffers(n, J, lambda k, shape, dt: self._grow("fast_" + k, int(np.prod(shape)), dt).view(shape))
        width, rows = self.width, n if rows is None else rows
        packed = self._grow("packed", rows * width, torch.float32, bufs=own).view(rows, width)
        full = self._parse(det_a, tag_a, packed[:n], d.data_ptr() + offs[-1], fb, (hw, d.data_ptr() + offs[-2]),
                           slot["parser"])
        done = torch.cuda.Event()
        done.record(main)
        slot["done"] = self._mixed_tail = done
        # the caller's images and plant hooks stay referenced until the result has been read
        return {"plan": mp, "det": det_a, "tag": tag_a, "inputs": xs_arena, "packed": packed, "full": full, "n": n,
                "refs": (images, plant)}

    def infer_mixed(self, images, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), half=True, plant=None):
        """infer_images for a list of uint8 [H_i,W_i,3] images of any sizes.  Per image the result equals, bit for bit,
        infer_images(image[None]); the list comes back in the caller's order.  The images are grouped by their per-scale
        network sizes (litepose_b200.mixed.MixedPlan); _mixed_enqueue queues the list's device work, then ONE D2H copy
        and a synchronise.  Launches run eagerly (no CUDA graph: the composition changes from batch to batch)."""
        self._mixed_init()
        sl = self._mixed_sync
        rec = self._last_mixed = self._mixed_enqueue(images, mean, std, half, plant, sl)
        n = rec["n"]
        rec["host"] = self._grow("host", n * self.width, torch.float32, pinned=True, bufs=sl["bufs"]).view(n, self.width)
        res = self._fetch(rec)
        return [res[int(p)] for p in rec["plan"].pos]

    # -- asynchronous list API: two mixed lists in flight ---------------------------------------------------------------
    def submit_images(self, images, plant=None, group=None, dst=0, plan=None, mean=(0.485, 0.456, 0.406),
                      std=(0.229, 0.224, 0.225), half=True):
        """Asynchronous form of infer_images on a list of uint8 [H_i,W_i,3] images of any sizes (``plant``: one batch-1
        PlantedCrowd or None per image).  Returns an ImagesTicket; ``collect_images(ticket)`` returns exactly what
        infer_images(images) returns.  Nothing here synchronises the host: the list is staged in its slot's pinned
        buffer and copied on a copy stream, so that the staging and H2D copy of list i+1 overlap the device work of list
        i; the device work is queued on the current stream, and the payload rows leave through the result stream.  At
        most two lists may be outstanding (a third submit raises); their tickets are apart from those of submit().

        ``group`` (a torch.distributed process group of one rank per GPU): ``images`` is this rank's shard of a list
        split by ``plan`` = litepose_b200.dist.plan_shards(shapes, cfg, world), the same on every rank, in the order of
        plan.indices[rank].  Every rank's payload, padded to plan.rows rows, is gathered on rank ``dst`` with ONE NCCL
        gather on the result stream and leaves that rank in ONE device->host copy.  The gathered payload carries
        ``keep`` persons per image: collect_images raises for an image with more (use a larger ``keep``)."""
        import torch.distributed as dist
        self._mixed_init()
        world, rank = 1, 0
        if group is not None:
            if plan is None:
                raise ValueError("submit_images(group=...): pass the shard plan (litepose_b200.dist.plan_shards)")
            world, rank = dist.get_world_size(group), dist.get_rank(group)
            if plan.world != world:
                raise ValueError("submit_images: a plan over %d ranks for a group of %d" % (plan.world, world))
            mine = [plan.shapes[i] for i in plan.indices[rank]]
            from .mixed import image_shapes
            got = image_shapes(images) if len(images) else []
            if got != mine:
                raise ValueError("submit_images: rank %d's images must be the list's images plan.indices[%d], in that "
                                 "order (sizes %r, expected %r)" % (rank, rank, got, mine))
        a = self._lists
        free = [k for k, s in enumerate(a["slots"]) if not s["busy"]]
        if not free:
            raise RuntimeError("LitePosePipeline.submit_images: two lists are already in flight - collect_images() one "
                               "first")
        k = free[0]
        sl = a["slots"][k]
        width = self.width
        rows = plan.rows if group is not None else None
        if len(images) or group is None:
            rec = self._mixed_enqueue(images, mean, std, half, plant, sl, copy=a["copy"], rows=rows)
            if group is not None and rec["plan"].order != list(range(rec["n"])):
                # the gathered rows are in arena order; dst maps them back through plan.indices alone
                raise ValueError("submit_images: plan.indices[%d] is not in the arena order of this pipeline's sizes "
                                 "(a plan made for another TEST.SCALE_FACTOR or INPUT_SIZE)" % rank)
        else:
            # an empty shard still takes part in the gather (its rows are padding)
            rec = {"plan": None, "n": 0, "full": None, "refs": None,
                   "packed": self._grow("packed", rows * width, torch.float32, bufs=sl["bufs"]).view(rows, width)}
            done = torch.cuda.Event()
            done.record(torch.cuda.current_stream())
            sl["done"] = done
        own = sl["bufs"]
        res = a["res"]
        gathered = None
        if group is None:
            host = self._grow("host", rec["n"] * width, torch.float32, pinned=True, bufs=own).view(rec["n"], width)
        elif rank == dst:
            host = self._grow("host", world * rows * width, torch.float32, pinned=True, bufs=own).view(world, rows, width)
            if world > 1:
                gathered = self._grow("gather", world * rows * width, torch.float32, bufs=own).view(world, rows, width)
        else:
            host = None
        with torch.cuda.stream(res):
            res.wait_event(sl["done"])
            if group is not None and world > 1:
                from .dist import gather_rows
                gather_rows(rec["packed"], gathered, dst=dst, group=group)
                if gathered is not None:
                    host.copy_(gathered, non_blocking=True)
            elif host is not None:
                host.view(-1, width).copy_(rec["packed"], non_blocking=True)
            d2h = torch.cuda.Event()
            d2h.record(res)
        rec["host"] = host
        a["serial"] += 1
        sl.update(busy=True, serial=a["serial"], rec=rec, d2h=d2h, dist=(group is not None, rank, dst, plan))
        return ImagesTicket(self, k, a["serial"])

    def collect_images(self, ticket):
        """Wait for the list behind ``ticket`` (submit_images).  Without a group: the list over images, in the caller's
        order, that infer_images returns; an ae image with more than ``keep`` persons is read in full from the slot's
        parser buffers.  With a group: on ``dst`` the per-rank lists (rank r's in the order of plan.indices[r];
        litepose_b200.dist.merge_shards restores the caller's order), None on the other ranks."""
        if not isinstance(ticket, ImagesTicket):
            raise TypeError("collect_images: a ticket of submit_images expected, got %r" % (ticket,))
        a = getattr(self, "_lists", None)
        sl = a["slots"][ticket.slot] if a is not None and ticket.owner is self else None
        if sl is None or not sl["busy"] or sl["serial"] != ticket.serial:
            raise RuntimeError("LitePosePipeline.collect_images: %r is not in flight" % (ticket,))
        sl["d2h"].synchronize()
        rec = sl.pop("rec")
        sl["busy"] = False
        grouped, rank, dst, plan = sl["dist"]
        if not grouped:
            res = self._decode(rec["host"], rec)
            return [res[int(p)] for p in rec["plan"].pos]
        if rank != dst:
            return None
        from .dist import split_rows
        out = []
        for r, host in enumerate(split_rows(rec["host"], plan)):
            if self.grouping == "ae":
                over = (host[:, -1] > self.keep).nonzero().flatten().tolist()
                if over:
                    q = over[0]
                    raise _lib.LitePoseError(
                        "image %d of the list (rank %d's image %d) holds %d persons but the gathered payload carries "
                        "keep=%d: construct the pipeline with a larger keep (up to %d)"
                        % (plan.indices[r][q], r, q, int(host[q, -1]), self.keep, self.parser.pcap))
            out.append(self._decode(host))
        return out

    # -- asynchronous end-to-end API: two steps in flight -----------------------------------------
    def submit(self, frames_pinned, plant=None, group=None, dst=0):
        """Enqueue one end-to-end step and return a ticket; ``collect(ticket)`` blocks until that step's keypoints are
        on the host.  Nothing here synchronises the host: the pinned->device copy of the frames runs on a copy stream,
        the step on the current stream, and the packed result leaves through one of two result slots on a result
        stream (D2H of step i overlaps the compute of step i+1; with ``group`` - a torch.distributed process group of
        one rank per GPU - the slot is first gathered on rank ``dst`` with ONE NCCL gather and leaves that rank in
        ONE device->host copy).  At most two tickets may be outstanding.  An image with more persons than ``keep``
        makes collect() raise (never clipped): use the blocking step(), or a larger ``keep``.

        ``frames_pinned`` is read by the copy stream after this call has returned, and is not copied here: the caller
        must leave it unchanged until collect(ticket) has returned."""
        import torch.distributed as dist
        n, _, s_h, s_w = frames_pinned.shape
        main = torch.cuda.current_stream()
        a = self._async
        if a is None or a["key"] != (n, s_h, s_w, frames_pinned.dtype, id(group)):
            if a is not None and any(sl["busy"] for sl in a["slots"]):
                raise RuntimeError("LitePosePipeline.submit: collect() the outstanding tickets before changing the batch "
                                   "shape, dtype or group")
            world = dist.get_world_size(group) if group is not None else 1
            rank = dist.get_rank(group) if group is not None else 0
            width = self.width
            slots = []
            for _ in range(2):
                sl = {"x": torch.empty((n, 3, s_h, s_w), dtype=frames_pinned.dtype, device=self.device),
                      "out": torch.empty((n, width), dtype=torch.float32, device=self.device),
                      "step_done": None, "d2h_done": None, "busy": False}
                if world > 1 and rank == dst:
                    sl["all"] = torch.empty((world, n, width), dtype=torch.float32, device=self.device)
                sl["host"] = torch.empty((world if rank == dst else 1, n, width), dtype=torch.float32).pin_memory()
                slots.append(sl)
            a = self._async = {"key": (n, s_h, s_w, frames_pinned.dtype, id(group)), "slots": slots, "next": 0,
                               "copy": torch.cuda.Stream(device=self.device), "res": torch.cuda.Stream(device=self.device),
                               "world": world, "rank": rank, "dst": dst, "group": group}
        i = a["next"]
        sl = a["slots"][i]
        if sl["busy"]:
            raise RuntimeError("LitePosePipeline.submit: two steps are already in flight - collect() one first")
        a["next"] = i ^ 1
        with torch.cuda.stream(a["copy"]):
            if sl["step_done"] is not None:
                a["copy"].wait_event(sl["step_done"])        # the step that last read this input slot
            sl["x"].copy_(frames_pinned, non_blocking=True)
            h2d = torch.cuda.Event()
            h2d.record(a["copy"])
        main.wait_event(h2d)
        if sl["d2h_done"] is not None:
            main.wait_event(sl["d2h_done"])                  # the result slot is free again
        # network passes on this stream, parser of this step on the pipeline's parser stream (it overlaps the next
        # step's network passes); the payload leaves through the result stream once the parser has finished
        packed, parsed = self.step_device_overlapped(sl["x"], plant)
        sl["step_done"] = torch.cuda.Event()
        sl["step_done"].record(main)              # the input slot may be refilled after the network passes
        with torch.cuda.stream(a["res"]):
            a["res"].wait_event(parsed)
            sl["out"].copy_(packed, non_blocking=True)
            st = self._get_state(n, s_h, s_w, frames_pinned.dtype, plant)
            done = torch.cuda.Event()
            done.record(a["res"])
            st["ov"]["consumer_done"][st["ov_last"]] = done
            if a["world"] > 1:
                glist = list(sl["all"].unbind(0)) if a["rank"] == a["dst"] else None
                dist.gather(sl["out"], glist, dst=a["dst"], group=group)
                if a["rank"] == a["dst"]:
                    sl["host"].copy_(sl["all"], non_blocking=True)
            else:
                sl["host"][0].copy_(sl["out"], non_blocking=True)
            sl["d2h_done"] = torch.cuda.Event()
            sl["d2h_done"].record(a["res"])
        sl["busy"] = True
        return i

    def collect(self, ticket, unpack=True):
        """Wait for the step behind ``ticket``.  Returns, per rank of the group (one entry without a group), the list
        over images of (ans [P,J,3+T], scores, P); on ranks other than ``dst`` of a group: None.  With unpack=False the
        pinned host tensor [ranks, N, width] itself is returned."""
        a = self._async
        sl = a["slots"][ticket]
        if not sl["busy"]:
            raise RuntimeError("LitePosePipeline.collect: ticket %r is not in flight" % (ticket,))
        sl["d2h_done"].synchronize()
        sl["busy"] = False
        if a["world"] > 1 and a["rank"] != a["dst"]:
            return None
        host = sl["host"]
        if self.grouping == "ae":
            if float(host[:, :, -1].max()) > self.keep:
                raise _lib.LitePoseError("an image holds more persons than the packed payload carries (%d): use step() "
                                         "or a larger keep" % self.keep)
            if not unpack:
                return host
        res = [self._decode(host[r]) for r in range(host.shape[0])]      # fast: raises on a KM status 1
        return res if unpack else host

    def fetch_overflow(self, st, host):
        """Second-chance copy for the images that found more than ``keep`` persons: {image index: (ans, scores)} read
        from the parser's own buffers of the step that produced ``host`` (must be called before the next step)."""
        counts = host[:, -1]
        over = (counts > self.keep).nonzero().flatten().tolist()
        if not over:
            return None
        ans, num, scores = st["full"]
        out = {}
        for i in over:
            p = int(counts[i])
            if p > ans.shape[1]:
                raise _lib.LitePoseError("person capacity exceeded: %d > %d" % (p, ans.shape[1]))
            out[i] = (ans[i, :p].cpu().numpy(), scores[i, :p].cpu().numpy())
        return out

    def unpack(self, host, row, T, overflow=None):
        """packed host tensor -> list over images of (ans ndarray [P,J,3+T], scores list, P).  Every person is
        returned: an image with P > keep needs its entry in ``overflow`` (fetch_overflow), else this raises."""
        a = host.numpy()
        J, k = self.params.num_joints, self.keep
        out = []
        for i in range(a.shape[0]):
            p = int(a[i, -1])
            if p > k:
                if overflow is None or i not in overflow:
                    raise _lib.LitePoseError("image %d holds %d persons but the packed payload carries %d: pass the "
                                             "result of fetch_overflow() or raise keep" % (i, p, k))
                ans, sc = overflow[i]
                out.append((ans.copy(), list(sc), p))
                continue
            ans = a[i, :k * row].reshape(k, J, 3 + T)[:p].copy()
            sc = a[i, k * row:k * row + k][:p].copy()
            out.append((ans, list(sc), p))
        return out
