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
from .parser import DeviceParser


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
        if grouping == "fast":
            from .fast_utils.group import Params as FastParams
            fp = FastParams(cfg)
            J = p.num_joints
            # the demo's parser hands joint_order to assign(), which reads the first C entries: the entries that name no
            # plane are dropped, as fast_utils.group.HeatmapParser._joint_order does
            self.fast = {"M": int(fp.max_num_people), "thr": float(fp.detection_threshold), "win": int(fp.window_size),
                         "tag_thr": float(fp.tag_threshold),
                         "jo": torch.tensor([j for j in fp.joint_order if j < J][:J], dtype=torch.int32,
                                            device=self.device)}
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
    def _network_part(self, st, x, slot=0, arena=False):
        """Both network passes -> ([o0, o1], [f0, f1]) in the engine's buffer set ``slot`` (``arena``: in the engine's
        shared arena plans, see LitePoseEngine.arena_plan_for)."""
        eng = self.engine
        if not self.flip:
            return eng.run(x, flip=False, out_fp32=True, clone=False, slot=slot, arena=arena), None
        # the plain and the mirrored pass are independent until the glue: fork onto a side stream so that one pass'
        # kernels fill the launch gaps and tails of the other (each pass has its own plan buffers)
        main = torch.cuda.current_stream()
        side = st["side"]
        side.wait_stream(main)
        with torch.cuda.stream(side):
            f = eng.run(x, flip=True, out_fp32=True, clone=False, slot=slot, arena=arena)
        o = eng.run(x, flip=False, out_fp32=True, clone=False, slot=slot, arena=arena)
        main.wait_stream(side)
        return o, f

    def _glue_part(self, st, o, f, det, tag):
        """Fused glue (+ the benchmark's planted persons) on the four model outputs -> det / tag of this step."""
        J = self.params.num_joints
        o0, o1 = o[0], o[1]
        n, _, h, w = o0.shape
        Hd, Wd = det.shape[2], det.shape[3]
        fl = 1 if self.flip else 0
        f0, f1 = (f[0].data_ptr(), f[1].data_ptr()) if self.flip else (None, None)
        stream = torch.cuda.current_stream().cuda_stream
        if self.canonical:
            _lib.check(self.lib.lp_glue_f32(o0.data_ptr(), o1.data_ptr(), f0, f1, self.fidx.data_ptr(), n, J, h, w, fl, Hd,
                                            Wd, det.data_ptr(), tag.data_ptr(), stream), "lp_glue_f32")
        else:
            _lib.check(self.lib.lp_glue_scale_f32(o0.data_ptr(), o1.data_ptr(), f0, f1, self.fidx.data_ptr(), n, J,
                                                  self.model_joints, 1 if self.tag_shared else 0, h, w, fl, Hd, Wd, 0, 1.0,
                                                  det.data_ptr(), tag.data_ptr(), stream), "lp_glue_scale_f32")
        if st["plant"] is not None:
            st["plant"].apply(det, tag)

    def _forward_part(self, st, x, det, tag):
        """Both network passes + fused glue (+ the benchmark's planted persons) -> det / tag of this step."""
        o, f = self._network_part(st, x)
        self._glue_part(st, o, f, det, tag)

    def _parser_part(self, st, det, tag, packed):
        """Device parser (+ get_final_preds) on det / tag -> packed fixed-size payload."""
        n = det.shape[0]
        if self.grouping == "fast":
            return self._fast_parser_part(st, det, tag, packed)
        if self.tag_shared:
            # MODEL.TAG_PER_JOINT off: the one tag map serves every joint (group.py:150-152); the parser kernels index
            # [N,J,H,W,T], so the map is tiled here (one strided copy; not the shipped configuration)
            tag = tag.expand(-1, det.shape[1], -1, -1, -1).contiguous()
        ans, num, scores = self.parser.run(det, tag, self.adjust, self.refine)
        if st["trans"] is not None:
            _lib.check(self.lib.lp_transform_preds_f32(ans.data_ptr(), num.data_ptr(), st["trans"].data_ptr(), n,
                                                       ans.shape[1], ans.shape[2], ans.shape[3],
                                                       torch.cuda.current_stream().cuda_stream), "lp_transform_preds_f32")
        st["full"] = (ans, num, scores)       # parser-owned buffers (capacity J*K persons), valid until the next step
        _lib.check(self.lib.lp_pack_payload_f32(ans.data_ptr(), num.data_ptr(), scores.data_ptr(), n, ans.shape[1],
                                                st["row"], self.keep, packed.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream), "lp_pack_payload_f32")
        return packed

    def _fast_buffers(self, n, J, alloc=None):
        """Peaks, persons and status of the fast grouping for n images; ``alloc(name, shape, dtype)`` (default: new
        device tensors) lets the mixed path serve them from its grow-only buffers."""
        if alloc is None:
            alloc = lambda name, shape, dt: torch.empty(shape, dtype=dt, device=self.device)
        f32, i32, M = torch.float32, torch.int32, self.fast["M"]
        spec = {"count": ((n, J), i32), "val": ((n, J, M), f32), "tag": ((n, J, M), f32), "ind": ((n, J, M, 2), i32),
                "ans": ((n, M, J, 4), f32), "num": ((n,), i32), "status": ((n,), i32)}
        return {k: alloc(k, shape, dt) for k, (shape, dt) in spec.items()}

    def _fast_parse(self, b, det, tag, n, J, T, tag_planes, hw, desc, trans, packed):
        """The demo's parser on det / tag where the glue left them: zero ans, find peaks (tag channel 0 read in place),
        KM assignment, get_final_preds (``trans``: device [N,6] float64 or None), pack.  Uniform maps: ``hw`` / ``desc``
        None, det [N,J,H,W]; ragged arena: ``hw`` [N,2] host int32 and ``desc`` the device lp_map_desc_t pointer."""
        f, M = self.fast, self.fast["M"]
        s = torch.cuda.current_stream().cuda_stream
        ans = b["ans"]
        # lp_assign_f32 writes only the entries it assigns: without this the rows of the previous step would remain
        ans.zero_()
        H, W = (det.shape[2], det.shape[3]) if desc is None else (0, 0)
        _lib.check(self.lib.lp_find_peaks_maps_f32(
            det.data_ptr(), tag.data_ptr(), n, H, W, None if hw is None else hw.ctypes.data, desc, J, T, tag_planes, M,
            f["thr"], f["win"], b["count"].data_ptr(), b["val"].data_ptr(), b["tag"].data_ptr(), b["ind"].data_ptr(), s),
            "lp_find_peaks_maps_f32")
        _lib.check(self.lib.lp_assign_f32(b["count"].data_ptr(), b["val"].data_ptr(), b["tag"].data_ptr(),
                                          b["ind"].data_ptr(), f["jo"].data_ptr(), n, J, M, f["tag_thr"],
                                          b["num"].data_ptr(), ans.data_ptr(), b["status"].data_ptr(), s), "lp_assign_f32")
        if trans is not None:
            _lib.check(self.lib.lp_transform_preds_f32(ans.data_ptr(), b["num"].data_ptr(), trans, n, M, J, 4, s),
                       "lp_transform_preds_f32")
        _lib.check(self.lib.lp_pack_fast_payload_f32(ans.data_ptr(), b["num"].data_ptr(), b["status"].data_ptr(), n, M,
                                                     J, packed.data_ptr(), s), "lp_pack_fast_payload_f32")
        return packed

    def _fast_parser_part(self, st, det, tag, packed):
        n, J = det.shape[0], det.shape[1]
        trans = st["trans"].data_ptr() if st["trans"] is not None else None
        return self._fast_parse(st["fast"], det, tag, n, J, tag.shape[4], tag.shape[1], None, None, trans, packed)

    def unpack_fast(self, host):
        """Fast-grouping payload (host) -> list over images of (ans ndarray [P,J,4], P); see unpack_fast_payload."""
        return unpack_fast_payload(host, self.fast["M"], self.params.num_joints)

    def _result(self, st, host):
        """Host payload of a blocking call -> per-image results of the pipeline's grouping mode."""
        if self.grouping == "fast":
            return self.unpack_fast(host)
        return self.unpack(host, st["row"], st["T"], self.fetch_overflow(st, host))

    # -- device step (everything between the H2D copy and the D2H copy) -------------
    def _device_step(self, st, x):
        self._forward_part(st, x, st["det"], st["tag"])
        return self._parser_part(st, st["det"], st["tag"], st["packed"])

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
            self.engine.use_graphs = False
            o, f = self._network_part(st, st["x"], slot=b)       # warm-up: builds plans, sets attributes
            self._glue_part(st, o, f, ov["det"][b], ov["tag"][b])
            self._parser_part(st, ov["det"][b], ov["tag"][b], ov["packed"][b])
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                o, f = self._network_part(st, st["x"], slot=b)
            ov["gF"][b] = g
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                # the glue writes 1.4 GB at the HBM write roofline: on the second stream it overlaps the FMA-bound network
                # passes of the next step (which write the other buffer set of the engine)
                self._glue_part(st, o, f, ov["det"][b], ov["tag"][b])
                self._parser_part(st, ov["det"][b], ov["tag"][b], ov["packed"][b])
            ov["gP"][b] = g
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
            T = 2 if self.flip else 1
            Hd, Wd = det_hw if det_hw is not None else ((s_h, s_w) if self.project else (s_h // 2, s_w // 2))
            dev = self.device
            row = J * (3 + T)
            width = self.keep * row + self.keep + 1
            if self.grouping == "fast":            # every person (M <= 32) x J x (x, y, val, tag) | count | KM status
                width = self.fast["M"] * J * 4 + 2
            st = {
                "x": torch.empty((n, 3, s_h, s_w), dtype=dtype, device=dev),
                "side": torch.cuda.Stream(device=dev),
                "det": torch.empty((n, J, Hd, Wd), dtype=torch.float32, device=dev),
                "tag": torch.empty((n, 1 if self.tag_shared else J, Hd, Wd, T), dtype=torch.float32, device=dev),
                "packed": torch.zeros((n, width), dtype=torch.float32, device=dev),
                "host": torch.empty((n, width), dtype=torch.float32).pin_memory(),
                "row": row, "T": T, "graph": None, "plant": plant, "trans": None, "full": None, "ov": None,
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
        st = self._get_state(n, s_h, s_w, x_dev.dtype, plant)
        ov = st.get("ov")
        if ov is not None:
            # det / tag / packed are shared with buffer set 0 of the overlapped form: an overlapped step that is still
            # running on the parser stream must finish before this stream overwrites them
            for ev in ov["P_done"]:
                if ev is not None:
                    torch.cuda.current_stream().wait_event(ev)
        if not self.use_graphs:
            return self._device_step(st, x_dev)
        st["x"].copy_(x_dev, non_blocking=True)
        if st["graph"] is None:
            self.engine.use_graphs = False
            self._device_step(st, st["x"])          # warm-up: builds plans, sets function attributes
            torch.cuda.current_stream().synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._device_step(st, st["x"])
            st["graph"] = g
        st["graph"].replay()
        return st["packed"]

    def step(self, frames_pinned, plant=None):
        """Public end-to-end call: pinned host frames in, host result out (blocking)."""
        x = frames_pinned.to(self.device, non_blocking=True)
        packed = self.step_device(x, plant)
        n = packed.shape[0]
        st = self._get_state(n, x.shape[2], x.shape[3], x.dtype, plant)
        st["host"].copy_(packed, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self._result(st, st["host"])

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
        x1 = xs[1.0]
        n = x1.shape[0]
        big = xs[scales[0]]
        det_hw = (x1.shape[2], x1.shape[3]) if self.project else (big.shape[2] // 2, big.shape[3] // 2)
        st = self._get_state(n, x1.shape[2], x1.shape[3], x1.dtype, plant, det_hw=det_hw)
        det, tag = st["det"], st["tag"]
        self.engine.use_graphs = False
        self._multiscale_part(st, xs, det, tag, det_hw)
        if st["plant"] is not None:
            st["plant"].apply(det, tag)
        return self._parser_part(st, det, tag, st["packed"])

    def _multiscale_part(self, st, xs, det, tag, det_hw, arena=False):
        """Per scale, largest first: both network passes and one lp_glue_scale_f32 launch accumulating into det (the
        tags from the scale-1 pass); the last launch divides by the number of scales."""
        scales = self.scales
        n = det.shape[0]
        J = self.params.num_joints
        stream = torch.cuda.current_stream().cuda_stream
        for i, s in enumerate(scales):
            x = xs[s]
            if x.shape[0] != n or x.shape[2] % 64 or x.shape[3] % 64:
                raise ValueError("step_device_multiscale: scale %r frames %r (batch %d, sides multiples of 64 expected)"
                                 % (s, tuple(x.shape), n))
            o, f = self._network_part(st, x, arena=arena)
            _, _, h, w = o[0].shape
            _lib.check(self.lib.lp_glue_scale_f32(
                o[0].data_ptr(), o[1].data_ptr(), f[0].data_ptr() if self.flip else None,
                f[1].data_ptr() if self.flip else None, self.fidx.data_ptr(), n, J, self.model_joints,
                1 if self.tag_shared else 0, h, w, 1 if self.flip else 0, det_hw[0], det_hw[1], 1 if i > 0 else 0,
                float(len(scales)) if i == len(scales) - 1 else 1.0,
                det.data_ptr(), tag.data_ptr() if s == 1.0 else None, stream), "lp_glue_scale_f32")

    def step_multiscale(self, frames, plant=None):
        """Public blocking call of the multi-scale test: {scale: pinned host frames} in, host result out (the list
        over images of (ans [P,J,3+T], scores, P), as step())."""
        xs = {float(s): f.to(self.device, non_blocking=True) for s, f in frames.items()}
        packed = self.step_device_multiscale(xs, plant)
        x1 = xs[1.0]
        big = xs[self.scales[0]]
        det_hw = (x1.shape[2], x1.shape[3]) if self.project else (big.shape[2] // 2, big.shape[3] // 2)
        st = self._get_state(x1.shape[0], x1.shape[2], x1.shape[3], x1.dtype, plant, det_hw=det_hw)
        st["host"].copy_(packed, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self._result(st, st["host"])

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
            x1 = xs[1.0]
            if len(self.scales) == 1:
                packed = self.step_device(x1, plant)
                det_hw = None
            else:
                packed = self.step_device_multiscale(xs, plant)
                big = xs[self.scales[0]]
                det_hw = (x1.shape[2], x1.shape[3]) if self.project else (big.shape[2] // 2, big.shape[3] // 2)
            st = self._get_state(n, x1.shape[2], x1.shape[3], x1.dtype, plant, det_hw=det_hw)
            self._last_state = st                 # det / tag of this call stay readable there until the next call
            st["host"].copy_(packed, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            return self._result(st, st["host"])
        finally:
            if prev is None:
                self.set_final_preds(None)
            else:
                self.set_final_preds(prev[0], prev[1])

    # -- mixed batches: differently sized images in one call --------------------------------------------------------
    def _grow(self, name, numel, dtype, pinned=False):
        """Grow-only buffer of the mixed path (``numel`` elements at least): its size follows the largest batch served,
        not the number of batch compositions."""
        buf = self._mixed_bufs.get(name)
        if buf is None or buf.numel() < numel or buf.dtype != dtype:
            if pinned:
                buf = torch.empty(max(int(numel), 1), dtype=dtype).pin_memory()
            else:
                buf = torch.empty(max(int(numel), 1), dtype=dtype, device=self.device)
            self._mixed_bufs[name] = buf
        return buf[:numel]

    def infer_mixed(self, images, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), half=True, plant=None):
        """infer_images for a list of uint8 [H_i,W_i,3] images of any sizes.  Per image the result equals, bit for bit,
        infer_images(image[None]); the list comes back in the caller's order.  The images are grouped by their per-scale
        network sizes (litepose_b200.mixed.MixedPlan).  Once per batch: one H2D copy of the packed images and
        descriptors, per scale ONE ragged warp launch (lp_warp_affine_normalize_ragged_u8) into the input arena of that
        scale; per size group the network passes and the glue on the existing kernels (arena plans of the engine: their
        activation memory is shared by every group size), writing the group's slice of the det / tag arena; then ONE
        ragged parser chain over the whole arena, one get_final_preds launch with per-image matrices, one payload pack
        and one D2H copy.  Launches run eagerly (no CUDA graph: the composition changes from batch to batch)."""
        import numpy as np
        from .mixed import MixedPlan, image_shapes
        shapes = image_shapes(images)
        n = len(shapes)
        if plant is not None and len(plant) != n:
            raise ValueError("infer_images: %d plant entries for %d images" % (len(plant), n))
        J = self.params.num_joints
        T = 2 if self.flip else 1
        mp = MixedPlan(shapes, self.scales, int(self.cfg.DATASET.INPUT_SIZE), self.project, J, T)
        if not hasattr(self, "_mixed_bufs"):
            self._mixed_bufs = {}
            self._mixed_side = torch.cuda.Stream(device=self.device)
        dev = self.device
        in_dtype = torch.float16 if half else torch.float32
        main = torch.cuda.current_stream()
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
        host = self._grow("stage", o, torch.uint8, pinned=True)
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
        d = self._grow("stage_dev", o, torch.uint8)
        d.copy_(host, non_blocking=True)
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
        self.engine.use_graphs = False
        specs = []
        for g in mp.groups:
            for s in self.scales:
                hs, ws = g.in_hw[s]
                specs.append((g.n, hs, ws, in_dtype, True, False))
                if self.flip:
                    specs.append((g.n, hs, ws, in_dtype, True, True))
        self.engine.reserve_arena(specs)
        st = {"side": self._mixed_side, "plant": None}
        for g in mp.groups:
            p0, p1 = g.start, g.start + g.n
            hd, wd = g.det_hw
            det = det_a[int(mp.det_off[p0]):int(mp.det_off[p1])].view(g.n, J, hd, wd)
            tag_full = tag_a[int(mp.tag_off[p0]):int(mp.tag_off[p1])].view(g.n, J, hd, wd, T)
            tag = self._grow("tag_shared", g.n * hd * wd * T, torch.float32).view(g.n, 1, hd, wd, T) \
                if self.tag_shared else tag_full
            xs = {s: xs_arena[s][int(mp.in_off[s][p0]):int(mp.in_off[s][p1])].view(g.n, 3, *g.in_hw[s])
                  for s in self.scales}
            if len(self.scales) == 1:
                o, f = self._network_part(st, xs[1.0], arena=True)
                self._glue_part(st, o, f, det, tag)
            else:
                self._multiscale_part(st, xs, det, tag, g.det_hw, arena=True)
            if plant is not None:
                for k, i in enumerate(g.images):
                    if plant[i] is not None:
                        plant[i].apply(det[k:k + 1], tag[k:k + 1])
            if self.tag_shared and self.grouping == "fast":
                tag_full[:, :1].copy_(tag)          # the peak finder reads the shared map as plane 0 of the image's block
            elif self.tag_shared:
                tag_full.copy_(tag.expand(-1, J, -1, -1, -1))
        # (4) once per batch: ragged parser, get_final_preds, payload, D2H
        hw = np.ascontiguousarray(mp.det_hw, np.int32)
        if self.grouping == "fast":
            M = self.fast["M"]
            b = self._fast_buffers(n, J, lambda k, shape, dt: self._grow("fast_" + k, int(np.prod(shape)), dt).view(shape))
            width = M * J * 4 + 2
            packed = self._grow("packed", n * width, torch.float32).view(n, width)
            self._fast_parse(b, det_a, tag_a, n, J, T, 1 if self.tag_shared else J, hw, d.data_ptr() + offs[-2],
                             d.data_ptr() + offs[-1], packed)
            out_h = self._grow("host", n * width, torch.float32, pinned=True).view(n, width)
            out_h.copy_(packed, non_blocking=True)
            main.synchronize()
            res = self.unpack_fast(out_h)
            self._last_mixed = {"plan": mp, "det": det_a, "tag": tag_a, "inputs": xs_arena}
            return [res[int(p)] for p in mp.pos]
        ans, num, scores = self.parser.run_ragged(det_a, tag_a, hw, d[offs[-2]:].data_ptr(), T, self.adjust, self.refine)
        pcap = ans.shape[1]
        _lib.check(self.lib.lp_transform_preds_f32(ans.data_ptr(), num.data_ptr(), d.data_ptr() + offs[-1], n, pcap, J,
                                                   ans.shape[3], stream), "lp_transform_preds_f32")
        row = J * (3 + T)
        width = self.keep * row + self.keep + 1
        packed = self._grow("packed", n * width, torch.float32).view(n, width)
        _lib.check(self.lib.lp_pack_payload_f32(ans.data_ptr(), num.data_ptr(), scores.data_ptr(), n, pcap, row,
                                                self.keep, packed.data_ptr(), stream), "lp_pack_payload_f32")
        out_h = self._grow("host", n * width, torch.float32, pinned=True).view(n, width)
        out_h.copy_(packed, non_blocking=True)
        main.synchronize()
        res = self.unpack(out_h, row, T, self.fetch_overflow({"full": (ans, num, scores)}, out_h))
        self._last_mixed = {"plan": mp, "det": det_a, "tag": tag_a, "inputs": xs_arena}
        return [res[int(p)] for p in mp.pos]

    # -- asynchronous end-to-end API: two steps in flight -----------------------------------------
    def submit(self, frames_pinned, plant=None, group=None, dst=0):
        """Enqueue one end-to-end step and return a ticket; ``collect(ticket)`` blocks until that step's keypoints are
        on the host.  Nothing here synchronises the host: the pinned->device copy of the frames runs on a copy stream,
        the step on the current stream, and the packed result leaves through one of two result slots on a result
        stream (D2H of step i overlaps the compute of step i+1; with ``group`` - a torch.distributed process group of
        one rank per GPU - the slot is first gathered on rank ``dst`` with ONE NCCL gather and leaves that rank in
        ONE device->host copy).  At most two tickets may be outstanding.  An image with more persons than ``keep``
        makes collect() raise (never clipped): use the blocking step(), or a larger ``keep``."""
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
            st = self._get_state(n, s_h, s_w, frames_pinned.dtype, plant)
            width = st["packed"].shape[1]
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
                               "world": world, "rank": rank, "dst": dst, "group": group, "row": st["row"], "T": st["T"]}
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
            st_ = self._get_state(n, s_h, s_w, frames_pinned.dtype, plant)
            done = torch.cuda.Event()
            done.record(a["res"])
            st_["ov"]["consumer_done"][st_["ov_last"]] = done
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
        if self.grouping == "fast":
            res = [self.unpack_fast(sl["host"][r]) for r in range(sl["host"].shape[0])]      # raises on a KM status 1
            return res if unpack else sl["host"]
        if float(sl["host"][:, :, -1].max()) > self.keep:
            raise _lib.LitePoseError("an image holds more persons than the packed payload carries (%d): use step() or "
                                     "a larger keep" % self.keep)
        if not unpack:
            return sl["host"]
        return [self.unpack(sl["host"][r], a["row"], a["T"]) for r in range(sl["host"].shape[0])]

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
