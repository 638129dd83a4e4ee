"""Host-side driver of the device associative-embedding parser (G1-G7 of SURVEY.md §8a).

Runs the reference ``HeatmapParser.parse`` pipeline (reference lib/core/group.py:269-291)
for a whole batch on the GPU: NMS+top-K, tag matching (Munkres), adjust, scores, refine,
with one D2H copy of the packed result at the end.  A batch of N images equals N
independent reference ``parse`` calls (the reference API is batch-1, SURVEY H5).
"""
import os
import re

import numpy as np
import torch

from . import _lib


def _header_define(name):
    path = os.path.join(os.path.dirname(_lib.HERE), "include", "litepose_b200.h")
    with open(path) as f:
        return int(re.search(r"#define\s+%s\s+(\d+)" % name, f.read()).group(1))


# the most top-K slots and matcher columns the parser kernels hold; the kernels refuse more with LP_ERR_BAD_ARG
PARSER_MAX_PEOPLE = _header_define("LP_PARSER_MAX_PEOPLE")


def check_max_people(max_num_people):
    """MAX_NUM_PEOPLE is K, the top-K slots per joint and the side of the matcher's cost matrices; the kernels take up
    to LP_PARSER_MAX_PEOPLE (include/litepose_b200.h)."""
    bound = PARSER_MAX_PEOPLE
    if int(max_num_people) > bound:
        raise ValueError("MAX_NUM_PEOPLE=%d exceeds LP_PARSER_MAX_PEOPLE=%d, the most top-K slots and matcher columns "
                         "the parser kernels hold" % (int(max_num_people), bound))


class DeviceParser(object):
    def __init__(self, num_joints, max_num_people, detection_threshold, tag_threshold, use_detection_val,
                 ignore_too_much, joint_order, nms_kernel, nms_padding=None):
        if nms_padding is not None and nms_kernel != 2 * nms_padding + 1:
            raise ValueError("NMS window must be centred: NMS_KERNEL == 2*NMS_PADDING+1 (got %d, %d)"
                             % (nms_kernel, nms_padding))
        if detection_threshold < 0:
            raise ValueError("DETECTION_THRESHOLD must be >= 0 (slots with val <= 0 are canonicalised)")
        check_max_people(max_num_people)
        self.lib = _lib.load()
        self.J = int(num_joints)
        self.K = int(max_num_people)
        self.det_thr = float(detection_threshold)
        self.tag_thr = float(tag_threshold)
        self.use_det_val = 1 if use_detection_val else 0
        self.ignore_too_much = 1 if ignore_too_much else 0
        self.joint_order = [int(v) for v in joint_order[: self.J]]
        self.nms_kernel = int(nms_kernel)
        self.pcap = self.J * self.K          # worst case: every candidate founds a person
        # K > 64: the uniform top-K and matching entry points keep their K <= 64 contract, so a uniform batch goes
        # through the ragged ones as N equal map descriptors (per image the same results)
        self.uniform_as_ragged = self.K > 64
        self._bufs = {}
        self._jo = {}

    def _buffers(self, dev, n, h, w, t):
        key = (dev, n, h, w, t)
        b = self._bufs.get(key)
        if b is None:
            J, K, pcap, lib = self.J, self.K, self.pcap, self.lib
            f32, i32, u8 = torch.float32, torch.int32, torch.uint8
            b = {
                "val_k": torch.empty((n, J, K), dtype=f32, device=dev),
                "ind_k": torch.empty((n, J, K), dtype=i32, device=dev),
                "tag_k": torch.empty((n, J, K, t), dtype=f32, device=dev),
                "ans": torch.empty((n, pcap, J, 3 + t), dtype=f32, device=dev),
                "num": torch.empty((n,), dtype=i32, device=dev),
                "scores": torch.empty((n, pcap), dtype=f32, device=dev),
                "ws_topk": torch.empty(max(1, lib.lp_nms_topk_workspace_bytes(n, J, h, w, K)), dtype=u8, device=dev)
                if not self.uniform_as_ragged else None,
                "ws_match": torch.empty(max(1, lib.lp_tag_match_workspace_bytes(n, J, K, t, pcap)), dtype=u8, device=dev),
                "ws_ref": torch.empty(max(1, lib.lp_adjust_refine_workspace_bytes(n, J, pcap)), dtype=u8, device=dev),
            }
            if self.uniform_as_ragged:
                from .mixed import MAP_DESC
                hw = np.ascontiguousarray(np.tile([[h, w]], (n, 1)), np.int32)
                desc = np.zeros(n, MAP_DESC)
                desc["h"], desc["w"] = h, w
                desc["det_offset"] = np.arange(n) * (J * h * w)
                desc["tag_offset"] = np.arange(n) * (J * h * w * t)
                b["hw"] = hw
                b["desc"] = torch.from_numpy(desc.view(np.uint8)).to(dev)
                b["ws_topk"] = torch.empty(max(1, lib.lp_nms_topk_ragged_workspace_bytes(n, hw.ctypes.data, J, K)),
                                           dtype=u8, device=dev)
            self._bufs[key] = b
        if dev not in self._jo:
            self._jo[dev] = torch.tensor(self.joint_order, dtype=torch.int32, device=dev)
        return b, self._jo[dev]

    # ---- stages (device tensors in, device tensors out; all on the current stream)
    def top_k_device(self, det, tag, min_value=0.0):
        """min_value 0: the reference's top_k.  run() passes the detection threshold: match_by_tag discards
        val <= DETECTION_THRESHOLD first (reference group.py:43-45), so the result of the parse is unchanged."""
        n, j, h, w = det.shape
        t = tag.shape[4]
        assert j == self.J and det.dtype == torch.float32 and tag.dtype == torch.float32
        det, tag = det.contiguous(), tag.contiguous()
        b, _ = self._buffers(det.device, n, h, w, t)
        s = torch.cuda.current_stream().cuda_stream
        if self.uniform_as_ragged:
            _lib.check(self.lib.lp_nms_topk_ragged_f32(
                det.data_ptr(), tag.data_ptr(), n, b["hw"].ctypes.data, b["desc"].data_ptr(), j, t, self.nms_kernel,
                self.K, float(min_value), b["val_k"].data_ptr(), b["ind_k"].data_ptr(), b["tag_k"].data_ptr(),
                b["ws_topk"].data_ptr(), b["ws_topk"].numel(), s), "lp_nms_topk_ragged_f32")
            return b["val_k"], b["ind_k"], b["tag_k"]
        _lib.check(self.lib.lp_nms_topk_f32(det.data_ptr(), tag.data_ptr(), n, j, h, w, t, self.nms_kernel, self.K,
                                            float(min_value), b["val_k"].data_ptr(), b["ind_k"].data_ptr(), b["tag_k"].data_ptr(),
                                            b["ws_topk"].data_ptr(), b["ws_topk"].numel(), s), "lp_nms_topk_f32")
        return b["val_k"], b["ind_k"], b["tag_k"]

    def match_device(self, dev, n, h, w, t):
        """tag matching on the top-K buffers of the (n, h, w, t) shape left by top_k_device -> device (ans, num)"""
        b, jo = self._buffers(dev, n, h, w, t)
        s = torch.cuda.current_stream().cuda_stream
        j = self.J
        tail = (jo.data_ptr(), self.det_thr, self.tag_thr, self.use_det_val, self.ignore_too_much, self.K, self.pcap,
                b["ans"].data_ptr(), b["num"].data_ptr(), b["ws_match"].data_ptr(), b["ws_match"].numel(), s)
        if self.uniform_as_ragged:
            _lib.check(self.lib.lp_tag_match_ragged_f32(b["val_k"].data_ptr(), b["ind_k"].data_ptr(),
                                                        b["tag_k"].data_ptr(), n, j, self.K, t, b["desc"].data_ptr(),
                                                        *tail), "lp_tag_match_ragged_f32")
        else:
            _lib.check(self.lib.lp_tag_match_f32(b["val_k"].data_ptr(), b["ind_k"].data_ptr(), b["tag_k"].data_ptr(),
                                                 n, j, self.K, t, w, *tail), "lp_tag_match_f32")
        return b["ans"], b["num"]

    def run(self, det, tag, adjust=True, refine=True):
        """det [N,J,H,W] fp32 CUDA, tag [N,J,H,W,T] fp32 CUDA -> device (ans, num_people, scores)."""
        if not det.is_cuda:
            raise RuntimeError("litepose_b200 parser runs on CUDA tensors only (no CPU fallback)")
        if tag.dim() == 4:
            tag = tag.unsqueeze(4)
        det, tag = det.contiguous(), tag.contiguous()
        n, j, h, w = det.shape
        t = tag.shape[4]
        with torch.cuda.device(det.device):
            b, jo = self._buffers(det.device, n, h, w, t)
            s = torch.cuda.current_stream().cuda_stream
            self.top_k_device(det, tag, self.det_thr)
            self.match_device(det.device, n, h, w, t)
            _lib.check(self.lib.lp_adjust_refine_f32(
                det.data_ptr(), tag.data_ptr(), n, j, h, w, t, self.pcap, b["ans"].data_ptr(), b["num"].data_ptr(),
                b["scores"].data_ptr(), 1 if adjust else 0, 1 if refine else 0, b["ws_ref"].data_ptr(),
                b["ws_ref"].numel(), s), "lp_adjust_refine_f32")
        return b["ans"], b["num"], b["scores"]

    def _ragged_buffers(self, dev, n, t, ws_topk, ws_match, ws_ref, outs=None):
        """Grow-only buffers of run_ragged: one set, sized for the largest batch seen (not one per composition).  The
        results (ans, num, scores) grow in ``outs`` instead when the caller passes its own dict."""
        J, K, pcap = self.J, self.K, self.pcap
        sizes = {"val_k": (n * J * K, torch.float32), "ind_k": (n * J * K, torch.int32),
                 "tag_k": (n * J * K * t, torch.float32), "ans": (n * pcap * J * (3 + t), torch.float32),
                 "num": (n, torch.int32), "scores": (n * pcap, torch.float32), "ws_topk": (ws_topk, torch.uint8),
                 "ws_match": (ws_match, torch.uint8), "ws_ref": (ws_ref, torch.uint8)}
        bufs = self._bufs.setdefault(("ragged", dev), {})
        out = {}
        for name, (numel, dtype) in sizes.items():
            home = outs if outs is not None and name in ("ans", "num", "scores") else bufs
            b = home.get(name)
            if b is None or b.numel() < numel:
                b = home[name] = torch.empty(max(int(numel), 1), dtype=dtype, device=dev)
            out[name] = b[:max(int(numel), 1)]
        if dev not in self._jo:
            self._jo[dev] = torch.tensor(self.joint_order, dtype=torch.int32, device=dev)
        return out, self._jo[dev]

    def workspace_bytes_ragged(self, hw, t):
        """(top-K, matching, adjust/refine) workspace bytes of a ragged call on maps of the sizes ``hw`` [N,2]."""
        hw = np.ascontiguousarray(hw, np.int32)
        n = hw.shape[0]
        return (int(self.lib.lp_nms_topk_ragged_workspace_bytes(n, hw.ctypes.data, self.J, self.K)),
                int(self.lib.lp_tag_match_workspace_bytes(n, self.J, self.K, t, self.pcap)),
                int(self.lib.lp_adjust_refine_workspace_bytes(n, self.J, self.pcap)))

    def run_ragged(self, det, tag, hw, desc, t, adjust=True, refine=True, outs=None):
        """The parse of run() on a det / tag arena of differently sized maps: image i's [J,h_i,w_i] det block and
        [J,h_i,w_i,T] tag block sit at the offsets of ``desc`` (device pointer to N lp_map_desc_t,
        litepose_b200.mixed.MAP_DESC); ``hw`` [N,2] int32 host array = the same sizes.  One ragged chain (NMS/top-K, tag
        matching, adjust/scores/refine) for the whole batch.  Per image the results equal, bit for bit, run() on that
        image alone.  Returns device (ans [N,pcap,J,3+T], num [N], scores [N,pcap]) in grow-only buffers, valid until
        the next ragged call with the same ``outs``: a caller's dict that owns the result buffers (None: the parser's
        own).  The top-K lists and workspaces are shared by every call, in stream order."""
        if not det.is_cuda:
            raise RuntimeError("litepose_b200 parser runs on CUDA tensors only (no CPU fallback)")
        hw = np.ascontiguousarray(hw, np.int32)
        n, j = hw.shape[0], self.J
        ws = self.workspace_bytes_ragged(hw, t)
        with torch.cuda.device(det.device):
            b, jo = self._ragged_buffers(det.device, n, t, *ws, outs=outs)
            s = torch.cuda.current_stream().cuda_stream
            _lib.check(self.lib.lp_nms_topk_ragged_f32(
                det.data_ptr(), tag.data_ptr(), n, hw.ctypes.data, desc, j, t, self.nms_kernel, self.K, self.det_thr,
                b["val_k"].data_ptr(), b["ind_k"].data_ptr(), b["tag_k"].data_ptr(), b["ws_topk"].data_ptr(),
                b["ws_topk"].numel(), s), "lp_nms_topk_ragged_f32")
            ans = b["ans"].view(n, self.pcap, j, 3 + t)
            _lib.check(self.lib.lp_tag_match_ragged_f32(
                b["val_k"].data_ptr(), b["ind_k"].data_ptr(), b["tag_k"].data_ptr(), n, j, self.K, t, desc,
                jo.data_ptr(), self.det_thr, self.tag_thr, self.use_det_val, self.ignore_too_much, self.K,
                self.pcap, ans.data_ptr(), b["num"].data_ptr(), b["ws_match"].data_ptr(), b["ws_match"].numel(), s),
                "lp_tag_match_ragged_f32")
            _lib.check(self.lib.lp_adjust_refine_ragged_f32(
                det.data_ptr(), tag.data_ptr(), n, hw.ctypes.data, desc, j, t, self.pcap, ans.data_ptr(),
                b["num"].data_ptr(), b["scores"].data_ptr(), 1 if adjust else 0, 1 if refine else 0,
                b["ws_ref"].data_ptr(), b["ws_ref"].numel(), s), "lp_adjust_refine_ragged_f32")
        self.last_ragged = b
        return ans, b["num"], b["scores"].view(n, self.pcap)

    @staticmethod
    def to_reference(ans, num, scores):
        """Device results -> list over images of (ans, scores) in the reference's return
        types: ans = float32 ndarray [P,J,3+T] (iterates over persons); scores = list of float32."""
        num_h = num.cpu().numpy()
        pmax = int(num_h.max()) if num_h.size else 0
        if pmax > ans.shape[1]:
            raise _lib.LitePoseError("person capacity exceeded: %d > %d" % (pmax, ans.shape[1]))
        ans_h = ans[:, :max(pmax, 1)].cpu().numpy()
        sc_h = scores[:, :max(pmax, 1)].cpu().numpy()
        out = []
        for i in range(ans_h.shape[0]):
            p = int(num_h[i])
            out.append((ans_h[i, :p].copy(), [sc_h[i, q] for q in range(p)]))
        return out
