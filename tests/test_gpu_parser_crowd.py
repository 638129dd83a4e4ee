"""-m gpu: the evaluation parser past 64 persons (64 < MAX_NUM_PEOPLE = K <= LP_PARSER_MAX_PEOPLE), bit for bit against
oracle/group_ref: the wide top-K (per-CTA candidate buffers) at every strip geometry with ties, NaN / inf / subnormal /
-0.0 pixels, tall planes, the width bound and ragged descriptors; the one-CTA-per-image matcher on the crowd goldens and
on the matcher edge families scaled past 64; adjust + refine at pcap = J * 256; the pipeline entry points at K = 128;
and the memory footprint of the new shapes (guard bands, poisoned neighbours, untouched inputs)."""
import os

import numpy as np
import pytest
import torch

from footprint_util import Guarded, Plain
from parity_util import assert_topk_equal
from litepose_b200 import _lib, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.mixed import MAP_DESC
from oracle import group_ref
from oracle import parser_cases as pc
from oracle.make_golden_parser_crowd import CROWD_CASES, crowd_inputs, digest
from oracle.make_golden_parser_edges import run_adjust_refine

pytestmark = pytest.mark.gpu

LP_ERR_BAD_ARG = 1


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _equal_desc(n, J, H, W, T):
    """the map descriptors of a uniform [n, J, H, W(, T)] batch: K > 64 runs through the ragged entry points"""
    desc = np.zeros(n, MAP_DESC)
    desc["h"], desc["w"] = H, W
    desc["det_offset"] = np.arange(n) * (J * H * W)
    desc["tag_offset"] = np.arange(n) * (J * H * W * T)
    return desc, np.ascontiguousarray(np.tile([[H, W]], (n, 1)), np.int32)


# ---- NMS + top-K, K > 64
def _topk_device(det, tag, kernel, K, min_value):
    lib = _lib.load()
    n, J, H, W = det.shape
    T = tag.shape[-1]
    d, t = torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda()
    val = torch.empty((n, J, K), device="cuda")
    ind = torch.empty((n, J, K), dtype=torch.int32, device="cuda")
    tk = torch.empty((n, J, K, T), device="cuda")
    desc, hw = _equal_desc(n, J, H, W, T)
    dd = torch.from_numpy(desc.view(np.uint8)).cuda()
    ws = torch.empty(lib.lp_nms_topk_ragged_workspace_bytes(n, hw.ctypes.data, J, K), dtype=torch.uint8, device="cuda")
    rc = lib.lp_nms_topk_ragged_f32(d.data_ptr(), t.data_ptr(), n, hw.ctypes.data, dd.data_ptr(), J, T, kernel, K,
                                    float(min_value), val.data_ptr(), ind.data_ptr(), tk.data_ptr(), ws.data_ptr(),
                                    ws.numel(), _stream())
    if rc != 0:
        return rc
    torch.cuda.synchronize()
    return val.cpu().numpy(), ind.cpu().numpy(), tk.cpu().numpy()


# (name, kind, seed, H, W, NMS kernel, min_value): one case per strip height (16 / 8 / 4 / 2 rows), the scalar path
# (W % 4 != 0), several bands per plane, tall planes (more strips per band), plateaus across strip borders, special
# values, NaN in every window offset and a threshold
WIDE_TOPK = [
    ("sr16_bands", "plateau_borders", 41, 16 * 4 * 3 + 5, 96, 5, 0.0),
    ("sr16_peaks", "peaks", 42, 200, 160, 5, 0.0),
    ("sr16_scalar", "plateau_borders", 43, 17, 1021, 5, 0.0),
    ("sr8_bands", "peaks", 44, 8 * 4 * 2 + 3, 1400, 5, 0.0),
    ("sr8_scalar", "plateau_borders", 45, 7, 1025, 3, 0.0),
    ("sr4_bands", "peaks", 46, 4 * 4 * 2 + 1, 1800, 5, 0.0),
    ("sr2_bands", "plateau_borders", 47, 2 * 4 * 2 + 1, 2100, 3, 0.0),
    ("tall", "peaks", 48, 2100, 64, 5, 0.0),
    ("tall_scalar", "plateau_borders", 49, 2100, 30, 5, 0.0),
    ("whole_plateau", "whole_plateau", 50, 64, 160, 5, 0.0),
    ("sparse", "sparse", 51, 48, 64, 5, 0.0),
    ("specials", "specials", 52, 90, 120, 5, 0.0),
    ("specials_k3_scalar", "specials", 53, 66, 81, 3, 0.0),
    ("subnormal_only", "subnormal_only", 54, 60, 80, 3, 0.0),
    ("nan_window_k5", "nan_window", 55, 160, 160, 5, 0.0),
    ("nan_window_k9", "nan_window", 56, 192, 192, 9, 0.0),
    ("peaks_thr01", "peaks", 57, 120, 128, 5, 0.1),
]


@pytest.mark.parametrize("K", [65, 96, 128, 256])
@pytest.mark.parametrize("case", WIDE_TOPK, ids=[c[0] for c in WIDE_TOPK])
def test_nms_topk_wide(case, K):
    name, kind, seed, h, w, kernel, mv = case
    J = 4 if kind == "nan_window" and kernel >= 7 else 2
    det, tag = pc.topk_case(kind, seed, h, w, kernel=kernel, K=K, J=J, min_value=mv)
    got = _topk_device(det, tag, kernel, K, mv)
    assert not isinstance(got, int), (name, _lib.load().lp_last_error())
    ev, ei, et = pc.expected_topk(group_ref, det, tag, kernel, K, mv)
    assert np.array_equal(_bits(got[0]), _bits(ev)), name
    assert np.array_equal(got[1], ei), name
    assert np.array_equal(_bits(got[2]), _bits(et)), name


@pytest.mark.parametrize("kernel,bound", [(5, 8533), (9, 5120)])
def test_nms_topk_wide_width_bound(kernel, bound):
    """the width bound of the strip buffer is the same at K > 64 (the candidate buffers sit beside it)"""
    for w, ok in ((bound, True), (bound + 1, False)):
        det = np.zeros((1, 1, 2, w), np.float32)
        det[0, 0, 1, ::7] = 0.5
        tag = np.zeros((1, 1, 2, w, 1), np.float32)
        got = _topk_device(det, tag, kernel, 128, 0.0)
        if not ok:
            assert got == LP_ERR_BAD_ARG
            continue
        ev, ei, et = pc.expected_topk(group_ref, det, tag, kernel, 128, 0.0)
        assert np.array_equal(_bits(got[0]), _bits(ev)) and np.array_equal(got[1], ei)


def test_nms_topk_wide_ragged_equals_uniform():
    """lp_nms_topk_ragged_f32 at K = 200 over images of different sizes (one with an odd offset) equals the call on
    each image alone"""
    lib = _lib.load()
    K, J, T, kernel = 200, 3, 2, 5
    sizes = [(96, 120), (37, 1021), (200, 64), (8, 1800)]
    dets, tags = [], []
    for i, (h, w) in enumerate(sizes):
        d, t = pc.topk_case("peaks" if i % 2 else "plateau_borders", 80 + i, h, w, kernel=kernel, K=K, J=J)
        dets.append(d[0])
        tags.append(t[0])
    desc = np.zeros(len(sizes), MAP_DESC)
    doff, toff = 1, 0                                              # odd det offset: the scalar staging path
    for i, (h, w) in enumerate(sizes):
        desc[i] = (h, w, doff, toff)
        doff += J * h * w
        toff += J * h * w * T
    det_a = np.zeros(doff, np.float32)
    tag_a = np.zeros(toff, np.float32)
    for i, (h, w) in enumerate(sizes):
        det_a[desc[i]["det_offset"]:desc[i]["det_offset"] + J * h * w] = dets[i].ravel()
        tag_a[desc[i]["tag_offset"]:desc[i]["tag_offset"] + J * h * w * T] = tags[i].ravel()
    hw = np.ascontiguousarray(sizes, np.int32)
    n = len(sizes)
    d, t = torch.from_numpy(det_a).cuda(), torch.from_numpy(tag_a).cuda()
    dd = torch.from_numpy(desc.view(np.uint8)).cuda()
    val = torch.empty((n, J, K), device="cuda")
    ind = torch.empty((n, J, K), dtype=torch.int32, device="cuda")
    tk = torch.empty((n, J, K, T), device="cuda")
    ws = torch.empty(lib.lp_nms_topk_ragged_workspace_bytes(n, hw.ctypes.data, J, K), dtype=torch.uint8, device="cuda")
    _lib.check(lib.lp_nms_topk_ragged_f32(d.data_ptr(), t.data_ptr(), n, hw.ctypes.data, dd.data_ptr(), J, T, kernel, K,
                                          0.0, val.data_ptr(), ind.data_ptr(), tk.data_ptr(), ws.data_ptr(), ws.numel(),
                                          _stream()), "ragged top-K")
    torch.cuda.synchronize()
    for i in range(n):
        u = _topk_device(dets[i][None], tags[i][None], kernel, K, 0.0)
        ev, ei, _ = pc.expected_topk(group_ref, dets[i][None], tags[i][None], kernel, K, 0.0)
        assert np.array_equal(_bits(u[0]), _bits(ev)) and np.array_equal(u[1], ei), i
        assert np.array_equal(_bits(val[i].cpu().numpy()), _bits(u[0][0])), i
        assert np.array_equal(ind[i].cpu().numpy(), u[1][0]), i
        assert np.array_equal(_bits(tk[i].cpu().numpy()), _bits(u[2][0])), i


# ---- tag matching, K > 64
def _match_device(cases, desc=None):
    lib = _lib.load()
    c0 = cases[0]
    n, J, K, T = len(cases), c0["J"], c0["K"], c0["T"]
    pcap = J * K
    val = torch.from_numpy(np.stack([c["val_k"] for c in cases])).cuda()
    ind = torch.from_numpy(np.stack([c["ind_k"] for c in cases])).cuda()
    tag = torch.from_numpy(np.stack([c["tag_k"] for c in cases])).cuda()
    jo = torch.tensor(c0["order"][:J], dtype=torch.int32, device="cuda")
    ans = torch.full((n, pcap, J, 3 + T), float("nan"), device="cuda")
    num = torch.zeros(n, dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.lp_tag_match_workspace_bytes(n, J, K, T, pcap), dtype=torch.uint8, device="cuda")
    args = (c0["det_thr"], c0["tag_thr"], int(c0["use_det_val"]), int(c0["ignore"]), K, pcap, ans.data_ptr(),
            num.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
    if desc is None:
        desc = np.zeros(n, MAP_DESC)
        desc["h"], desc["w"] = c0["H"], c0["W"]
    d = torch.from_numpy(desc.view(np.uint8)).cuda()
    rc = lib.lp_tag_match_ragged_f32(val.data_ptr(), ind.data_ptr(), tag.data_ptr(), n, J, K, T, d.data_ptr(),
                                     jo.data_ptr(), *args)
    _lib.check(rc, "tag match")
    torch.cuda.synchronize()
    num_h, ans_h = num.cpu().numpy(), ans.cpu().numpy()
    return [ans_h[i, :num_h[i]] for i in range(n)]


def _match_oracle(c, W=None):
    loc = pc.loc_from_ind(c["ind_k"], c["W"] if W is None else W)
    ans = group_ref.match_by_tag((c["tag_k"], loc, c["val_k"]), pc.params_of(c))
    return np.asarray(ans, np.float32).reshape(-1, c["J"], 3 + c["T"])


# the edge families of oracle/parser_cases.py scaled past 64 candidates / persons: lattice crowds (multi-prime
# augmenting paths, zeros found after the wrap), half-integer distances (.5 rounding ties), distances equal to
# TAG_THRESHOLD, key collisions including +-0.0, raw distances as costs (step 6 with non-integer costs), more persons
# than candidates and the reverse (pad rows / pad columns), IGNORE_TOO_MUCH, T = 1 and 4
WIDE_MATCH = [
    ("lattice", 1, dict(persons=90, clutter=20, spread=12)),
    ("lattice_quarter", 2, dict(persons=60, clutter=30, step=0.25, spread=10)),
    ("lattice_coco", 3, dict(joints="coco", persons=80, clutter=20, spread=10)),
    ("half_dist_t1", 7, dict(T=1, offsets=[(0.5,), (1.5,), (-2.5,), (0.0,)], persons=70, spread=40)),
    ("half_dist_t2", 8, dict(offsets=pc.AXIS_HALF, persons=70, spread=12, step=1.0)),
    ("at_threshold", 11, dict(offsets=pc.AXIS_ONE, persons=70, spread=12, step=1.0)),
    ("keys_signed_zero", 14, dict(keys=[pc.NEG0, 0.0, 1.0, 2.0], persons=70, clutter=10)),
    ("keys_dense", 15, dict(keys=[pc.NEG0, 0.0, 0.5], persons=80, clutter=20)),
    ("crowd_ignore", 18, dict(persons=120, clutter=30, ignore=True, spread=20)),
    ("raw_costs", 22, dict(use_det_val=False, noise=0.3, persons=80, clutter=20, spread=12)),
    ("sparse_pad_rows", 30, dict(persons=80, clutter=0, presence=0.3, spread=12)),
    ("t4_lattice", 26, dict(T=4, persons=70, clutter=10)),
]


@pytest.mark.parametrize("K", [65, 128, 256])
@pytest.mark.parametrize("case", WIDE_MATCH, ids=[c[0] for c in WIDE_MATCH])
def test_tag_match_wide_edges(case, K):
    name, seed, kw = case
    c = pc.matcher_case(seed, K=K, **kw)
    got = _match_device([c])[0]
    exp = _match_oracle(c)
    assert got.shape == exp.shape, (name, got.shape, exp.shape)
    assert np.array_equal(_bits(got), _bits(exp)), name


def test_tag_match_wide_ragged_widths():
    """one ragged call at K = 128 over images of different map widths"""
    widths = [40, 97, 640, 33]
    cases = [pc.matcher_case(160 + i, K=128, persons=70, clutter=10, spread=12, W=w, H=50) for i, w in enumerate(widths)]
    desc = np.zeros(len(cases), MAP_DESC)
    desc["h"], desc["w"] = 50, widths
    got = _match_device(cases, desc)
    for c, w, g in zip(cases, widths, got):
        exp = _match_oracle(c, w)
        assert g.shape == exp.shape and np.array_equal(_bits(g), _bits(exp)), w


@pytest.mark.parametrize("case", CROWD_CASES, ids=[c[0] for c in CROWD_CASES])
def test_parser_crowd_golden(golden_dir, case):
    """the reference's HeatmapParser.parse on planted crowds of 80 / 150 / 240 persons, through the drop-in parser"""
    from litepose_b200.lib.core.group import HeatmapParser
    z = np.load(os.path.join(golden_dir, "parser_crowd_%s.npz" % case[0]))
    cfg, (det, tag) = crowd_inputs(case)
    assert digest(det, tag) == str(z["in_digest"])
    p = HeatmapParser(cfg)
    dd, td = torch.from_numpy(det)[None].cuda(), torch.from_numpy(tag)[None].cuda()
    assert_topk_equal(p.top_k(dd, td), {k: z[k] for k in ("val_k", "loc_k", "tag_k")}, case[0])
    ans, scores = p.parse(dd, td, True, True)
    a = np.asarray(ans[0], np.float32).reshape(z["ans"].shape[0], -1, z["ans"].shape[2]) if len(ans[0]) else \
        np.zeros((0,) + z["ans"].shape[1:], np.float32)
    assert a.shape == z["ans"].shape and z["ans"].shape[0] > 64, (a.shape, z["ans"].shape)
    assert np.array_equal(_bits(a), _bits(z["ans"]))
    assert np.array_equal(_bits(np.asarray(scores, np.float32)), _bits(z["scores"]))


# ---- adjust + refine at pcap = J * 256
def test_adjust_refine_full_capacity():
    lib = _lib.load()
    c = pc.refine_case("many_missing", 39, T=2)
    det, tag, base = c["det"], c["tag"], c["ans"]
    J = det.shape[0]
    P = J * 256
    rs = np.random.RandomState(5)
    ans0 = base[rs.randint(base.shape[0], size=P)].copy()
    ans0[rs.rand(P, J) < 0.3] = 0.0                                 # drop joints: refine fills them
    ans0[np.all(ans0[:, :, 2] == 0, axis=1), 0, :] = base[0, 0]     # every person keeps one detected joint
    T = c["T"]
    d = torch.from_numpy(det)[None].cuda()
    t = torch.from_numpy(tag)[None].cuda()
    ans = torch.from_numpy(ans0)[None].cuda().contiguous()
    num = torch.tensor([P], dtype=torch.int32, device="cuda")
    scores = torch.empty((1, P), device="cuda")
    ws = torch.empty(lib.lp_adjust_refine_workspace_bytes(1, J, P), dtype=torch.uint8, device="cuda")
    _lib.check(lib.lp_adjust_refine_f32(d.data_ptr(), t.data_ptr(), 1, J, det.shape[1], det.shape[2], T, P,
                                        ans.data_ptr(), num.data_ptr(), scores.data_ptr(), 1, 1, ws.data_ptr(),
                                        ws.numel(), _stream()), "adjust/refine")
    torch.cuda.synchronize()
    exp_ans, exp_scores = run_adjust_refine(group_ref.adjust, group_ref.refine, dict(c, ans=ans0), True, True)
    assert np.array_equal(_bits(ans[0].cpu().numpy()), _bits(exp_ans))
    assert np.array_equal(_bits(scores[0].cpu().numpy()), _bits(exp_scores))


# ---- the pipeline entry points at K = 128
def _model(cfg, name="XS"):
    from litepose_b200.lib.models.pose_mobilenet import get_pose_net
    torch.manual_seed(0)
    return synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch(name)), 1)).eval().cuda()


def _check_step(cfg, got, det_g, tag_g, final=None):
    op = group_ref.HeatmapParser(cfg)
    J = cfg.DATASET.NUM_JOINTS
    found = []
    for i in range(det_g.shape[0]):
        ans, scores = op.parse(det_g[i:i + 1].copy(), tag_g[i:i + 1].copy(), True, True)
        if final is None:
            e = np.asarray(ans[0], np.float32).reshape(-1, J, 3 + tag_g.shape[-1])
        else:
            e = np.stack(final(ans)).astype(np.float32)
        assert got[i][2] == e.shape[0], (i, got[i][2], e.shape)
        assert np.array_equal(_bits(got[i][0]), _bits(e)), i
        assert np.array_equal(_bits(np.asarray(got[i][1], np.float32)), _bits(np.asarray(scores, np.float32))), i
        found.append(e.shape[0])
    return found


def test_pipeline_step_k128_flip():
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    n, size = 2, 256
    cfg = get_cfg(input_size=size)
    cfg.DATASET.MAX_NUM_PEOPLE = 128
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, keep=128)
    plant = PlantedCrowd(n, 14, size, size, 2, num_people=100, seed=31, device="cuda")
    frames = synth.make_frames(n, size, seed=5)
    got = pipe.step(frames.half().pin_memory(), plant)
    st = pipe._get_state(n, size, size, torch.float16, plant)
    found = _check_step(cfg, got, st["det"].cpu().numpy(), st["tag"].cpu().numpy())
    assert max(found) > 64, found


def test_pipeline_step_multiscale_k128():
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    n, size, scales = 2, 128, [0.5, 1, 2]
    cfg = get_cfg(input_size=size)
    cfg.TEST.SCALE_FACTOR = scales
    cfg.DATASET.MAX_NUM_PEOPLE = 128
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, keep=128)
    frames = {float(s): synth.make_frames(n, int(size * s), seed=40 + i).half().pin_memory()
              for i, s in enumerate(scales)}
    plant = PlantedCrowd(n, 14, size, size, 2, num_people=80, seed=9, device="cuda")
    got = pipe.step_multiscale(frames, plant)
    st = pipe._get_state(n, size, size, torch.float16, plant, det_hw=(size, size))
    found = _check_step(cfg, got, st["det"].cpu().numpy(), st["tag"].cpu().numpy())
    assert max(found) > 64, found


def test_infer_images_mixed_list_k128_final_preds():
    """a mixed-size list through infer_images (keypoints mapped back by get_final_preds on the device): per image equal
    to the oracle parser on the maps of that image's own call, mapped back with the host get_final_preds, and to the
    one-image call"""
    from litepose_b200.lib.utils import transforms as T
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    size = 128
    cfg = get_cfg(input_size=size)
    cfg.DATASET.MAX_NUM_PEOPLE = 128
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, keep=128)
    rs = np.random.RandomState(3)
    shapes = [(150, 200), (200, 150), (128, 128)]
    imgs = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    plants, exp = [], []
    for i, im in enumerate(imgs):
        (bw, bh), center, scale = T.get_multi_scale_size(im, size, 1.0, 1.0)
        plants.append(PlantedCrowd(1, 14, bh, bw, 2, num_people=90, seed=60 + i, device="cuda"))
        one = pipe.infer_images(torch.from_numpy(im)[None].pin_memory(), plant=plants[i])[0]
        st = pipe._last_state
        det_g, tag_g = st["det"].cpu().numpy(), st["tag"].cpu().numpy()
        _check_step(cfg, [one], det_g, tag_g, final=lambda a: T.get_final_preds(a, center, scale, [bw, bh]))
        exp.append(one)
    got = pipe.infer_images([torch.from_numpy(im) for im in imgs], plant=plants)
    assert max(e[2] for e in exp) > 64, [e[2] for e in exp]
    for i in range(len(imgs)):
        assert got[i][2] == exp[i][2], i
        assert np.array_equal(_bits(got[i][0]), _bits(exp[i][0])), i
        assert np.array_equal(_bits(np.asarray(got[i][1], np.float32)), _bits(np.asarray(exp[i][1], np.float32))), i


# ---- memory footprint of the new shapes
def _footprint_chain(A, det, tag, K, desc, hw):
    """top-K then tag matching (ragged entry points) on the buffers of A (Guarded or Plain) -> list of return codes"""
    lib = _lib.load()
    n, J, T = len(hw), 14, 2
    pcap = J * K
    d, t = A.inp("det", det.ravel()), A.inp("tag", tag.ravel())
    val = A.out("val_k", (n, J, K), np.float32)
    ind = A.out("ind_k", (n, J, K), np.int32)
    tk = A.out("tag_k", (n, J, K, T), np.float32)
    ans = A.out("ans", (n, pcap, J, 3 + T), np.float32)
    num = A.out("num", (n,), np.int32)
    jo = A.inp("jo", np.arange(J, dtype=np.int32))
    dd = A.desc("desc", desc)
    ws = A.ws("ws_topk", lib.lp_nms_topk_ragged_workspace_bytes(n, hw.ctypes.data, J, K))
    rcs = [lib.lp_nms_topk_ragged_f32(d.data_ptr(), t.data_ptr(), n, hw.ctypes.data, dd.data_ptr(), J, T, 5, K, 0.1,
                                      val.data_ptr(), ind.data_ptr(), tk.data_ptr(), ws.data_ptr(), ws.numel(),
                                      _stream())]
    wm = A.ws("ws_match", lib.lp_tag_match_workspace_bytes(n, J, K, T, pcap))
    rcs.append(lib.lp_tag_match_ragged_f32(val.data_ptr(), ind.data_ptr(), tk.data_ptr(), n, J, K, T, dd.data_ptr(),
                                           jo.data_ptr(), 0.1, 1.0, 1, 0, K, pcap, ans.data_ptr(), num.data_ptr(),
                                           wm.data_ptr(), wm.numel(), _stream()))
    return rcs


@pytest.mark.parametrize("mixed", [False, True])
def test_footprint_wide_parser(mixed):
    """K = 128: every byte the wide top-K and the CTA matcher write lies inside their outputs and workspaces; inputs
    and guard bands stay as they were; outputs equal an unguarded run.  Equal map sizes (a uniform batch) and mixed."""
    K, J, T = 128, 14, 2
    if mixed:
        hw = np.array([[96, 100], [64, 130]], np.int32)
        dets, tags = synth.plant_crowd_batch(1, J, 96, 100, T, num_people=80, seed=3)
        d2, t2 = synth.plant_crowd_batch(1, J, 64, 130, T, num_people=70, seed=4)
        det = np.concatenate([dets.ravel(), d2.ravel()])
        tag = np.concatenate([tags.ravel(), t2.ravel()])
        desc = np.zeros(2, MAP_DESC)
        desc[0] = (96, 100, 0, 0)
        desc[1] = (64, 130, dets.size, tags.size)
    else:
        det, tag = synth.plant_crowd_batch(2, J, 96, 128, T, num_people=90, seed=5)
        desc, hw = _equal_desc(2, J, 96, 128, T)
    P = Plain()
    assert _footprint_chain(P, det, tag, K, desc, hw) == [0, 0]
    want = P.outputs()
    G = Guarded()
    assert _footprint_chain(G, det, tag, K, desc, hw) == [0, 0]
    assert want["num"].max() > 64, want["num"]
    errs = G.verify(want, untouched=("ans",))
    assert not errs, errs
