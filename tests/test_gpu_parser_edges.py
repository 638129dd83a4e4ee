"""-m gpu: the three parser stages called through their C entry points on the edge cases of oracle/parser_cases.py,
bit for bit against the oracle (compared as uint32, so NaN and -0.0 count): tag matching through both matcher
kernels and the ragged entry, NMS + top-K at every strip geometry with NaN / inf / subnormal pixels and the width
bound, adjust + refine for every flag combination; and the pipeline on frames whose det maps are wider than 2:1."""
import os

import numpy as np
import pytest
import torch

from litepose_b200 import _lib, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.mixed import MAP_DESC
from oracle import group_ref
from oracle import parser_cases as pc
from oracle.make_golden_parser_edges import ADJ_REF, run_adjust_refine

pytestmark = pytest.mark.gpu

LP_ERR_BAD_ARG = 1


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def matcher_cases():
    return dict(pc.matcher_cases())


@pytest.fixture
def wide_matcher():
    """routes every lp_tag_match_* call through the two-columns-per-lane kernel (read per call by the library)"""
    os.environ["LP_MATCH_WIDE"] = "1"
    yield
    os.environ.pop("LP_MATCH_WIDE", None)


def _match_device(cases, desc=None):
    """lp_tag_match_f32 (one width) or lp_tag_match_ragged_f32 (desc: per-image widths) on a batch of matcher cases
    that share J, K, T and the thresholds -> list of ans [P,J,3+T]."""
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
        rc = lib.lp_tag_match_f32(val.data_ptr(), ind.data_ptr(), tag.data_ptr(), n, J, K, T, c0["W"], jo.data_ptr(),
                                  *args)
    else:
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


def _check_match(name, c):
    got = _match_device([c])[0]
    exp = _match_oracle(c)
    assert got.shape == exp.shape, (name, got.shape, exp.shape)
    assert np.array_equal(_bits(got), _bits(exp)), name


@pytest.mark.parametrize("name", pc.MATCHER_NAMES)
def test_tag_match_edges(matcher_cases, name):
    _check_match(name, matcher_cases[name])


@pytest.mark.parametrize("name", [n for n, c in pc.matcher_cases() if c["K"] <= 32])
def test_tag_match_edges_wide_kernel(matcher_cases, name, wide_matcher):
    """K <= 32: the same cases through the 64-wide kernel"""
    _check_match(name, matcher_cases[name])


def test_tag_match_ragged_widths():
    """one ragged call over images of different map widths: ind -> (x, y) uses each image's desc[n].w"""
    widths = [40, 97, 640, 33, 1152]
    cases = [pc.matcher_case(60 + i, persons=6, clutter=3, W=w, H=50) for i, w in enumerate(widths)]
    desc = np.zeros(len(cases), MAP_DESC)
    desc["h"], desc["w"] = 50, widths
    got = _match_device(cases, desc)
    for c, w, g in zip(cases, widths, got):
        exp = _match_oracle(c, w)
        assert g.shape == exp.shape and np.array_equal(_bits(g), _bits(exp)), w


# ---- NMS + top-K
def _topk_device(det, tag, kernel, K, min_value):
    lib = _lib.load()
    n, J, H, W = det.shape
    T = tag.shape[-1]
    d, t = torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda()
    val = torch.empty((n, J, K), device="cuda")
    ind = torch.empty((n, J, K), dtype=torch.int32, device="cuda")
    tk = torch.empty((n, J, K, T), device="cuda")
    ws = torch.empty(lib.lp_nms_topk_workspace_bytes(n, J, H, W, K), dtype=torch.uint8, device="cuda")
    rc = lib.lp_nms_topk_f32(d.data_ptr(), t.data_ptr(), n, J, H, W, T, kernel, K, float(min_value), val.data_ptr(),
                             ind.data_ptr(), tk.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
    if rc != 0:
        return rc
    torch.cuda.synchronize()
    return val.cpu().numpy(), ind.cpu().numpy(), tk.cpu().numpy()


def _check_topk(name, det, tag, kernel, K, mv):
    got = _topk_device(det, tag, kernel, K, mv)
    assert not isinstance(got, int), (name, _lib.load().lp_last_error())
    ev, ei, et = pc.expected_topk(group_ref, det, tag, kernel, K, mv)
    assert np.array_equal(_bits(got[0]), _bits(ev)), name
    assert np.array_equal(got[1], ei), name
    assert np.array_equal(_bits(got[2]), _bits(et)), name


@pytest.mark.parametrize("name", [c[0] for c in pc.TOPK_CASES])
def test_nms_topk_edges(name):
    (_, det, tag, kernel, K, mv), = [c for c in pc.topk_cases() if c[0] == name]
    _check_topk(name, det, tag, kernel, K, mv)


def test_nms_topk_ragged_odd_offset_equals_uniform():
    """the ragged entry on an arena whose first map starts one float in (16-byte loads impossible: scalar path)
    equals the uniform call on every image"""
    lib = _lib.load()
    sel = ["k5", "sr16_h17_scalar", "sr8_h9", "specials", "nan_window_k5"]
    cases = [c for c in pc.topk_cases() if c[0] in sel]
    J, T, K, kernel, mv = 2, 2, 64, 5, 0.1
    n = len(cases)
    desc = np.zeros(n, MAP_DESC)
    hw = np.zeros((n, 2), np.int32)
    dparts, tparts = [np.zeros(1, np.float32)], [np.zeros(3, np.float32)]
    d0, t0 = 1, 3
    for i, (_, det, tag, _, _, _) in enumerate(cases):
        h, w = det.shape[2:]
        desc[i] = (h, w, d0, t0)
        hw[i] = (h, w)
        dparts.append(det.ravel())
        tparts.append(tag.ravel())
        d0 += det.size
        t0 += tag.size
    darena = torch.from_numpy(np.concatenate(dparts)).cuda()
    tarena = torch.from_numpy(np.concatenate(tparts)).cuda()
    dd = torch.from_numpy(desc.view(np.uint8)).cuda()
    val = torch.empty((n, J, K), device="cuda")
    ind = torch.empty((n, J, K), dtype=torch.int32, device="cuda")
    tk = torch.empty((n, J, K, T), device="cuda")
    ws = torch.empty(lib.lp_nms_topk_ragged_workspace_bytes(n, hw.ctypes.data, J, K), dtype=torch.uint8, device="cuda")
    _lib.check(lib.lp_nms_topk_ragged_f32(darena.data_ptr(), tarena.data_ptr(), n, hw.ctypes.data, dd.data_ptr(), J, T,
                                          kernel, K, mv, val.data_ptr(), ind.data_ptr(), tk.data_ptr(), ws.data_ptr(),
                                          ws.numel(), _stream()), "ragged top-K")
    torch.cuda.synchronize()
    for i, (name, det, tag, _, _, _) in enumerate(cases):
        uv, ui, ut = _topk_device(det, tag, kernel, K, mv)
        assert np.array_equal(_bits(val[i].cpu().numpy()), _bits(uv[0])), name
        assert np.array_equal(ind[i].cpu().numpy(), ui[0]), name
        assert np.array_equal(_bits(tk[i].cpu().numpy()), _bits(ut[0])), name
        ev, ei, _ = pc.expected_topk(group_ref, det, tag, kernel, K, mv)
        assert np.array_equal(_bits(uv), _bits(ev)) and np.array_equal(ui, ei), name


@pytest.mark.parametrize("kernel,bound", [(5, 8533), (9, 5120)])
def test_nms_topk_width_bound(kernel, bound):
    """W <= 51200 / (NMS_KERNEL + 1) (include/litepose_b200.h): the widest map runs and is exact, one column more is
    refused with LP_ERR_BAD_ARG"""
    det, tag = pc.topk_case("peaks", 70 + kernel, 2, bound, kernel=kernel, K=40)
    _check_topk("W=%d" % bound, det, tag, kernel, 40, 0.0)
    det, tag = pc.topk_case("peaks", 70 + kernel, 2, bound + 1, kernel=kernel, K=40)
    assert _topk_device(det, tag, kernel, 40, 0.0) == LP_ERR_BAD_ARG
    assert b"too wide" in _lib.load().lp_last_error()


# ---- adjust + refine
def _adjust_refine_device(c, do_adjust, do_refine, T=None):
    lib = _lib.load()
    det, tag, ans0 = c["det"], c["tag"], c["ans"]
    J, H, W = det.shape
    T = c["T"] if T is None else T
    P = ans0.shape[0]
    d = torch.from_numpy(det)[None].cuda()
    t = torch.from_numpy(tag)[None].cuda()
    ans = torch.from_numpy(ans0)[None].cuda().contiguous()
    num = torch.tensor([P], dtype=torch.int32, device="cuda")
    scores = torch.empty((1, P), device="cuda")
    ws = torch.empty(lib.lp_adjust_refine_workspace_bytes(1, J, P), dtype=torch.uint8, device="cuda")
    rc = lib.lp_adjust_refine_f32(d.data_ptr(), t.data_ptr(), 1, J, H, W, T, P, ans.data_ptr(), num.data_ptr(),
                                  scores.data_ptr(), do_adjust, do_refine, ws.data_ptr(), ws.numel(), _stream())
    if rc != 0:
        return rc
    torch.cuda.synchronize()
    return ans[0].cpu().numpy(), scores[0].cpu().numpy()


@pytest.mark.parametrize("name", [c[0] for c in pc.REFINE_CASES])
def test_adjust_refine_edges(name):
    c = dict(pc.refine_cases())[name]
    for a, r in ADJ_REF:
        got_ans, got_scores = _adjust_refine_device(c, a, r)
        exp_ans, exp_scores = run_adjust_refine(group_ref.adjust, group_ref.refine, c, a, r)
        assert np.array_equal(_bits(got_ans), _bits(exp_ans)), (name, a, r)
        assert np.array_equal(_bits(got_scores), _bits(exp_scores)), (name, a, r)


def test_adjust_refine_rejects_t5():
    c = pc.refine_case("random", 50, T=4)
    c = dict(c, tag=np.concatenate((c["tag"], c["tag"][..., :1]), axis=-1),
             ans=np.concatenate((c["ans"], c["ans"][..., :1]), axis=-1))
    assert _adjust_refine_device(c, 1, 1, T=5) == LP_ERR_BAD_ARG


# ---- wide frames
@pytest.mark.parametrize("h,w", [(640, 896), (640, 1152), (448, 1408)])
def test_parser_wide_det_maps_vs_oracle(h, w):
    """the det maps of a 640x480 and a 1920x1080 frame at input 640 and of a 640x213 frame at 448 (PROJECT2IMAGE):
    more than 256 per-warp lists under 8-byte strip sizing; the parse is exact against the oracle"""
    from litepose_b200.lib.core.group import HeatmapParser
    cfg = get_cfg(input_size=640)
    det, tag = synth.plant_crowd_batch(1, 14, h, w, 2, num_people=8, seed=h + w)
    got = HeatmapParser(cfg).parse_batch(torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda(), True, True)
    exp = group_ref.HeatmapParser(cfg).parse_batch(det.copy(), tag.copy(), True, True)
    a = np.asarray(got[0][0][0], np.float32).reshape(-1, 14, 5)
    e = np.asarray(exp[0][0][0], np.float32).reshape(-1, 14, 5)
    assert a.shape == e.shape and e.shape[0] > 0 and np.array_equal(a, e)
    assert np.array_equal(np.asarray(got[0][1], np.float32), np.asarray(exp[0][1], np.float32))


@pytest.mark.parametrize("frame_hw", [(480, 640), (1080, 1920)])
def test_infer_images_wide_frames(frame_hw):
    """LitePose-XS at input 640 on an ordinary 4:3 frame and on a 1080p frame returns a result"""
    from litepose_b200.lib.models.pose_mobilenet import get_pose_net
    from litepose_b200.pipeline import LitePosePipeline
    cfg = get_cfg(input_size=640)
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch("XS")), 1)).eval()
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=False)
    img = np.random.RandomState(1).randint(0, 256, (1,) + frame_hw + (3,)).astype(np.uint8)
    res = pipe.infer_images(torch.from_numpy(img))
    torch.cuda.synchronize()
    assert len(res) == 1
    final, scores, p = res[0]
    assert final.shape[0] == p and len(scores) == p
