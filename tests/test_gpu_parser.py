"""-m gpu: device parser (NMS/top-K, tag match, adjust, refine) bit-exact against the
oracle and the committed golden vectors from the unmodified reference; fused glue
within the stated fp tolerance."""
import hashlib
import os

import numpy as np
import pytest

from parity_util import assert_topk_equal
import torch

from litepose_b200 import _lib, synth
from litepose_b200.config import flip_index_for, get_cfg
from oracle import glue_ref, group_ref
from oracle.make_golden import PARSER_CASES

pytestmark = pytest.mark.gpu


def _parser(cfg):
    from litepose_b200.lib.core.group import HeatmapParser
    return HeatmapParser(cfg)


@pytest.mark.parametrize("case", PARSER_CASES, ids=[c[0] for c in PARSER_CASES])
def test_parser_golden(golden_dir, case):
    name, ds, h, w, t, people, seed = case
    z = np.load(os.path.join(golden_dir, "parser_%s.npz" % name))
    cfg = get_cfg(dataset=ds, input_size=256)
    nj = cfg.DATASET.NUM_JOINTS
    det, tag = synth.plant_crowd(nj, h, w, t, num_people=people, seed=seed)
    assert hashlib.sha256(det.tobytes() + tag.tobytes()).hexdigest() == str(z["in_digest"])
    p = _parser(cfg)
    dd, td = torch.from_numpy(det)[None].cuda(), torch.from_numpy(tag)[None].cuda()
    top = p.top_k(dd, td)
    assert_topk_equal(top, {k: z[k] for k in ("val_k", "loc_k", "tag_k")}, name)
    for adj, ref in ((True, True), (True, False), (False, False)):
        ans, scores = p.parse(dd, td, adj, ref)
        a = np.asarray(ans[0], dtype=np.float32).reshape(-1, nj, 3 + t)
        exp = z["ans_a%d_r%d" % (adj, ref)]
        assert a.shape == exp.shape, (adj, ref, a.shape, exp.shape)
        assert np.array_equal(a, exp), (adj, ref, np.abs(a - exp).max())
        assert np.array_equal(np.asarray(scores, np.float32), z["scores_a%d_r%d" % (adj, ref)])


# the config knobs HeatmapParser hands to the kernels, each away from its shipped value
KNOBS = {
    "nodetval": {"USE_DETECTION_VAL": False},
    "ignore": {"IGNORE_TOO_MUCH": True, "MAX_NUM_PEOPLE": 8},
    "nms3": {"NMS_KERNEL": 3, "NMS_PADDING": 1},
    "nms7": {"NMS_KERNEL": 7, "NMS_PADDING": 3},
    "tagthr05": {"TAG_THRESHOLD": 0.5},
    "detthr02": {"DETECTION_THRESHOLD": 0.2},
}
BATCH_CASES = [pytest.param(64, 64, 2, 4, None, id="64-64-2-4"), pytest.param(96, 160, 1, 9, None, id="96-160-1-9"),
               pytest.param(200, 120, 2, 20, None, id="200-120-2-20")]
BATCH_CASES += [pytest.param(h, w, t, p, k, id="%d-%d-%d-%d-%s" % (h, w, t, p, k))
                for k in KNOBS for h, w, t, p in [(96, 160, 1, 9), (200, 120, 2, 20)]]


@pytest.mark.parametrize("h,w,t,people,knob", BATCH_CASES)
def test_parser_batch_vs_oracle(h, w, t, people, knob):
    cfg = get_cfg(input_size=256)
    for key, v in KNOBS.get(knob, {}).items():
        setattr(cfg.DATASET if key == "MAX_NUM_PEOPLE" else cfg.TEST, key, v)
    n = 5
    det, tag = synth.plant_crowd_batch(n, 14, h, w, t, num_people=people, seed=100)
    det[3] = np.random.RandomState(1).uniform(0, 0.02, det[3].shape).astype(np.float32)   # an image with nobody
    p = _parser(cfg)
    got = p.parse_batch(torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda(), True, True)
    op = group_ref.HeatmapParser(cfg)
    exp = op.parse_batch(det.copy(), tag.copy(), True, True)
    for i in range(n):
        a = np.asarray(got[i][0][0], np.float32).reshape(-1, 14, 3 + t)
        e = np.asarray(exp[i][0][0], np.float32).reshape(-1, 14, 3 + t)
        assert a.shape == e.shape, (i, a.shape, e.shape)
        assert np.array_equal(a, e), i
        assert np.array_equal(np.asarray(got[i][1], np.float32), np.asarray(exp[i][1], np.float32))


def test_topk_plateau_and_empty():
    """plateaus keep every equal maximum (canonical index order); all-zero planes give empty slots."""
    cfg = get_cfg(input_size=256)
    det = np.zeros((1, 14, 48, 40), np.float32)
    det[0, 0, 10:14, 10:14] = 0.5            # 4x4 plateau: all 16 survive
    det[0, 1, 5, 7] = 0.9
    det[0, 1, 5, 8] = 0.9                    # tie inside one window: both survive, index order
    tag = np.random.RandomState(0).randn(1, 14, 48, 40, 2).astype(np.float32)
    p = _parser(cfg)
    top = p.top_k(torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda())
    exp = group_ref.HeatmapParser(cfg).top_k(det, tag)
    for k in ("val_k", "loc_k", "tag_k"):
        assert np.array_equal(top[k], exp[k]), k
    assert (top["val_k"][0, 0, :16] == 0.5).all() and top["val_k"][0, 0, 16] == 0
    assert (top["val_k"][0, 2:] == 0).all()


def test_detection_threshold_prefilter_is_exact():
    """parse() hands DETECTION_THRESHOLD to the NMS/top-K kernel (match_by_tag drops val <= threshold first,
    reference group.py:43-45).  The compare must be the reference's: float32 value widened to double against the
    Python float - peaks sitting exactly on float32(0.1) (> 0.1 in double) and one ulp below it pin the edge."""
    cfg = get_cfg(input_size=256)
    thr = cfg.TEST.DETECTION_THRESHOLD
    f = np.float32(thr)
    assert float(f) > thr                                  # float32(0.1) lies above the double 0.1
    below = np.nextafter(f, np.float32(0))
    rs = np.random.RandomState(3)
    det = (rs.rand(2, 14, 40, 48) * 0.05).astype(np.float32)
    tag = rs.randn(2, 14, 40, 48, 2).astype(np.float32)
    for n in range(2):
        for j in range(14):
            det[n, j, 8, 9] = f                            # kept by the reference (0.10000000149 > 0.1)
            det[n, j, 20, 30] = below                      # dropped
            det[n, j, 30, 12] = np.float32(0.6)
            tag[n, j, 8, 9] = 1.0
            tag[n, j, 30, 12] = 5.0
    p = _parser(cfg)
    dd, td = torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda()
    got = p.parse_batch(dd, td, True, True)
    exp = group_ref.HeatmapParser(cfg).parse_batch(det.copy(), tag.copy(), True, True)
    for g, e in zip(got, exp):
        a = np.asarray(g[0][0], np.float32).reshape(-1, 14, 5)
        b = np.asarray(e[0][0], np.float32).reshape(-1, 14, 5)
        assert a.shape == b.shape and np.array_equal(a, b)
        assert (b[:, :, 2] == f).any() and not (b[:, :, 2] == below).any()
    val_k, ind_k, _ = p.device_parser.top_k_device(dd, td, thr)
    v = val_k.cpu().numpy()
    assert ((v > 0).sum(axis=2) == 2).all() and (v[:, :, 1] == f).all()


@pytest.mark.parametrize("flip,proj", [(1, 1), (0, 1), (1, 0)])
def test_glue_golden(golden_dir, flip, proj):
    lib = _lib.load()
    z = np.load(os.path.join(golden_dir, "glue_flip%d_proj%d.npz" % (flip, proj)))
    cfg = get_cfg(input_size=64, flip_test=bool(flip), project2image=bool(proj))
    a0, a1, b0, b1 = [torch.from_numpy(z[k]).cuda() for k in ("a0", "a1", "b0", "b1")]
    n, j2, h, w = a0.shape
    J = j2 // 2
    T = 2 if flip else 1
    Hd, Wd = (64, 64) if proj else (2 * h, 2 * w)
    det = torch.full((n, J, Hd, Wd), float("nan"), device="cuda")
    tag = torch.full((n, J, Hd, Wd, T), float("nan"), device="cuda")
    fidx = torch.tensor(flip_index_for(cfg), dtype=torch.int32, device="cuda")
    _lib.check(lib.lp_glue_f32(a0.data_ptr(), a1.data_ptr(), b0.data_ptr() if flip else None,
                               b1.data_ptr() if flip else None, fidx.data_ptr(), n, J, h, w, flip, Hd, Wd,
                               det.data_ptr(), tag.data_ptr(), torch.cuda.current_stream().cuda_stream), "glue")
    torch.cuda.synchronize()
    ed, et = z["final_heatmaps"], z["tags"]
    assert np.abs(det.cpu().numpy() - ed).max() <= 2e-3 * np.abs(ed).max() * 1e-2 + 1e-5
    assert np.abs(tag.cpu().numpy() - et).max() <= 2e-3 * np.abs(et).max() * 1e-2 + 1e-5


def test_glue_nonsquare_projection():
    lib = _lib.load()
    cfg = get_cfg(input_size=64, flip_test=True, project2image=True)
    g = torch.Generator().manual_seed(3)
    n, J, h, w = 2, 14, 16, 24
    a0, b0 = torch.randn(n, 2 * J, h, w, generator=g), torch.randn(n, 2 * J, h, w, generator=g)
    a1, b1 = torch.randn(n, J, 2 * h, 2 * w, generator=g), torch.randn(n, J, 2 * h, 2 * w, generator=g)
    Hd, Wd = 61, 93
    calls = []

    def fake(img):
        calls.append(1)
        return [a0, a1] if len(calls) == 1 else [b0, b1]

    _, hm, tg = glue_ref.multi_stage_outputs(cfg, fake, torch.zeros(n, 3, 64, 96), True, True, (Wd, Hd))
    ed, et = glue_ref.aggregate(cfg, hm, tg)
    det = torch.empty((n, J, Hd, Wd), device="cuda")
    tag = torch.empty((n, J, Hd, Wd, 2), device="cuda")
    fidx = torch.tensor(flip_index_for(cfg), dtype=torch.int32, device="cuda")
    args = [t.cuda() for t in (a0, a1, b0, b1)]
    _lib.check(lib.lp_glue_f32(args[0].data_ptr(), args[1].data_ptr(), args[2].data_ptr(), args[3].data_ptr(),
                               fidx.data_ptr(), n, J, h, w, 1, Hd, Wd, det.data_ptr(), tag.data_ptr(),
                               torch.cuda.current_stream().cuda_stream), "glue")
    torch.cuda.synchronize()
    assert (det.cpu() - ed).abs().max().item() <= 1e-5 * max(1.0, ed.abs().max().item())
    assert (tag.cpu() - et).abs().max().item() <= 1e-5 * max(1.0, et.abs().max().item())


def test_topk_dense_fallback():
    """a whole-plane plateau (every pixel survives the NMS, the K slots are the first K indices) and a plateau over
    most of a plane broken by one higher peak"""
    cfg = get_cfg(input_size=256)
    rng = np.random.RandomState(4)
    det = rng.uniform(0, 0.02, (1, 14, 64, 160)).astype(np.float32)
    det[0, 0] = 0.3                               # whole plane is one plateau: every pixel survives
    det[0, 1, :40, :] = 0.25
    det[0, 1, 7, 9] = 0.9
    tag = rng.randn(1, 14, 64, 160, 1).astype(np.float32)
    p = _parser(cfg)
    top = p.top_k(torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda())
    exp = group_ref.HeatmapParser(cfg).top_k(det, tag)
    for k in ("val_k", "loc_k", "tag_k"):
        assert np.array_equal(top[k], exp[k]), k
    assert np.array_equal(top["loc_k"][0, 0, :, 0], np.arange(30)) and (top["loc_k"][0, 0, :, 1] == 0).all()


@pytest.mark.parametrize("size,n,people,min_found", [(512, 4, 5, 5), (640, 2, 36, 65)])
def test_parser_bench_geometry_vs_oracle(size, n, people, min_found):
    """The parser at the geometry the bench runs it (BASELINE configs 3 and 5: 512^2 -> 8 strips per plane with the
    cross-CTA threshold; 640^2 crowd with more persons than the 64-person packed payload), bit-exact against the
    oracle for every person (reference lib/core/group.py:96,269-291 returns all of them)."""
    cfg = get_cfg(input_size=size)
    det, tag = synth.plant_crowd_batch(n, 14, size, size, 2, num_people=people, seed=300 + size)
    p = _parser(cfg)
    got = p.parse_batch(torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda(), True, True)
    exp = group_ref.HeatmapParser(cfg).parse_batch(det.copy(), tag.copy(), True, True)
    found = []
    for i in range(n):
        a = np.asarray(got[i][0][0], np.float32).reshape(-1, 14, 5)
        e = np.asarray(exp[i][0][0], np.float32).reshape(-1, 14, 5)
        assert a.shape == e.shape, (i, a.shape, e.shape)
        assert np.array_equal(a, e), i
        assert np.array_equal(np.asarray(got[i][1], np.float32), np.asarray(exp[i][1], np.float32))
        found.append(e.shape[0])
    assert max(found) >= min_found, found


# ---- round 2: wide matcher (MAX_NUM_PEOPLE up to 64), shared tag map, multi-scale glue -------------------------------
@pytest.fixture
def wide_matcher():
    """routes every lp_tag_match_f32 call through the two-columns-per-lane kernel (read per call by the library)"""
    os.environ["LP_MATCH_WIDE"] = "1"
    yield
    os.environ.pop("LP_MATCH_WIDE", None)


@pytest.mark.parametrize("case", [c for c in PARSER_CASES if c[0] in ("p5_128_t2", "p30_256_t2", "p30_256_t1",
                                                                      "coco_p8_128_t2", "p30_640_t2")],
                         ids=lambda c: c[0])
def test_parser_golden_wide_matcher(golden_dir, case, wide_matcher):
    """The reference goldens (K = 30) through the 64-wide matcher kernel: bit-exact like the 32-wide one."""
    test_parser_golden(golden_dir, case)


@pytest.mark.parametrize("k,people,size", [(48, 40, 320), (64, 60, 384), (33, 12, 192)])
def test_parser_more_than_32_people(k, people, size):
    """DATASET.MAX_NUM_PEOPLE above the warp width (the reference has no limit: lib/config/default.py, group.py:54):
    top-K with K > 32 and cost matrices up to 64 x 64, bit-exact against the oracle."""
    cfg = get_cfg(input_size=size)
    cfg.DATASET.MAX_NUM_PEOPLE = k
    n = 2
    det, tag = synth.plant_crowd_batch(n, 14, size, size, 2, num_people=people, seed=700 + k)
    p = _parser(cfg)
    got = p.parse_batch(torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda(), True, True)
    exp = group_ref.HeatmapParser(cfg).parse_batch(det.copy(), tag.copy(), True, True)
    found = []
    for i in range(n):
        a = np.asarray(got[i][0][0], np.float32).reshape(-1, 14, 5)
        e = np.asarray(exp[i][0][0], np.float32).reshape(-1, 14, 5)
        assert a.shape == e.shape, (i, a.shape, e.shape)
        assert np.array_equal(a, e), i
        assert np.array_equal(np.asarray(got[i][1], np.float32), np.asarray(exp[i][1], np.float32))
        found.append(e.shape[0])
    assert max(found) >= min(people, 33), found


def test_parser_shared_tag_golden(golden_dir):
    """MODEL.TAG_PER_JOINT=False (one tag map shared by all joints, reference group.py:150-152): top_k and the parse
    without refine against the reference's outputs; with refine (where the reference itself stops on an unassigned
    name, recorded in the fixture) against the oracle on the tiled maps."""
    from oracle.make_golden import shared_tag_case
    z = np.load(os.path.join(golden_dir, "parser_shared_tag_p6.npz"))
    cfg = get_cfg(input_size=256)
    cfg.MODEL.TAG_PER_JOINT = False
    det, tag = shared_tag_case(14, 128, 160, 2, 6, 31)
    assert hashlib.sha256(det.tobytes() + tag.tobytes()).hexdigest() == str(z["in_digest"])
    assert str(z["refine_raises"]).startswith("NameError")
    p = _parser(cfg)
    dd, td = torch.from_numpy(det)[None].cuda(), torch.from_numpy(tag)[None].cuda()
    assert_topk_equal(p.top_k(dd, td), {k: z[k] for k in ("val_k", "loc_k", "tag_k")}, "shared tag")
    for adj in (True, False):
        ans, scores = p.parse(dd, td, adj, False)
        a = np.asarray(ans[0], np.float32).reshape(-1, 14, 5)
        assert np.array_equal(a, z["ans_a%d_r0" % adj])
        assert np.array_equal(np.asarray(scores, np.float32), z["scores_a%d_r0" % adj])
    ans, scores = p.parse(dd, td, True, True)
    ea, es = group_ref.HeatmapParser(cfg).parse(det[None].copy(), tag[None].copy(), True, True)
    assert np.array_equal(np.asarray(ans[0], np.float32).reshape(-1, 14, 5), np.asarray(ea[0], np.float32).reshape(-1, 14, 5))
    assert np.array_equal(np.asarray(scores, np.float32), np.asarray(es, np.float32))


def _glue_scales_device(cfg, log, base_wh, first_hw):
    """the multi-scale loop through lp_glue_scale_f32: ``log`` = per scale (largest first) [plain outs, flipped outs]"""
    lib = _lib.load()
    flip = bool(cfg.TEST.FLIP_TEST)
    scales = sorted(cfg.TEST.SCALE_FACTOR, reverse=True)
    J = cfg.DATASET.NUM_JOINTS
    n = log[0][0].shape[0]
    Hd, Wd = (base_wh[1], base_wh[0]) if cfg.TEST.PROJECT2IMAGE else first_hw
    T = 2 if flip else 1
    det = torch.full((n, J, Hd, Wd), float("nan"), device="cuda")
    tag = torch.full((n, J, Hd, Wd, T), float("nan"), device="cuda")
    fidx = torch.tensor(flip_index_for(cfg), dtype=torch.int32, device="cuda")
    keep = []
    per = 2 if flip else 1
    for i, s in enumerate(scales):
        a = [t.cuda() for t in log[i * per]]
        b = [t.cuda() for t in log[i * per + 1]] if flip else [None, None]
        keep.append((a, b))
        h, w = a[0].shape[2], a[0].shape[3]
        _lib.check(lib.lp_glue_scale_f32(a[0].data_ptr(), a[1].data_ptr(), _lib.ptr(b[0]), _lib.ptr(b[1]), fidx.data_ptr(),
                                         n, J, J, 0, h, w, 1 if flip else 0, Hd, Wd, 1 if i > 0 else 0,
                                         float(len(scales)) if i == len(scales) - 1 else 1.0, det.data_ptr(),
                                         tag.data_ptr() if s == 1 else None, torch.cuda.current_stream().cuda_stream),
                   "lp_glue_scale_f32")
    torch.cuda.synchronize()
    return det.cpu(), tag.cpu()


def test_glue_multiscale_golden(golden_dir):
    """valid.py:205-225 with several TEST.SCALE_FACTOR entries: one lp_glue_scale_f32 launch per scale against the
    outputs of the reference's own get_multi_stage_outputs / aggregate_results loop."""
    from oracle.make_golden import MULTISCALE_CASES, FakeScaleModel, multiscale_inputs
    for name, scales, proj, flip, size, seed in MULTISCALE_CASES:
        z = np.load(os.path.join(golden_dir, "glue_%s.npz" % name))
        cfg = get_cfg(input_size=size, flip_test=flip, project2image=proj)
        cfg.TEST.SCALE_FACTOR = list(scales)
        base, images = multiscale_inputs(cfg, size)
        fake = FakeScaleModel(cfg.DATASET.NUM_JOINTS, seed)
        for s in sorted(scales, reverse=True):
            for _ in range(2 if flip else 1):
                fake(images[s])
        dig = hashlib.sha256(b"".join(o.numpy().tobytes() for outs in fake.log for o in outs)).hexdigest()
        assert dig == str(z["in_digest"]), "seeded inputs differ from the ones the fixture was generated with"
        first = images[max(scales)]
        det, tag = _glue_scales_device(cfg, fake.log, base, (first.shape[2] // 2, first.shape[3] // 2))
        ed, et = z["final_heatmaps"], z["tags"]
        assert det.shape == ed.shape and tag.shape == et.shape
        assert np.abs(det.numpy() - ed).max() <= 1e-5 * max(1.0, np.abs(ed).max()), name
        assert np.abs(tag.numpy() - et).max() <= 1e-5 * max(1.0, np.abs(et).max()), name


@pytest.mark.parametrize("scales,proj,hw", [([0.75, 1, 1.25], True, (192, 256)), ([1, 1.5, 2.5], True, (128, 128)),
                                            ([0.5, 1, 2], False, (128, 192)), ([1, 2], True, (64, 64))])
def test_glue_multiscale_ratios_vs_oracle(scales, proj, hw):
    """projection ratios other than x2 / x4 (1.6x, 1.33x, identity, 0.8x shrink), non-square frames, three scales"""
    from oracle.make_golden import FakeScaleModel
    cfg = get_cfg(input_size=hw[0], flip_test=True, project2image=proj)
    cfg.TEST.SCALE_FACTOR = list(scales)
    smin = min(scales)
    images = {s: torch.zeros(2, 3, int(round(hw[0] * s / 64)) * 64, int(round(hw[1] * s / 64)) * 64) for s in scales}
    images[1] = torch.zeros(2, 3, hw[0], hw[1])
    base = (hw[1], hw[0])
    fake = FakeScaleModel(14, 5)
    ed, et = glue_ref.multi_scale(cfg, fake, images, base)
    first = images[max(scales)]
    det, tag = _glue_scales_device(cfg, fake.log, base, (first.shape[2] // 2, first.shape[3] // 2))
    assert det.shape == ed.shape and tag.shape == et.shape, (det.shape, ed.shape, smin)
    assert (det - ed).abs().max().item() <= 1e-5 * max(1.0, ed.abs().max().item())
    assert (tag - et).abs().max().item() <= 1e-5 * max(1.0, et.abs().max().item())


def test_glue_cfg_branches_golden(golden_dir):
    """DATASET.WITH_CENTER (centre joint kept / ignored) and MODEL.TAG_PER_JOINT off through lp_glue_scale_f32 against the
    outputs of the unmodified reference (lib/core/inference.py:95-150)."""
    from oracle.make_golden import GLUE_CFG_CASES, GLUE_CFG_SIZE, FakeScaleModel, glue_cfg
    lib = _lib.load()
    for name, center, ignore, per_joint, proj, seed in GLUE_CFG_CASES:
        z = np.load(os.path.join(golden_dir, "glue_cfg_%s.npz" % name))
        cfg = glue_cfg(center, ignore, per_joint, proj)
        jm = cfg.DATASET.NUM_JOINTS
        fake = FakeScaleModel(jm, seed, None if per_joint else 1)
        img = torch.zeros(2, 3, GLUE_CFG_SIZE, GLUE_CFG_SIZE)
        a, b = [t.cuda() for t in fake(img)], [t.cuda() for t in fake(img)]
        dig = hashlib.sha256(b"".join(o.numpy().tobytes() for outs in fake.log for o in outs)).hexdigest()
        assert dig == str(z["in_digest"])
        ed, et = z["final_heatmaps"], z["tags"]
        n, J, Hd, Wd = ed.shape
        assert J == (jm - 1 if (center and ignore) else jm) and et.shape[1] == (J if per_joint else 1)
        det = torch.full(ed.shape, float("nan"), device="cuda")
        tag = torch.full(et.shape, float("nan"), device="cuda")
        fidx = torch.tensor(flip_index_for(cfg), dtype=torch.int32, device="cuda")
        h, w = a[0].shape[2], a[0].shape[3]
        _lib.check(lib.lp_glue_scale_f32(a[0].data_ptr(), a[1].data_ptr(), b[0].data_ptr(), b[1].data_ptr(), fidx.data_ptr(),
                                         n, J, jm, 0 if per_joint else 1, h, w, 1, Hd, Wd, 0, 1.0, det.data_ptr(),
                                         tag.data_ptr(), torch.cuda.current_stream().cuda_stream), "lp_glue_scale_f32")
        torch.cuda.synchronize()
        assert np.abs(det.cpu().numpy() - ed).max() <= 1e-5 * max(1.0, np.abs(ed).max()), name
        assert np.abs(tag.cpu().numpy() - et).max() <= 1e-5 * max(1.0, np.abs(et).max()), name
