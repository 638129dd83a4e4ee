"""-m gpu: mixed batches (LitePosePipeline.infer_images on a list of differently sized images).  The ragged kernels
against the uniform ones image by image (bit for bit), one ragged parse against the oracle, and the whole mixed call
against one batch-1 call per image; plus the memory bound of a stream of mixed batches."""
import numpy as np
import pytest
import torch

from litepose_b200 import _lib, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.core.group import Params
from litepose_b200.lib.models.pose_mobilenet import get_pose_net
from litepose_b200.lib.utils import transforms as T
from litepose_b200.mixed import MAP_DESC, MixedPlan
from litepose_b200.parser import DeviceParser
from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
from oracle import group_ref
from parity_util import assert_topk_equal

pytestmark = pytest.mark.gpu

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
SHAPES = [(150, 200), (200, 150), (150, 200), (100, 300), (120, 120), (201, 149)]


def _images(shapes, seed=3):
    rng = np.random.RandomState(seed)
    return [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]


@pytest.mark.parametrize("half", [True, False])
@pytest.mark.parametrize("scales", [[1.0], [2.0, 1.0, 0.5]])
def test_ragged_warp_equals_uniform_per_image(half, scales):
    imgs = _images(SHAPES)
    size = 128
    mp = MixedPlan([im.shape[:2] for im in imgs], scales, size, True, 14, 2)
    lib = _lib.load()
    src = torch.from_numpy(np.concatenate([imgs[i].ravel() for i in mp.order])).cuda()
    dt = torch.float16 if half else torch.float32
    mean_a, std_a = np.asarray(MEAN, np.float32), np.asarray(STD, np.float32)
    for s in scales:
        desc = torch.from_numpy(mp.warp_desc(s).view(np.uint8)).cuda()
        out = torch.full((int(mp.in_off[s][-1]),), float("nan"), dtype=dt, device="cuda")
        mh, mw = mp.max_in_hw(s)
        _lib.check(lib.lp_warp_affine_normalize_ragged_u8(src.data_ptr(), mp.n, desc.data_ptr(), mw, mh,
                                                           mean_a.ctypes.data, std_a.ctypes.data, out.data_ptr(),
                                                           2 if half else 1, torch.cuda.current_stream().cuda_stream),
                   "ragged warp")
        for p, i in enumerate(mp.order):
            exp, _, _ = T.resize_align_normalize_device(imgs[i], size, s, min(scales), MEAN, STD, half=half)
            got = out[int(mp.in_off[s][p]):int(mp.in_off[s][p + 1])].view(exp.shape)
            assert torch.equal(got.view(torch.int16 if half else torch.int32),
                               exp.view(torch.int16 if half else torch.int32)), (s, i)


def _parser(cfg):
    p = Params(cfg)
    return DeviceParser(p.num_joints, p.max_num_people, p.detection_threshold, p.tag_threshold, p.use_detection_val,
                        p.ignore_too_much, p.joint_order, cfg.TEST.NMS_KERNEL, cfg.TEST.NMS_PADDING)


def _arena(maps, t):
    """maps: [(det [J,h,w], tag [J,h,w,t])] -> device det / tag arena, host hw, device lp_map_desc_t."""
    n = len(maps)
    desc = np.zeros(n, MAP_DESC)
    d0 = t0 = 0
    for i, (d, g) in enumerate(maps):
        desc[i] = (d.shape[1], d.shape[2], d0, t0)
        d0 += d.size
        t0 += g.size
    det = torch.from_numpy(np.concatenate([d.ravel() for d, _ in maps])).cuda()
    tag = torch.from_numpy(np.concatenate([g.ravel() for _, g in maps])).cuda()
    hw = np.ascontiguousarray(np.stack([desc["h"], desc["w"]], 1), np.int32)
    return det, tag, hw, torch.from_numpy(desc.view(np.uint8)).cuda()


MAP_CASES = [((64, 96), 0), ((128, 128), 4), ((96, 160), 40), ((128, 64), 2), ((64, 96), 6)]


@pytest.mark.parametrize("t", [1, 2])
@pytest.mark.parametrize("people_cap", [30, 64])
def test_ragged_parser_equals_uniform_per_image(t, people_cap):
    """Different map sizes in one arena: an image with nobody, one with more persons than MAX_NUM_PEOPLE, the wide
    matcher (MAX_NUM_PEOPLE 64); val_k / ind_k / tag_k, ans, num, scores bit-identical to the uniform chain."""
    cfg = get_cfg(input_size=128)
    cfg.DATASET.MAX_NUM_PEOPLE = people_cap
    par = _parser(cfg)
    J, K = par.J, par.K
    maps = [synth.plant_crowd(J, h, w, t, num_people=pp, seed=31 + i) for i, ((h, w), pp) in enumerate(MAP_CASES)]
    det, tag, hw, desc = _arena(maps, t)
    ans, num, scores = par.run_ragged(det, tag, hw, desc.data_ptr(), t, True, True)
    n = len(maps)
    rb = par.last_ragged
    vk = rb["val_k"][:n * J * K].view(n, J, K).cpu()
    ik = rb["ind_k"][:n * J * K].view(n, J, K).cpu()
    tk = rb["tag_k"][:n * J * K * t].view(n, J, K, t).cpu()
    ans, num, scores = ans.cpu(), num.cpu(), scores.cpu()
    assert int(num[0]) == 0 and int(num[2]) > 30
    for i, (d, g) in enumerate(maps):
        dd, gg = torch.from_numpy(d[None]).cuda(), torch.from_numpy(g[None]).cuda()
        ua, un, us = [x.cpu() for x in par.run(dd, gg, True, True)]
        uv, ui, ut = [x.cpu() for x in par.top_k_device(dd, gg, par.det_thr)]
        assert torch.equal(vk[i], uv[0]) and torch.equal(ik[i], ui[0]) and torch.equal(tk[i], ut[0]), i
        p = int(un[0])
        assert int(num[i]) == p, i
        assert torch.equal(ans[i, :p], ua[0, :p]) and torch.equal(scores[i, :p], us[0, :p]), i


def test_ragged_parse_equals_oracle():
    """One mixed case against oracle/group_ref: the full-range top-K (min_value 0) with the tie rule of
    parity_util, and the parse (keypoints and scores) bit for bit."""
    cfg = get_cfg(input_size=128)
    par = _parser(cfg)
    J, K, t = par.J, par.K, 2
    maps = [synth.plant_crowd(J, h, w, t, num_people=pp, seed=51 + i) for i, ((h, w), pp) in enumerate(MAP_CASES)]
    det, tag, hw, desc = _arena(maps, t)
    n = len(maps)
    lib = _lib.load()
    ws = torch.empty(par.workspace_bytes_ragged(hw, t)[0], dtype=torch.uint8, device="cuda")
    vk = torch.empty((n, J, K), dtype=torch.float32, device="cuda")
    ik = torch.empty((n, J, K), dtype=torch.int32, device="cuda")
    tk = torch.empty((n, J, K, t), dtype=torch.float32, device="cuda")
    _lib.check(lib.lp_nms_topk_ragged_f32(det.data_ptr(), tag.data_ptr(), n, hw.ctypes.data, desc.data_ptr(), J, t,
                                          par.nms_kernel, K, 0.0, vk.data_ptr(), ik.data_ptr(), tk.data_ptr(),
                                          ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream), "topk")
    vk, ik, tk = vk.cpu().numpy(), ik.cpu().numpy(), tk.cpu().numpy()
    ans, num, scores = [x.cpu().numpy() for x in par.run_ragged(det, tag, hw, desc.data_ptr(), t, True, True)]
    op = group_ref.HeatmapParser(cfg)
    for i, (d, g) in enumerate(maps):
        w = d.shape[2]
        exp = op.top_k(d[None].copy(), g[None].copy())
        got = {"val_k": vk[i:i + 1], "tag_k": tk[i:i + 1],
               "loc_k": np.stack([ik[i:i + 1] % w, ik[i:i + 1] // w], -1).astype(np.int64)}
        assert_topk_equal(got, exp, "image %d" % i)
        e_ans, e_sc = op.parse(d[None].copy(), g[None].copy(), True, True)
        e = np.asarray(e_ans[0], np.float32).reshape(-1, J, 3 + t)
        assert int(num[i]) == e.shape[0], i
        assert np.array_equal(ans[i, :e.shape[0]], e), i
        assert np.array_equal(scores[i, :e.shape[0]], np.asarray(e_sc, np.float32)), i


def _pipe(cfg, keep=64):
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch("XS")), 1)).eval()
    return LitePosePipeline(model.cuda(), cfg, use_graphs=True, keep=keep)


def _plants(pipe, mp, shapes, heat_only=False):
    J, t = pipe.params.num_joints, 2 if pipe.flip else 1
    out = []
    for i in range(len(shapes)):
        if i == 4:
            out.append(None)                       # one image without planted persons
            continue
        hd, wd = mp.det_hw[mp.pos[i]]
        pl = PlantedCrowd(1, J, int(hd), int(wd), t, num_people=3, seed=40 + i, device="cuda")
        if heat_only:
            pl.tidx, pl.tval = pl.tidx[:0], pl.tval[:0]
        out.append(pl)
    return out


def _cfg_case(name):
    from oracle.make_golden import glue_cfg
    if name == "shipped":
        return get_cfg(input_size=128)
    if name == "nano":
        cfg = get_cfg(input_size=128)
        cfg.TEST.FLIP_TEST = False
        cfg.TEST.ADJUST = False
        cfg.TEST.REFINE = False
        return cfg
    if name == "multiscale":
        cfg = get_cfg(input_size=128)
        cfg.TEST.SCALE_FACTOR = [0.5, 1, 2]
        return cfg
    if name == "coco":
        return glue_cfg(False, False, True, True, size=128, dataset="coco")
    if name == "shared_tag":
        return glue_cfg(False, True, False, True, size=128)
    raise KeyError(name)


@pytest.mark.parametrize("case", ["shipped", "nano", "multiscale", "coco", "shared_tag"])
def test_infer_images_list_equals_one_call_per_image(case):
    cfg = _cfg_case(case)
    pipe = _pipe(cfg, keep=2)                      # keep 2: the planted crowds overflow the payload of some images
    imgs = _images(SHAPES, seed=7)
    shapes = [im.shape[:2] for im in imgs]
    mp = MixedPlan(shapes, pipe.scales, 128, pipe.project, pipe.params.num_joints, 2 if pipe.flip else 1)
    assert len(mp.groups) >= 4
    plants = _plants(pipe, mp, shapes, heat_only=case == "shared_tag")
    got = pipe.infer_images(imgs, plant=plants)
    got2 = pipe.infer_images([torch.from_numpy(im) for im in imgs], plant=plants)
    assert len(got) == len(imgs)
    found = 0
    for i, im in enumerate(imgs):
        exp = pipe.infer_images(torch.from_numpy(im)[None].pin_memory(), plant=plants[i])[0]
        for res in (got, got2):
            assert res[i][2] == exp[2], (case, i)
            assert np.array_equal(res[i][0], exp[0]), (case, i)
            assert np.array_equal(np.asarray(res[i][1], np.float32), np.asarray(exp[1], np.float32)), (case, i)
        found += exp[2]
    assert found > 0


def test_mixed_batches_memory_bound():
    """A stream of mixed batches of different compositions: after a batch that holds the largest group and the most
    images, neither the device memory nor the number of plans grows."""
    from litepose_b200.engine import ARENA_PLANS
    cfg = get_cfg(input_size=128)
    pipe = _pipe(cfg)
    rng = np.random.RandomState(5)
    pool = [(150, 200), (200, 150), (100, 300), (120, 120), (300, 100), (130, 170)]
    first = pool * 6                               # every group at least as large as in any batch below
    pipe.infer_images(_images(first, seed=1))
    torch.cuda.synchronize()
    mem0 = torch.cuda.memory_allocated()
    plans0 = len(pipe.engine.plans)
    for b in range(5):
        k = rng.randint(3, 7)
        shapes = [pool[j] for j in rng.randint(0, len(pool), k)]
        res = pipe.infer_images(_images(shapes, seed=10 + b))
        assert len(res) == k
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() <= mem0, b
        assert len(pipe.engine.plans) == plans0 and len(pipe.engine.arena_plans) <= ARENA_PLANS
