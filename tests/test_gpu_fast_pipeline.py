"""-m gpu: the pipeline's fast grouping mode (LitePosePipeline(grouping="fast"): the demo's peak finder + KM assignment
inside the step).  The new peak finder on the glue's maps against lp_find_peaks_f32 bit for bit (uniform, in-place tag
channel 0, shared tag map, ragged arena); every entry point of the pipeline against the standalone parser
fast_utils.group.HeatmapParser.parse_batch on the same step's maps; the reference's own compiled code on two images."""
import numpy as np
import pytest
import torch

from litepose_b200 import _lib, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.fast_utils import plugins
from litepose_b200.fast_utils.group import HeatmapParser as FastParser
from litepose_b200.lib.models.pose_mobilenet import get_pose_net
from litepose_b200.lib.utils import transforms as T
from litepose_b200.mixed import MAP_DESC, MixedPlan
from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd, unpack_fast_payload

pytestmark = pytest.mark.gpu

THR, WIN = 0.1, 5


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _peak_outputs(n, j, m):
    """count / val / tag / ind pre-filled with -7: entries past the count must stay untouched."""
    return (torch.full((n, j), -7, dtype=torch.int32, device="cuda"), torch.full((n, j, m), -7.0, device="cuda"),
            torch.full((n, j, m), -7.0, device="cuda"), torch.full((n, j, m, 2), -7, dtype=torch.int32, device="cuda"))


def _peaks_uniform(det, tmap, m):
    """lp_find_peaks_f32 on det [N,J,H,W] and a plain [N,J,H,W] tag map."""
    n, j, h, w = det.shape
    out = _peak_outputs(n, j, m)
    _lib.check(_lib.load().lp_find_peaks_f32(det.data_ptr(), tmap.contiguous().data_ptr(), n, j, h, w, m, THR, WIN,
                                             *[t.data_ptr() for t in out], _stream()), "lp_find_peaks_f32")
    return [t.cpu() for t in out]


def _peaks_maps(det, tag, n, j, t, tag_planes, m, hw=None, desc=None):
    out = _peak_outputs(n, j, m)
    h, w = (det.shape[2], det.shape[3]) if desc is None else (0, 0)
    _lib.check(_lib.load().lp_find_peaks_maps_f32(
        det.data_ptr(), tag.data_ptr(), n, h, w, None if hw is None else hw.ctypes.data,
        None if desc is None else desc.data_ptr(), j, t, tag_planes, m, THR, WIN, *[x.data_ptr() for x in out],
        _stream()), "lp_find_peaks_maps_f32")
    return [x.cpu() for x in out]


def _assert_same(got, exp, what):
    for name, g, e in zip(("count", "val", "tag", "ind"), got, exp):
        assert torch.equal(g.view(torch.int32) if g.is_floating_point() else g,
                           e.view(torch.int32) if e.is_floating_point() else e), (what, name)


# ---------------------------------------------------------------------------------------------- kernel parity
@pytest.mark.parametrize("t", [1, 2])
@pytest.mark.parametrize("m", [8, 30])
def test_find_peaks_maps_uniform_reads_tag_channel_0_in_place(t, m):
    det, tag = synth.plant_crowd_batch(3, 14, 64, 96, t, num_people=12, seed=5)
    det, tag = torch.from_numpy(det).cuda(), torch.from_numpy(tag).cuda()
    got = _peaks_maps(det, tag, 3, 14, t, 14, m)
    exp = _peaks_uniform(det, tag[..., 0].contiguous(), m)
    _assert_same(got, exp, "uniform T=%d" % t)
    assert int(exp[0].max()) > 0 and (m > 8 or int(exp[0].max()) == 8)


def test_find_peaks_maps_shared_tag_map():
    det, tag = synth.plant_crowd_batch(2, 14, 80, 64, 2, num_people=6, seed=8)
    det = torch.from_numpy(det).cuda()
    shared = torch.from_numpy(tag[:, 3:4]).cuda().contiguous()           # [N,1,H,W,T]: one map for every joint
    got = _peaks_maps(det, shared, 2, 14, 2, 1, 30)
    exp = _peaks_uniform(det, shared[..., 0].expand(-1, 14, -1, -1).contiguous(), 30)
    _assert_same(got, exp, "shared")


RAGGED = [(64, 96), (96, 64), (128, 128), (40, 200), (200, 40), (64, 96)]


@pytest.mark.parametrize("shared", [False, True])
def test_find_peaks_maps_ragged_equals_uniform_per_image(shared):
    """Planes of different sizes (portrait and landscape) in one launch; each image against the uniform call on it."""
    J, t, m = 14, 2, 30
    maps = [synth.plant_crowd(J, h, w, t, num_people=3 + i, seed=60 + i) for i, (h, w) in enumerate(RAGGED)]
    if shared:
        maps = [(d, np.ascontiguousarray(g[:1])) for d, g in maps]
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
    got = _peaks_maps(det, tag, n, J, t, 1 if shared else J, m, hw, torch.from_numpy(desc.view(np.uint8)).cuda())
    for i, (d, g) in enumerate(maps):
        tm = torch.from_numpy(g[None, ..., 0]).cuda().expand(-1, J, -1, -1)
        exp = _peaks_uniform(torch.from_numpy(d[None]).cuda(), tm, m)
        _assert_same([x[i:i + 1] for x in got], exp, "ragged image %d" % i)


def test_pack_fast_payload_rows():
    n, m, c = 3, 4, 5
    ans = torch.randn(n, m, c, 4, device="cuda")
    num = torch.tensor([0, 4, 2], dtype=torch.int32, device="cuda")
    status = torch.tensor([0, 0, 1], dtype=torch.int32, device="cuda")
    packed = torch.full((n, m * c * 4 + 2), -1.0, device="cuda")
    _lib.check(_lib.load().lp_pack_fast_payload_f32(ans.data_ptr(), num.data_ptr(), status.data_ptr(), n, m, c,
                                                    packed.data_ptr(), _stream()), "lp_pack_fast_payload_f32")
    exp = torch.cat([ans.view(n, -1), num.float()[:, None], status.float()[:, None]], 1)
    assert torch.equal(packed, exp)


# ---------------------------------------------------------------------------------------------- pipeline
def _model(cfg):
    torch.manual_seed(0)
    return synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch("XS")), 1)).eval().cuda()


def _fast_cfg(size=128, flip=True, dataset="crowd_pose", per_joint=True, scales=(1,)):
    from oracle.make_golden import glue_cfg
    cfg = glue_cfg(False, True, per_joint, True, size=size, dataset=dataset)
    cfg.TEST.FLIP_TEST = flip
    cfg.TEST.ADJUST = cfg.TEST.REFINE = False
    cfg.TEST.SCALE_FACTOR = list(scales)
    return cfg


def _plant(pipe, n, h, w, people, seed):
    J, t = pipe.params.num_joints, 2 if pipe.flip else 1
    pl = PlantedCrowd(n, J, h, w, t, num_people=people, seed=seed, device="cuda")
    if pipe.tag_shared:
        pl.tidx, pl.tval = pl.tidx[:0], pl.tval[:0]          # the tag patches index J maps: heat peaks only
    return pl


def _expected(pipe, det, tag):
    """parse_batch of the standalone parser on the step's det / tag -> (num [N], ans [N,M,J,4]) host."""
    if tag.shape[1] == 1:
        tag = tag.expand(-1, det.shape[1], -1, -1, -1)
    num, ans = FastParser(pipe.cfg).parse_batch(det, tag)
    assert int(plugins.last_status().abs().sum()) == 0
    return num.cpu().numpy(), ans.cpu().numpy()


def _check_packed(pipe, packed, det, tag):
    """The step's payload equals parse_batch element for element, zeroed tails included; returns the counts."""
    num, ans = _expected(pipe, det, tag)
    M, J = pipe.fast["M"], pipe.params.num_joints
    p = packed.cpu().numpy()
    n = p.shape[0]
    assert p.shape[1] == M * J * 4 + 2
    assert np.array_equal(p[:, :-2].reshape(n, M, J, 4), ans)
    assert np.array_equal(p[:, -2], num.astype(np.float32)) and (p[:, -1] == 0).all()
    return num


@pytest.mark.parametrize("flip,dataset,per_joint,people", [
    (True, "crowd_pose", True, 5), (False, "crowd_pose", True, 5), (True, "coco", True, 5),
    (True, "crowd_pose", False, 5), (False, "coco", False, 3)])
def test_step_device_equals_parse_batch(flip, dataset, per_joint, people):
    n, size = 2, 128
    cfg = _fast_cfg(size, flip, dataset, per_joint)
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
    assert pipe.params.num_joints == (14 if dataset == "crowd_pose" else 17)
    x = synth.make_frames(n, size, seed=11).half().cuda()
    plant = _plant(pipe, n, size, size, people, seed=3)
    for _ in range(2):                                        # capture, then replay
        packed = pipe.step_device(x, plant).clone()
        st = pipe._get_state(n, size, size, torch.float16, plant)
        num = _check_packed(pipe, packed, st["det"], st["tag"])
    assert num.min() >= 1


def test_step_crowds_0_5_30_zeroed_tails():
    """One pipeline, one set of buffers: a 30-person crowd, then 5, then nobody - the rows a smaller crowd leaves
    unassigned read zero, as in the allocate-and-return parser."""
    n, size = 2, 256
    cfg = _fast_cfg(size)
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
    x = synth.make_frames(n, size, seed=12).half().cuda()
    counts = []
    for people in (30, 5, 0):
        plant = _plant(pipe, n, size, size, people, seed=20 + people)
        packed = pipe.step_device(x, plant).clone()
        st = pipe._get_state(n, size, size, torch.float16, plant)
        counts.append(_check_packed(pipe, packed, st["det"], st["tag"]))
    assert counts[0].max() > 20 and counts[1].max() <= 12 and counts[2].max() == 0, counts
    res = pipe.step(synth.make_frames(n, size, seed=12).half().pin_memory(), plant)
    assert [r[1] for r in res] == [0, 0] and res[0][0].shape == (0, 14, 4)


def test_step_multiscale_equals_parse_batch():
    n, size = 2, 128
    cfg = _fast_cfg(size, scales=(0.5, 1, 2))
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
    frames = {float(s): synth.make_frames(n, int(size * s), seed=40 + i) for i, s in enumerate((0.5, 1, 2))}
    plant = _plant(pipe, n, size, size, 4, seed=9)
    got = pipe.step_multiscale({s: f.half().pin_memory() for s, f in frames.items()}, plant)
    st = pipe._get_state(n, size, size, torch.float16, plant, det_hw=(size, size))
    num = _check_packed(pipe, st["packed"], st["det"], st["tag"])
    _, ans = _expected(pipe, st["det"], st["tag"])
    for i in range(n):
        assert got[i][1] == num[i] >= 1 and np.array_equal(got[i][0], ans[i, :num[i]])


def test_step_equals_compiled_reference():
    """The reference's own find_peaks.cpp / assign.cpp (compiled into oracle/_ref/ by build()) on the step's maps."""
    from oracle import fast_utils_ref as fu
    if not fu.available("ref"):
        pytest.skip("oracle/_ref/libfastutils_ref.so absent: build() found no reference checkout to compile")
    n, size = 2, 128
    cfg = _fast_cfg(size)
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
    plant = _plant(pipe, n, size, size, 5, seed=31)
    got = pipe.step(synth.make_frames(n, size, seed=13).half().pin_memory(), plant)
    st = pipe._get_state(n, size, size, torch.float16, plant)
    det, tag = st["det"].cpu().numpy(), st["tag"].cpu().numpy()
    J = pipe.params.num_joints
    params = dict(detection_threshold=THR, window_size=WIN, max_num_people=30, tag_threshold=1.0,
                  joint_order=[j for j in pipe.params.joint_order if j < J][:J])
    exp = fu.parse(det, tag, params, "ref")
    for i, (num, ans, _) in enumerate(exp):
        assert num >= 3 and got[i][1] == num
        assert np.array_equal(got[i][0], ans[:num]), i


def test_submit_collect_equals_step():
    n, size = 2, 128
    cfg = _fast_cfg(size)
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
    plant = _plant(pipe, n, size, size, 4, seed=5)
    fa = synth.make_frames(n, size, seed=1).half().pin_memory()
    fb = synth.make_frames(n, size, seed=2).half().pin_memory()
    ref = {"a": pipe.step(fa, plant), "b": pipe.step(fb, plant)}
    seq = ["a", "b", "b", "a"]
    got, prev = [], None
    for k in seq:
        tk = pipe.submit(fa if k == "a" else fb, plant)
        if prev is not None:
            got.append(pipe.collect(prev)[0])
        prev = tk
    got.append(pipe.collect(prev)[0])
    for k, g in zip(seq, got):
        assert [r[1] for r in g] == [r[1] for r in ref[k]] and all(r[1] >= 1 for r in g)
        assert all(np.array_equal(x[0], y[0]) for x, y in zip(g, ref[k]))


def test_set_final_preds_equals_host_get_final_preds():
    n, size = 2, 128
    cfg = _fast_cfg(size)
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
    plant = _plant(pipe, n, size, size, 5, seed=17)
    centers, scales = [[150.0, 100.0], [60.5, 90.25]], [[300.0, 300.0], [121.0, 121.0]]
    pipe.set_final_preds(centers, scales)
    got = pipe.step(synth.make_frames(n, size, seed=4).half().pin_memory(), plant)
    st = pipe._get_state(n, size, size, torch.float16, plant)
    num, ans = _expected(pipe, st["det"], st["tag"])
    for i in range(n):
        assert got[i][1] == num[i] >= 1
        exp = T.get_final_preds([list(ans[i, :num[i]])], np.asarray(centers[i]), np.asarray(scales[i]), [size, size])
        assert np.array_equal(got[i][0], np.stack(exp).astype(np.float32)), i


def test_infer_images_list_equals_one_call_per_image():
    cfg = _fast_cfg(128)
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
    shapes = [(150, 200), (200, 150), (150, 200), (100, 300), (120, 120), (201, 149)]
    rng = np.random.RandomState(7)
    imgs = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    mp = MixedPlan(shapes, pipe.scales, 128, pipe.project, 14, 2)
    plants = []
    for i in range(len(shapes)):
        hd, wd = mp.det_hw[mp.pos[i]]
        plants.append(None if i == 4 else _plant(pipe, 1, int(hd), int(wd), 3, seed=40 + i))
    got = pipe.infer_images(imgs, plant=plants)
    found = 0
    for i, im in enumerate(imgs):
        exp = pipe.infer_images(torch.from_numpy(im)[None].pin_memory(), plant=plants[i])[0]
        assert got[i][1] == exp[1] and np.array_equal(got[i][0], exp[0]), i
        found += exp[1]
    assert found >= 5


def test_shared_tag_infer_images_list():
    cfg = _fast_cfg(128, per_joint=False)
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
    shapes = [(150, 200), (100, 300), (200, 150)]
    rng = np.random.RandomState(9)
    imgs = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    mp = MixedPlan(shapes, pipe.scales, 128, pipe.project, 14, 2)
    plants = [_plant(pipe, 1, int(mp.det_hw[mp.pos[i]][0]), int(mp.det_hw[mp.pos[i]][1]), 3, seed=70 + i)
              for i in range(len(shapes))]
    got = pipe.infer_images(imgs, plant=plants)
    for i, im in enumerate(imgs):
        exp = pipe.infer_images(torch.from_numpy(im)[None].pin_memory(), plant=plants[i])[0]
        assert got[i][1] == exp[1] >= 1 and np.array_equal(got[i][0], exp[0]), i


def test_ae_mode_unchanged():
    """A pipeline built without grouping= and one with grouping="ae" produce the same packed payload (the persons
    found: the slots past the count are not written by the parser), with a fast pipeline on the same model stepping
    in between."""
    n, size = 2, 128
    cfg = get_cfg(input_size=size)
    model = _model(cfg)
    default = LitePosePipeline(model, cfg, use_graphs=True)
    ae = LitePosePipeline(model, cfg, use_graphs=True, grouping="ae")
    fast = LitePosePipeline(model, _fast_cfg(size), use_graphs=True, grouping="fast")
    fr = synth.make_frames(n, size, seed=6).half().pin_memory()
    plant = PlantedCrowd(n, 14, size, size, 2, num_people=4, seed=2, device="cuda")
    a = default.step(fr, plant)
    fast.step(fr, plant)
    b = ae.step(fr, plant)
    assert default._get_state(n, size, size, torch.float16, plant)["packed"].shape == (n, 64 * 14 * 5 + 64 + 1)
    assert [r[2] for r in a] == [r[2] for r in b] and min(r[2] for r in a) >= 1
    for x, y in zip(a, b):
        assert x[0].shape[1:] == (14, 5) and np.array_equal(x[0], y[0])
        assert np.array_equal(np.asarray(x[1], np.float32), np.asarray(y[1], np.float32))


def test_graph_captured_fast_step_launch_count():
    """The fast parser is three library kernels (find_peaks_maps, assign, pack) plus get_final_preds when final
    predictions are set; the zeroing of ans is a torch fill node of the same graph."""
    n, size = 2, 128
    cfg = _fast_cfg(size)
    pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
    lib = _lib.load()
    x = synth.make_frames(n, size, seed=8).half().cuda()
    plant = _plant(pipe, n, size, size, 3, seed=4)
    for final, expected in ((False, 3), (True, 4)):
        pipe.set_final_preds([[64.0, 64.0]] * n if final else None, [[128.0, 128.0]] * n if final else None)
        pipe.step_device(x, plant)
        st = pipe._get_state(n, size, size, torch.float16, plant)
        torch.cuda.synchronize()
        lib.lp_reset_launch_count()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            pipe._parser_part(st, st["det"], st["tag"], st["packed"])
        assert lib.lp_launch_count() == expected
        g.replay()
        torch.cuda.synchronize()
    # the whole step: the network + glue launches plus those of the parser
    pipe.set_final_preds(None)
    st = pipe._get_state(n, size, size, torch.float16, plant)
    lib.lp_reset_launch_count()
    pipe._forward_part(st, x, st["det"], st["tag"])
    fwd = lib.lp_launch_count()
    lib.lp_reset_launch_count()
    pipe._device_step(st, x)
    torch.cuda.synchronize()
    assert lib.lp_launch_count() == fwd + 3


def test_status_one_raises():
    cfg = _fast_cfg(128)
    pipe = LitePosePipeline(_model(cfg), cfg, grouping="fast")
    row = np.zeros((2, 30 * 14 * 4 + 2), np.float32)
    row[1, -1] = 1
    with pytest.raises(_lib.LitePoseError):
        pipe.unpack_fast(torch.from_numpy(row))
    assert unpack_fast_payload(row[:1], 30, 14)[0][1] == 0


def _two_rank_worker(rank, port, q):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=2)
    try:
        n, size = 2, 128
        cfg = _fast_cfg(size)
        pipe = LitePosePipeline(_model(cfg), cfg, use_graphs=True, grouping="fast")
        plant = _plant(pipe, n, size, size, 4, seed=10 + rank)
        fr = synth.make_frames(n, size, seed=100, rank=rank).half().pin_memory()
        tk = pipe.submit(fr, plant, group=dist.group.WORLD, dst=0)
        res = pipe.collect(tk)
        own = pipe.step(fr, plant)
        q.put((rank, None if res is None else [[(a.tolist(), p) for a, p in r] for r in res],
               [(a.tolist(), p) for a, p in own]))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (one rank per GPU, NCCL gather)")
def test_two_rank_gather():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_two_rank_worker, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = {}
    for _ in range(2):
        rank, res, own = q.get(timeout=600)
        out[rank] = (res, own)
    for p in procs:
        p.join(timeout=60)
    assert out[1][0] is None
    gathered = out[0][0]
    assert len(gathered) == 2
    for r in range(2):
        assert gathered[r] == out[r][1]
