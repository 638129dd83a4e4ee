"""-m gpu: the glue kernels (csrc/glue.cu) equal their CPU restatement tests/glue_emul.py bit for bit, on every path
glue_launch can choose, for every input kind of glue_emul.KINDS.  det and tag are prefilled with NaN inside a guard
region, compared as uint32, and the guard (and the tag planes a call must not write) stay NaN."""
import numpy as np
import pytest
import torch

import glue_emul as ge
from litepose_b200 import _lib

pytestmark = pytest.mark.gpu

_NAN_BITS = np.float32(np.nan).view(np.uint32)
_GUARD = 4096


def _buffer(shape):
    """a NaN-filled device tensor of ``shape`` with _GUARD NaNs after it; returns (view, whole)"""
    whole = torch.full((int(np.prod(shape)) + _GUARD,), float("nan"), device="cuda")
    return whole[:int(np.prod(shape))].view(shape), whole


def _run_device(case, inputs):
    lib = _lib.load()
    J, N, Hd, Wd = case["J"], case["N"], case["Hd"], case["Wd"]
    T = 2 if case["flip"] else 1
    det, det_all = _buffer((N, J, Hd, Wd))
    tag, tag_all = _buffer((N, 1 if case["tag_shared"] else J, Hd, Wd, T))
    fidx = torch.tensor(ge.flip_index(J), dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    keep = []
    for (h, w, acc, div, wt), arrs in zip(case["calls"], inputs):
        o0, o1, f0, f1 = [None if a is None else torch.from_numpy(a).cuda() for a in arrs]
        keep.append((o0, o1, f0, f1))
        if case["entry"] == "f32":
            assert case["Jm"] == J and not case["tag_shared"] and not acc and div == 1.0 and wt
            rc = lib.lp_glue_f32(o0.data_ptr(), o1.data_ptr(), _lib.ptr(f0), _lib.ptr(f1), fidx.data_ptr(), N, J, h, w,
                                 1 if case["flip"] else 0, Hd, Wd, det.data_ptr(), tag.data_ptr(), stream)
        else:
            rc = lib.lp_glue_scale_f32(o0.data_ptr(), o1.data_ptr(), _lib.ptr(f0), _lib.ptr(f1), fidx.data_ptr(), N, J,
                                       case["Jm"], 1 if case["tag_shared"] else 0, h, w, 1 if case["flip"] else 0, Hd,
                                       Wd, 1 if acc else 0, div, det.data_ptr(), tag.data_ptr() if wt else None, stream)
        _lib.check(rc, "glue")
    torch.cuda.synchronize()
    det_all, tag_all = det_all.cpu().numpy(), tag_all.cpu().numpy()
    assert (det_all[det.numel():].view(np.uint32) == _NAN_BITS).all(), "det written past its end"
    assert (tag_all[tag.numel():].view(np.uint32) == _NAN_BITS).all(), "tag written past its end"
    return det_all[:det.numel()].reshape(det.shape), tag_all[:tag.numel()].reshape(tag.shape)


def _assert_bits(got, exp, what):
    g, e = got.view(np.uint32), exp.view(np.uint32)
    bad = g != e
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d of %d differ; first at %s: device %r (0x%08x), emulation %r (0x%08x)" % (
            what, bad.sum(), bad.size, i, got[i], g[i], exp[i], e[i]))


@pytest.mark.parametrize("kind", ge.KINDS)
@pytest.mark.parametrize("case", ge.CASES, ids=[c["name"] for c in ge.CASES])
def test_glue_equals_emulation(case, kind):
    inputs = ge.case_inputs(case, kind, 17)
    det, tag = _run_device(case, inputs)
    ed, et = ge.run_case(case, inputs)
    _assert_bits(det, ed, "%s/%s det (%s)" % (case["name"], kind, sorted(ge.case_paths(case))))
    if any(c[4] for c in case["calls"]):
        _assert_bits(tag, et, "%s/%s tag" % (case["name"], kind))
    else:                                                 # tag == NULL on every call: the buffer stays untouched
        assert et is None and (tag.view(np.uint32) == _NAN_BITS).all()


def test_glue_entry_points_agree():
    """lp_glue_f32 equals lp_glue_scale_f32 on the canonical layout (per-joint tags, no accumulation), with and
    without flip, on the x4, generic and unprojected geometries"""
    for flip in (True, False):
        for h, w, Hd, Wd in ((16, 16, 64, 64), (16, 24, 61, 93), (16, 24, 32, 48)):
            outs = []
            for entry in ("f32", "scale"):
                case = ge._case("entry", 2, 14, h, w, Hd, Wd, flip=flip, entry=entry)
                outs.append(_run_device(case, ge.case_inputs(case, "randn", 5)))
            for a, b in zip(*outs):
                _assert_bits(a, b, "entry points %s %s" % (flip, (h, w, Hd, Wd)))


def test_fmul_d4_rounds_once():
    """glue_x4_kernel's FMUL.D4 (the halving of (up + o1) folded into proj4's 0.25 * m[3]) on sums whose eighth is
    an fp32 subnormal with a remainder: one rounding (s / 8) and two (s / 2, then / 4) give different bits there, and
    the device agrees with glue_emul.D4_ROUNDS_ONCE.  The other paths of the x4 kernel are unaffected."""
    case = ge._case("d4", 1, 14, 4, 4, 16, 16)
    rng = np.random.default_rng(9)
    o0 = np.zeros((1, 28, 4, 4), np.float32)
    f0 = np.zeros_like(o0)
    # o1 alone reaches the mid rows: s = 0 + o1, with o1 odd multiples of the smallest subnormal
    o1 = (rng.integers(0, 1 << 12, (1, 14, 8, 8)) * 2 + 1).astype(np.float32) * np.float32(2.0 ** -149)
    f1 = (rng.integers(0, 1 << 12, (1, 14, 8, 8)) * 2 + 1).astype(np.float32) * np.float32(2.0 ** -149)
    det, _ = _run_device(case, [[o0, o1, f0, f1]])
    once, twice = [], []
    for flag, out in ((True, once), (False, twice)):
        old = ge.D4_ROUNDS_ONCE
        ge.D4_ROUNDS_ONCE = flag
        try:
            out.append(ge.run_case(case, [[o0, o1, f0, f1]])[0])
        finally:
            ge.D4_ROUNDS_ONCE = old
    assert not np.array_equal(once[0].view(np.uint32), twice[0].view(np.uint32)), "inputs do not separate the models"
    match = "once" if np.array_equal(det.view(np.uint32), once[0].view(np.uint32)) else \
        "twice" if np.array_equal(det.view(np.uint32), twice[0].view(np.uint32)) else "neither"
    assert match == ("once" if ge.D4_ROUNDS_ONCE else "twice"), match


# ---------------------------------------------------------------- the whole step, bit for bit
def _glue_step_emul(pipe, outs, Hd, Wd, plant_cpu):
    """det / tag of one step from the network outputs ``outs`` (per scale, largest first: ([o0, o1], [f0, f1] or
    None) as float32 numpy), through glue_emul as LitePosePipeline._glue launches it, then the planted persons"""
    J, fidx = pipe.params.num_joints, pipe.fidx.cpu().tolist()
    last = len(pipe.scales) - 1
    det = tag = None
    for i, (s, (o, f)) in enumerate(zip(pipe.scales, outs)):
        f0, f1 = f if f is not None else (None, None)
        if pipe.canonical and last == 0:
            det, tag = ge.glue(o[0], o[1], f0, f1, fidx, J, Hd, Wd, entry="f32")
            continue
        if s == 1.0 and tag is None:
            tag = np.full((o[0].shape[0], 1 if pipe.tag_shared else J, Hd, Wd, 2 if f is not None else 1), np.nan,
                          np.float32)
        det, _ = ge.glue(o[0], o[1], f0, f1, fidx, J, Hd, Wd, Jm=pipe.model_joints, tag_shared=pipe.tag_shared,
                         accumulate=i > 0, divide_by=float(len(pipe.scales)) if i == last else 1.0, det=det,
                         tag=tag if s == 1.0 else None, write_tag=s == 1.0)
    det_t, tag_t = torch.from_numpy(det), torch.from_numpy(tag)
    if plant_cpu is not None:
        plant_cpu.apply(det_t, tag_t)
    return det_t.numpy(), tag_t.numpy()


def _emul_outs(forward, frames, flip):
    """([o0, o1], [f0, f1]) of the network restatement ``forward(x, flip)`` on fp16 frames"""
    x = frames.half().numpy()
    return forward(x, False), (forward(x, True) if flip else None)


def _assert_step(pipe, cfg, got, st, det_e, tag_e, J):
    """the step's maps equal the restatement as bits, and its keypoints / scores are group_ref's on those maps"""
    _assert_bits(st["det"].cpu().numpy(), det_e, "step det")
    _assert_bits(st["tag"].cpu().numpy(), tag_e, "step tag")
    from oracle import group_ref
    op = group_ref.HeatmapParser(cfg)
    found = 0
    for i in range(det_e.shape[0]):
        ans, scores = op.parse(det_e[i:i + 1].copy(), tag_e[i:i + 1].copy(), cfg.TEST.ADJUST, cfg.TEST.REFINE)
        e = np.asarray(ans[0], np.float32).reshape(-1, J, 3 + tag_e.shape[-1])
        assert got[i][2] == e.shape[0], i
        assert np.array_equal(got[i][0], e), i
        assert np.array_equal(np.asarray(got[i][1], np.float32), np.asarray(scores, np.float32)), i
        found += e.shape[0]
    assert found >= det_e.shape[0]


def _xs_model(cfg, module="pose_mobilenet", name="XS"):
    import importlib
    from litepose_b200 import synth
    from litepose_b200.config import get_arch
    get_pose_net = importlib.import_module("litepose_b200.lib.models." + module).get_pose_net
    arch = get_arch(name)
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, arch), 1)).eval()
    return model, arch, {k: v.float().clone() for k, v in model.state_dict().items()}


def test_step_bench_geometry_exact():
    """The bench geometry (LitePose-S 512^2, flip, PROJECT2IMAGE, adjust + refine, 5 planted persons), batch 2: the
    det / tag the parser reads equal glue_emul of the engine's two passes on the same frames + the CPU PlantedCrowd
    bit for bit (the x4 path at the bench's per-image shape), and the returned keypoints and scores are group_ref's on
    those CPU maps.  The engine's forward is the one LitePoseEngine.run computes; net_emul restates it exactly at
    the 128-pixel shapes of test_gpu_mma_exact and in the XS steps below (S at 512 costs minutes per pass on the CPU)."""
    from litepose_b200 import synth
    from litepose_b200.config import get_cfg
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    n, size = 2, 512
    cfg = get_cfg(input_size=size)
    model, _, _ = _xs_model(cfg, name="S")
    frames = synth.make_frames(n, size, seed=1234)
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True)
    plant_dev = PlantedCrowd(n, 14, size, size, 2, num_people=5, seed=77, device="cuda")
    plant_cpu = PlantedCrowd(n, 14, size, size, 2, num_people=5, seed=77, device="cpu")
    got = pipe.step(frames.half().pin_memory(), plant_dev)
    st = pipe._get_state(n, size, size, torch.float16, plant_dev)
    det_g, tag_g = st["det"].clone(), st["tag"].clone()
    x = frames.half().cuda()
    run = lambda flip: [t.float().cpu().numpy() for t in pipe.engine.run(x, flip=flip, out_fp32=True)]
    outs = [(run(False), run(True))]
    assert ge.glue_path(n, 14, size // 4, size // 4, size, size, entry="f32") == "x4"
    det_e, tag_e = _glue_step_emul(pipe, outs, size, size, plant_cpu)
    _assert_step(pipe, cfg, got, {"det": det_g, "tag": tag_g}, det_e, tag_e, 14)


def test_step_xs_net_emul_exact():
    """LitePose-XS 128^2, batch 2, flip + PROJECT2IMAGE: step's maps = glue_emul(net_emul(x), net_emul(x, flip=True))
    + plant bit for bit; keypoints and scores = group_ref on them."""
    import net_emul
    from litepose_b200 import synth
    from litepose_b200.config import get_cfg
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    n, size = 2, 128
    cfg = get_cfg(input_size=size)
    model, arch, sd = _xs_model(cfg)
    frames = synth.make_frames(n, size, seed=21)
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True)
    plants = [PlantedCrowd(n, 14, size, size, 2, num_people=4, seed=12, device=d) for d in ("cuda", "cpu")]
    got = pipe.step(frames.half().pin_memory(), plants[0])
    st = pipe._get_state(n, size, size, torch.float16, plants[0])
    outs = [_emul_outs(lambda x, fl: net_emul.forward(sd, arch, x, fl, True), frames, True)]
    _assert_step(pipe, cfg, got, st, *_glue_step_emul(pipe, outs, size, size, plants[1]), 14)


def test_step_multiscale_net_emul_exact():
    """step_multiscale, XS at 128 with TEST.SCALE_FACTOR [0.5, 1, 2] (generic branch: accumulate, divide_by on the
    last launch, tags of scale 1 only), batch 1, bit for bit against the restatement, keypoints = group_ref."""
    import net_emul
    from litepose_b200 import synth
    from litepose_b200.config import get_cfg
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    n, size, scales = 1, 128, [0.5, 1, 2]
    cfg = get_cfg(input_size=size)
    cfg.TEST.SCALE_FACTOR = list(scales)
    model, arch, sd = _xs_model(cfg)
    frames = {float(s): synth.make_frames(n, int(size * s), seed=40 + i) for i, s in enumerate(scales)}
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True)
    plants = [PlantedCrowd(n, 14, size, size, 2, num_people=3, seed=9, device=d) for d in ("cuda", "cpu")]
    got = pipe.step_multiscale({s: f.half().pin_memory() for s, f in frames.items()}, plants[0])
    st = pipe._get_state(n, size, size, torch.float16, plants[0], det_hw=(size, size))
    fwd = lambda x, fl: net_emul.forward(sd, arch, x, fl, True)
    outs = [_emul_outs(fwd, frames[s], True) for s in pipe.scales]
    _assert_step(pipe, cfg, got, st, *_glue_step_emul(pipe, outs, size, size, plants[1]), 14)


def test_step_center_ignored_quad_exact():
    """DATASET.WITH_CENTER with the centre joint ignored (15-joint heads, 14 joints parsed): the glue takes the quad
    branch; XS at 128, batch 2, bit for bit against the restatement, keypoints = group_ref."""
    import net_emul
    from litepose_b200 import synth
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    from oracle.make_golden import glue_cfg
    n, size = 2, 128
    cfg = glue_cfg(True, True, True, True, size=size)
    model, arch, sd = _xs_model(cfg)
    frames = synth.make_frames(n, size, seed=21)
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True)
    J = pipe.params.num_joints
    assert J == 14 and pipe.model_joints == 15 and not pipe.canonical
    assert ge.glue_path(n, J, size // 4, size // 4, size, size, Jm=15) == "quad"
    plants = [PlantedCrowd(n, J, size, size, 2, num_people=3, seed=12, device=d) for d in ("cuda", "cpu")]
    got = pipe.step(frames.half().pin_memory(), plants[0])
    st = pipe._get_state(n, size, size, torch.float16, plants[0])
    outs = [_emul_outs(lambda x, fl: net_emul.forward(sd, arch, x, fl, True), frames, True)]
    _assert_step(pipe, cfg, got, st, *_glue_step_emul(pipe, outs, size, size, plants[1]), J)


def test_step_simplenet_exact():
    """One pose_simplenet step (XS at 128, batch 2): maps = glue_emul(simplenet_emul) + plant bit for bit,
    keypoints = group_ref."""
    import simplenet_emul
    from litepose_b200 import synth
    from litepose_b200.config import get_cfg
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    n, size = 2, 128
    cfg = get_cfg(input_size=size)
    model, arch, sd = _xs_model(cfg, "pose_simplenet")
    frames = synth.make_frames(n, size, seed=5)
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True)
    plants = [PlantedCrowd(n, 14, size, size, 2, num_people=4, seed=3, device=d) for d in ("cuda", "cpu")]
    got = pipe.step(frames.half().pin_memory(), plants[0])
    st = pipe._get_state(n, size, size, torch.float16, plants[0])
    outs = [_emul_outs(lambda x, fl: simplenet_emul.forward(sd, arch, x, fl, True), frames, True)]
    _assert_step(pipe, cfg, got, st, *_glue_step_emul(pipe, outs, size, size, plants[1]), 14)


def test_step_fast_grouping_exact():
    """grouping="fast": the step's maps equal the restatement bit for bit, and where build() compiled the reference's
    own find_peaks.cpp / assign.cpp (oracle/_ref/), the payload equals it on the emulated maps."""
    import net_emul
    from litepose_b200 import synth
    from litepose_b200.pipeline import LitePosePipeline
    from oracle import fast_utils_ref as fu
    from test_gpu_fast_pipeline import THR, WIN, _fast_cfg, _plant
    n, size = 2, 128
    cfg = _fast_cfg(size)
    model, arch, sd = _xs_model(cfg)
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True, grouping="fast")
    plant = _plant(pipe, n, size, size, 5, seed=31)
    plant_cpu = _plant(pipe, n, size, size, 5, seed=31)
    plant_cpu.didx, plant_cpu.dval = plant_cpu.didx.cpu(), plant_cpu.dval.cpu()
    plant_cpu.tidx, plant_cpu.tval = plant_cpu.tidx.cpu(), plant_cpu.tval.cpu()
    frames = synth.make_frames(n, size, seed=13)
    got = pipe.step(frames.half().pin_memory(), plant)
    st = pipe._get_state(n, size, size, torch.float16, plant)
    outs = [_emul_outs(lambda x, fl: net_emul.forward(sd, arch, x, fl, True), frames, True)]
    det_e, tag_e = _glue_step_emul(pipe, outs, size, size, plant_cpu)
    _assert_bits(st["det"].cpu().numpy(), det_e, "fast step det")
    _assert_bits(st["tag"].cpu().numpy(), tag_e, "fast step tag")
    if not fu.available("ref"):
        pytest.skip("oracle/_ref/libfastutils_ref.so absent: the maps are checked, the payload is not")
    J = pipe.params.num_joints
    params = dict(detection_threshold=THR, window_size=WIN, max_num_people=30, tag_threshold=1.0,
                  joint_order=[j for j in pipe.params.joint_order if j < J][:J])
    for i, (num, ans, _) in enumerate(fu.parse(det_e, tag_e, params, "ref")):
        assert num >= 3 and got[i][1] == num
        assert np.array_equal(got[i][0], ans[:num]), i
