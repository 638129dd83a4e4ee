"""-m gpu: pose_simplenet (LitePose without the fusion head) on the sm_90a kernels.

(a) The single-branch fusion deconv (Cw = 0, raw NULL) on the row kernel and on the tiled kernel equals
    simplenet_emul.deconv_single value for value, on the plan shapes of LitePose-XS/S/M/L simplenet at 128, 256 and 512 and
    on odd H / W, Cr and Co.
(b) The single-branch unfused head (lp_head_pw_dual_f16 with C2 = 0) equals simplenet_emul.head_single, and the fused head
    (lp_head_fused_f16 with C2 = 0) equals that unfused chain (lp_dwconv_f16 k5, ReLU, then lp_head_pw_dual_f16).
(c) LitePoseEngine.run on the simplenet state dict equals simplenet_emul.forward bit for bit (every intermediate tensor
    too), the mirrored pass equals the forward of the flipped input, the module's outputs are within
    2e-3 max|ref| + 1e-4 of the reference's fp32 goldens, and a folded-checkpoint engine equals the state-dict engine.
(d) LitePosePipeline on the simplenet module: step parses exactly what the oracle parser gives on the device maps, and
    those maps are the oracle glue of the oracle forward within tolerance; the other entry points agree with step; a
    mixed-size infer_images list equals one batch-1 call per image with both groupings."""
import os

import numpy as np
import pytest
import torch

import conv_ref as cr
import dw_emul as de
import simplenet_emul as se
from gpu_util import stream
from litepose_b200 import _lib, engine, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models.pose_simplenet import get_pose_net

pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def assert_equal_values(got, want, what):
    got = np.asarray(got)
    assert got.shape == np.shape(want), (what, got.shape, np.shape(want))
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    neq = got != want
    assert not neq.any(), "%s: %d of %d elements differ (first at %s: %r vs %r)" % (
        what, neq.sum(), neq.size, np.argwhere(neq)[0], got[neq][0], np.asarray(want)[neq][0])


@pytest.fixture(autouse=True)
def default_dw_precision():
    _lib.load().lp_set_dw_precision(-1)
    yield
    _lib.load().lp_set_dw_precision(-1)


def _model(name, size):
    torch.manual_seed(0)
    return synth.randomize_bn_(get_pose_net(get_cfg(input_size=size), False, get_arch(name)), 1).eval()


_plan_cache = {}


def _plan(name, size):
    if (name, size) not in _plan_cache:
        eng = engine.LitePoseEngine(_model(name, size).state_dict(), get_arch(name), "cpu")
        _plan_cache[(name, size)] = eng._build_plan(1, size, size, torch.float16, True, alloc=engine._Bump())["ops"]
    return _plan_cache[(name, size)]


PLAN = [(a, s) for a in ("XS", "S", "M", "L") for s in (128, 256, 512)]


def _plan_deconv_shapes():
    out = set()
    for a, s in PLAN:
        for op in _plan(a, s):
            if op.name == "deconv":
                assert op.args[1] is None and op.args[9] == 0
                out.add(tuple(op.args[5:9]) + (op.args[10],))     # n, h, w, Cr, Co
    return sorted(out)


def _plan_head_shapes():
    out = set()
    for a, s in PLAN:
        for op in _plan(a, s):
            if op.name == "head_fused":
                assert op.args[1] is None and op.args[11] == 0
                out.add(tuple(op.args[7:11]) + (op.args[12],))    # n, h, w, C1, Co
    return sorted(out)


# ---------------------------------------------------------------- (a) single-branch deconv
DECONV_ODD = [
    # (n, h, w, cr, co)
    (1, 3, 65, 24, 8),          # W = 65: row kernel, one partial strip; Cr = 24: K = 32 with 8 zero channels
    (2, 5, 130, 40, 24),        # Cr = 40: odd chunk count (5), K = 48; a 2-pixel second strip
    (1, 7, 200, 8, 32),         # Cr = 8: one chunk; Co = 32, the widest the row kernel takes
    (3, 9, 11, 56, 16),         # tiled: odd H and W
    (1, 6, 100, 24, 40),        # tiled although wide: Co = 40
    (2, 5, 13, 136, 56),        # tiled: Cr = 136, three K blocks, the last of 8 channels; Co = 56
    (1, 4, 70, 72, 8),          # tiled although wide: Cr = 72 > 64
]


def _run_deconv(n, h, w, crr, co, seed):
    lib = _lib.load()
    xr, _, wr, _, b = cr.deconv_inputs(n, h, w, crr, 0, co, seed)
    wp = np.zeros(lib.lp_deconv_packed_elems(crr, 0, co), np.uint16)
    bp = np.zeros(lib.lp_deconv_packed_bias_elems(co), np.float32)
    _lib.check(lib.lp_deconv_pack(wr.view(np.uint16).ctypes.data, None, b.ctypes.data, crr, 0, co, wp.ctypes.data,
                                  bp.ctypes.data), "deconv_pack")
    wd, bd, rd = _dev(wp.view(np.float16)), _dev(bp), _dev(xr)
    out = torch.full((n, 2 * h, 2 * w, co), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_fusion_deconv_f16(rd.data_ptr(), None, wd.data_ptr(), bd.data_ptr(), out.data_ptr(), n, h, w,
                                        crr, 0, co, stream()), "deconv")
    torch.cuda.synchronize()
    rows = cr.uses_rows_kernel(crr, 0, co, w)
    want = se.deconv_single(xr, wr, b, rows)
    assert_equal_values(out.cpu().numpy(), want, "deconv_single %s n%d %dx%d cr%d co%d"
                        % ("rows" if rows else "tiled", n, h, w, crr, co))
    return rows


@pytest.mark.parametrize("n,h,w,crr,co", DECONV_ODD)
def test_deconv_single_odd_shapes(n, h, w, crr, co):
    _run_deconv(n, h, w, crr, co, n + h * 3 + w * 5 + crr + co)


def test_deconv_single_plan_shapes():
    kinds = set()
    for n, h, w, crr, co in _plan_deconv_shapes():
        kinds.add(_run_deconv(n, h, w, crr, co, h + crr + co))
    assert kinds == {True, False}, "the plan shapes cover both deconv kernels"


# ---------------------------------------------------------------- (b) single-branch heads
HEAD_ODD = [
    # (n, h, w, c1, co, fp32)
    (2, 17, 23, 24, 28, True),    # one partial slab; ragged 16x16 tiles
    (1, 9, 40, 40, 14, False),    # two slabs, the second partial (K block of 1.25 slabs)
    (3, 5, 5, 8, 17, True),       # Co = 17: a partial n_tile, odd
    (1, 33, 31, 72, 120, False),  # three slabs; Co = 120
]


def _run_head(n, h, w, c1, co, fp32, seed):
    lib = _lib.load()
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, h, w, c1)).astype(np.float16)
    dw = (rng.standard_normal((25, c1)) * 0.2).astype(np.float16)
    bdw = (rng.standard_normal(c1) * 0.1).astype(np.float32)
    w1 = (rng.standard_normal((co, c1)) / c1 ** 0.5).astype(np.float16)
    odt = torch.float32 if fp32 else torch.float16
    xd, dwd, bdwd = _dev(x), _dev(dw), _dev(bdw)
    # fused, single branch
    dwc = np.zeros(lib.lp_head_fused_dw_elems(c1, 0), np.uint16)
    bdc = np.zeros(dwc.size // 25, np.float32)
    pwc = np.zeros(lib.lp_head_fused_pw_elems(c1, 0, co), np.uint16)
    _lib.check(lib.lp_head_fused_pack(dw.view(np.uint16).ctypes.data, bdw.ctypes.data, None, None,
                                      w1.view(np.uint16).ctypes.data, None, c1, 0, co, dwc.ctypes.data,
                                      bdc.ctypes.data, pwc.ctypes.data), "head_fused_pack")
    assert dwc.size == 25 * ((c1 + 31) // 32) * 32
    fused = torch.full((n, co, h, w), float("nan"), dtype=odt, device="cuda")
    pd, bd, wcd = _dev(dwc.view(np.float16)), _dev(bdc), _dev(pwc.view(np.float16))
    _lib.check(lib.lp_head_fused_f16(xd.data_ptr(), None, pd.data_ptr(), bd.data_ptr(), wcd.data_ptr(),
                                     fused.data_ptr(), 1 if fp32 else 0, n, h, w, c1, 0, co, stream()), "head_fused")
    # the unfused chain: depthwise 5x5 + ReLU, then the single-branch head GEMM
    t = torch.full((n, h, w, c1), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_dwconv_f16(xd.data_ptr(), dwd.data_ptr(), bdwd.data_ptr(), t.data_ptr(), n, c1, h, w, 5, 1,
                                 de.ACT_RELU, stream()), "dwconv")
    wp = np.zeros(lib.lp_head_packed_elems(c1, 0, co), np.uint16)
    _lib.check(lib.lp_head_pack(w1.view(np.uint16).ctypes.data, None, c1, 0, co, wp.ctypes.data), "head_pack")
    wpd = _dev(wp.view(np.float16))
    chain = torch.full((n, co, h, w), float("nan"), dtype=odt, device="cuda")
    _lib.check(lib.lp_head_pw_dual_f16(t.data_ptr(), None, wpd.data_ptr(), chain.data_ptr(), 1 if fp32 else 0, n, h,
                                       w, c1, 0, co, stream()), "head_pw_dual")
    torch.cuda.synchronize()
    what = "head_single n%d %dx%d c1 %d co %d fp32 %d" % (n, h, w, c1, co, fp32)
    t = t.cpu().numpy()
    assert_equal_values(t, de.dwconv(x, dw, bdw, 5, 1, de.ACT_RELU, de.default_prec(5)), what + " dwconv vs dw_emul")
    want = se.head_single(t.reshape(-1, c1), w1, fp32).reshape(n, h, w, co).transpose(0, 3, 1, 2)
    assert_equal_values(chain.cpu().numpy(), want, what + " unfused vs simplenet_emul")
    assert_equal_values(fused.cpu().numpy(), chain.cpu().numpy(), what + " fused vs unfused")


@pytest.mark.parametrize("n,h,w,c1,co,fp32", HEAD_ODD)
def test_head_single_odd_shapes(n, h, w, c1, co, fp32):
    _run_head(n, h, w, c1, co, fp32, n + h + w + c1 + co)


@pytest.mark.parametrize("fp32", [True, False])
def test_head_single_plan_shapes(fp32):
    for n, h, w, c1, co in _plan_head_shapes():
        _run_head(n, h, w, c1, co, fp32, h + c1 + co + fp32)


# ---------------------------------------------------------------- (c) the engine
# (the emulation of one S 512 batch-2 forward takes minutes on the CPU: that shape runs with one output dtype)
ENGINE_CASES = [("XS", 1, 128, "fp16", True), ("S", 1, 128, "fp32", True), ("S", 2, 512, "fp16", True),
                ("XS", 2, 128, "fp32", False)]


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("name,n,size,dt,out_fp32", ENGINE_CASES)
def test_engine_equals_simplenet_emul(name, n, size, dt, out_fp32, flip):
    arch = get_arch(name)
    sd = {k: v.clone() for k, v in _model(name, size).state_dict().items()}
    x = synth.make_frames(n, size, seed=size + n)
    x = x.half() if dt == "fp16" else x
    eng = engine.LitePoseEngine(sd, arch, "cuda")
    assert eng.topology == engine.SIMPLE
    got = eng.run(x.cuda(), flip=flip, out_fp32=out_fp32)
    torch.cuda.synchronize()
    plan = next(iter(eng.plans.values()))
    keep = plan["keep"]
    fused_stem = any(op.name == "stem_fused" for op in plan["ops"])
    inner = [keep[0]] + [t for t in keep[1 if fused_stem else 3:] if t.dim() == 4]
    trace = []
    want = se.forward(sd, arch, x.numpy(), flip, out_fp32, trace)
    assert len(inner) == len(trace)
    case = "%s n%d %d %s out_fp32 %d flip %d" % (name, n, size, dt, out_fp32, flip)
    for t, (nm, wt) in zip(inner, trace):
        assert_equal_values(t.cpu().numpy(), wt, "%s %s" % (case, nm))
    for i, (g, wt) in enumerate(zip(got, want)):
        g = g.cpu().numpy()
        assert g.dtype == (np.float32 if out_fp32 else np.float16)
        assert_equal_values(g, wt, "%s output %d" % (case, i))


def test_mirrored_pass_equals_flipped_input():
    model = _model("S", 256).cuda()
    eng = model.lp_engine()
    assert eng.topology == engine.SIMPLE
    x = synth.make_frames(2, 256, seed=5).cuda().half()
    a = eng.run(torch.flip(x, [3]).contiguous(), flip=False)
    b = eng.run(x, flip=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("name", ["XS", "S"])
def test_outputs_within_tolerance_of_reference_golden(golden_dir, name):
    z = np.load(os.path.join(golden_dir, "model_simplenet_%s_128.npz" % name))
    model = _model(name, 128).cuda()
    x = synth.make_frames(1, 128, seed=11).cuda()
    with torch.no_grad():
        outs = [model(x), model(x.half())]
    for o in outs:
        for g, k in zip(o, ("out0", "out1")):
            err = np.abs(g.float().cpu().numpy() - z[k]).max()
            lim = 2e-3 * np.abs(z[k]).max() + 1e-4
            assert err <= lim, "%s %s: %.3e > %.3e" % (name, k, err, lim)


def test_folded_checkpoint_engine_matches(tmp_path):
    sd = _model("XS", 128).state_dict()
    arch = get_arch("XS")
    x = synth.make_frames(2, 128, seed=11).cuda().half()
    a = engine.LitePoseEngine(sd, arch, "cuda")
    path = str(tmp_path / "simple.folded.npz")
    engine.LitePoseEngine(sd, arch, "cpu").export_folded(path)
    b = engine.LitePoseEngine.from_folded(path, "cuda")
    assert b.topology == engine.SIMPLE
    for flip in (False, True):
        for u, v in zip(a.run(x, flip=flip), b.run(x, flip=flip)):
            assert torch.equal(u, v)


# ---------------------------------------------------------------- (d) the pipeline
def _pipeline_model(name, size):
    torch.manual_seed(0)
    cfg = get_cfg(input_size=size)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch(name)), 1)).eval()
    return cfg, model


def test_pipeline_entry_points_vs_oracle():
    from oracle import glue_ref, group_ref
    from oracle import model_ref_simplenet
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    n, size = 2, 256
    cfg, model = _pipeline_model("S", size)
    arch = get_arch("S")
    sd = {k: v.float().clone() for k, v in model.state_dict().items()}
    frames = synth.make_frames(n, size, seed=1234)
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True)
    plant_dev = PlantedCrowd(n, 14, size, size, 2, num_people=4, seed=77, device="cuda")
    plant_cpu = PlantedCrowd(n, 14, size, size, 2, num_people=4, seed=77, device="cpu")
    got = pipe.step(frames.half().pin_memory(), plant_dev)
    got2 = pipe.step(frames.half().pin_memory(), plant_dev)            # graph replay
    st = pipe._get_state(n, size, size, torch.float16, plant_dev)
    det_g, tag_g = st["det"].cpu().numpy(), st["tag"].cpu().numpy()
    with torch.no_grad():
        _, hm, tg = glue_ref.multi_stage_outputs(cfg, lambda im: model_ref_simplenet.forward(sd, arch, im), frames,
                                                 True, True, (size, size))
        det_o, tag_o = glue_ref.aggregate(cfg, hm, tg)
        det_o, tag_o = det_o.contiguous(), tag_o.contiguous()
        det_raw, tag_raw = det_o.clone(), tag_o.clone()
        plant_cpu.apply(det_o, tag_o)
    for nm, g, o, raw in (("det", det_g, det_o.numpy(), det_raw.numpy()), ("tag", tag_g, tag_o.numpy(), tag_raw.numpy())):
        err = np.abs(g - o).max()
        lim = 2e-3 * np.abs(raw).max() + 1e-4
        assert err <= lim, "%s: %.3e > %.3e" % (nm, err, lim)
    op = group_ref.HeatmapParser(cfg)
    found = 0
    for i in range(n):
        ans, scores = op.parse(det_g[i:i + 1].copy(), tag_g[i:i + 1].copy(), True, True)
        e = np.asarray(ans[0], np.float32).reshape(-1, 14, 5)
        for res in (got, got2):
            assert res[i][2] == e.shape[0]
            assert np.array_equal(res[i][0], e), i
            assert np.array_equal(np.asarray(res[i][1], np.float32), np.asarray(scores, np.float32))
        found += e.shape[0]
    assert found > 0

    # the asynchronous and the overlapped entry points give what step gives
    res = pipe.collect(pipe.submit(frames.half().pin_memory(), plant_dev))[0]
    assert [r[2] for r in res] == [r[2] for r in got]
    for a, b in zip(res, got):
        assert np.array_equal(a[0], b[0]) and np.array_equal(np.asarray(a[1]), np.asarray(b[1]))
    x_dev = frames.half().cuda()
    want = pipe.step_device(x_dev, plant_dev).clone()
    for _ in range(2):                               # both buffer sets of the overlapped form
        packed, ev = pipe.step_device_overlapped(x_dev, plant_dev)
        ev.synchronize()
        assert torch.equal(packed, want)


def test_multiscale_step_vs_oracle():
    from oracle import glue_ref, group_ref
    from oracle import model_ref_simplenet
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    n, size, scales = 2, 128, [0.5, 1, 2]
    cfg, model = _pipeline_model("XS", size)
    cfg.TEST.SCALE_FACTOR = list(scales)
    arch = get_arch("XS")
    sd = {k: v.float().clone() for k, v in model.state_dict().items()}
    frames = {float(s): synth.make_frames(n, int(size * s), seed=40 + i) for i, s in enumerate(scales)}
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True)
    plant_dev = PlantedCrowd(n, 14, size, size, 2, num_people=3, seed=9, device="cuda")
    plant_cpu = PlantedCrowd(n, 14, size, size, 2, num_people=3, seed=9, device="cpu")
    got = pipe.step_multiscale({s: f.half().pin_memory() for s, f in frames.items()}, plant_dev)
    st = pipe._get_state(n, size, size, torch.float16, plant_dev, det_hw=(size, size))
    det_g, tag_g = st["det"].cpu().numpy(), st["tag"].cpu().numpy()
    with torch.no_grad():
        det_o, tag_o = glue_ref.multi_scale(cfg, lambda im: model_ref_simplenet.forward(sd, arch, im), frames,
                                            (size, size))
        det_raw, tag_raw = det_o.clone(), tag_o.clone()
        det_o, tag_o = det_o.contiguous(), tag_o.contiguous()
        plant_cpu.apply(det_o, tag_o)
    for nm, g, o, raw in (("det", det_g, det_o.numpy(), det_raw.numpy()), ("tag", tag_g, tag_o.numpy(), tag_raw.numpy())):
        err = np.abs(g - o).max()
        lim = 2e-3 * np.abs(raw).max() + 1e-4
        assert err <= lim, "%s: %.3e > %.3e" % (nm, err, lim)
    op = group_ref.HeatmapParser(cfg)
    for i in range(n):
        ans, scores = op.parse(det_g[i:i + 1].copy(), tag_g[i:i + 1].copy(), True, True)
        e = np.asarray(ans[0], np.float32).reshape(-1, 14, 5)
        assert got[i][2] == e.shape[0] and np.array_equal(got[i][0], e), i


MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
SHAPES = [(150, 200), (200, 150), (100, 300), (120, 120), (201, 149)]


@pytest.mark.parametrize("grouping", ["ae", "fast"])
def test_infer_images_list_equals_one_call_per_image(grouping):
    from litepose_b200.pipeline import LitePosePipeline
    cfg, model = _pipeline_model("XS", 128)
    if grouping == "fast":                      # the demo's parser: no adjust / refine steps
        cfg.TEST.ADJUST = cfg.TEST.REFINE = False
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True, grouping=grouping)
    rng = np.random.RandomState(7)
    imgs = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in SHAPES]
    got = pipe.infer_images(imgs)
    assert len(got) == len(imgs)
    for i, im in enumerate(imgs):
        exp = pipe.infer_images(torch.from_numpy(im)[None].pin_memory())[0]
        assert got[i][-1] == exp[-1], (grouping, i)
        assert np.array_equal(got[i][0], exp[0]), (grouping, i)
