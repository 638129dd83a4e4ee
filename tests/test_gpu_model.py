"""-m gpu: the drop-in LitePose module on the sm_90a kernels against the golden
outputs of the unmodified reference (fp32) -- tolerance 2e-3*max|ref| + 1e-4 --
plus state_dict / network_to_half / deepcopy contract and a full-size batch property."""
import copy
import os

import numpy as np
import pytest
import torch

from litepose_b200 import synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models.pose_mobilenet import get_pose_net
from oracle import model_ref
from oracle.make_golden import TINY_ARCH

pytestmark = pytest.mark.gpu


def _tol(got, ref, what):
    from gpu_util import _record
    err = float(np.abs(got - ref).max())
    lim = float(2e-3 * np.abs(ref).max() + 1e-4)
    _record(what, err, lim)
    assert err <= lim, "%s: %.3e > %.3e" % (what, err, lim)
    return err


def test_tiny_golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "model_tiny.npz"))
    cfg = get_cfg(input_size=64)
    model = get_pose_net(cfg, False, TINY_ARCH)
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    x = torch.from_numpy(z["x"]).cuda()
    with torch.no_grad():
        outs = model(x)
    assert outs[0].dtype == torch.float32
    _tol(outs[0].cpu().numpy(), z["out0"], "tiny out0")
    _tol(outs[1].cpu().numpy(), z["out1"], "tiny out1")


@pytest.mark.parametrize("name,size", [("XS", 128), ("S", 128)])
def test_shipped_arch_golden(golden_dir, name, size):
    z = np.load(os.path.join(golden_dir, "model_%s_%d.npz" % (name, size)))
    cfg = get_cfg(input_size=size)
    torch.manual_seed(0)
    model = get_pose_net(cfg, False, get_arch(name))
    synth.randomize_bn_(model, 1)
    x = synth.make_frames(1, size, seed=11)
    # fp32 module on CUDA
    m32 = copy.deepcopy(model).cuda().eval()
    with torch.no_grad():
        o = m32(x.cuda())
    _tol(o[0].cpu().numpy(), z["out0"], name + " out0")
    _tol(o[1].cpu().numpy(), z["out1"], name + " out1")
    # the reference's fp16 wrapper: tofp16 -> half model with fp32 BN -> tofp32
    class tofp16(torch.nn.Module):
        def forward(self, t):
            return t.half()

    class tofp32(torch.nn.Module):
        def forward(self, t):
            return [u.float() for u in t]

    def bn_float(mod):
        if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
            mod.float()
        for c in mod.children():
            bn_float(c)
        return mod

    half = torch.nn.Sequential(tofp16(), bn_float(copy.deepcopy(model).half()), tofp32()).cuda().eval()
    with torch.no_grad():
        oh = half(x.cuda())
    assert oh[0].dtype == torch.float32
    _tol(oh[0].cpu().numpy(), z["out0"], name + " half out0")
    _tol(oh[1].cpu().numpy(), z["out1"], name + " half out1")
    # fresh tensors per call (the glue keeps the first call's outputs alive)
    with torch.no_grad():
        o2 = m32(torch.flip(x, [3]).cuda())
    assert o2[0].data_ptr() != o[0].data_ptr()
    _tol(o[0].cpu().numpy(), z["out0"], name + " out0 still intact")


def test_flip_forward_equals_flipped_input():
    cfg = get_cfg(input_size=128)
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(cfg, False, get_arch("XS")), 1).cuda().eval()
    x = synth.make_frames(2, 128, seed=5).cuda()
    eng = model.lp_engine()
    a = eng.run(torch.flip(x, [3]).contiguous(), flip=False)
    b = eng.run(x, flip=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_batch_independence_full_size():
    """size-independent property at the benchmark shape: a frame's output does not depend on its
    batch neighbours (S @ 512x512, N = 4 vs N = 1), and CUDA graphs replay bit-identically."""
    cfg = get_cfg(input_size=512)
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(cfg, False, get_arch("S")), 1).cuda().eval()
    x = synth.make_frames(4, 512, seed=9).cuda().half()
    eng = model.lp_engine()
    full = eng.run(x)
    one = eng.run(x[2:3].contiguous())
    assert torch.equal(full[0][2:3], one[0]) and torch.equal(full[1][2:3], one[1])
    assert torch.isfinite(full[0]).all() and torch.isfinite(full[1]).all()
    eng.use_graphs = True
    g1 = eng.run(x)
    g2 = eng.run(x)
    eng.use_graphs = False
    assert torch.equal(g1[0], full[0]) and torch.equal(g2[1], full[1])
    # against the fp32 oracle on one frame
    with torch.no_grad():
        ref = model_ref.forward({k: v.cpu() for k, v in model.state_dict().items()}, get_arch("S"), x[2:3].float().cpu())
    _tol(one[0].cpu().numpy(), ref[0].numpy(), "S512 out0")
    _tol(one[1].cpu().numpy(), ref[1].numpy(), "S512 out1")


@pytest.mark.parametrize("name,size", [("M", 512), ("L", 640), ("XS", 448)])
def test_baseline_config_archs_vs_oracle(name, size):
    """BASELINE configs 2, 4 and 5 (LitePose-XS @448, -M @512, -L @640): one frame through the fp16 engine (plain and
    mirrored pass) against the fp32 oracle forward (reference lib/models/pose_mobilenet.py:137-156)."""
    cfg = get_cfg(input_size=size)
    arch = get_arch(name)
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(cfg, False, arch), 1).eval()
    x = synth.make_frames(1, size, seed=21)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    with torch.no_grad():
        ref = model_ref.forward(sd, arch, x)
        ref_f = model_ref.forward(sd, arch, torch.flip(x, [3]))
    eng = model.cuda().lp_engine()
    got = eng.run(x.cuda().half(), flip=False)
    got_f = eng.run(x.cuda().half(), flip=True)
    for i in range(2):
        _tol(got[i].cpu().numpy(), ref[i].numpy(), "%s@%d out%d" % (name, size, i))
        _tol(got_f[i].cpu().numpy(), ref_f[i].numpy(), "%s@%d flip out%d" % (name, size, i))


@pytest.mark.parametrize("name,size", [("XS", 128), ("S", 128)])
def test_shipped_arch_golden_fp16_rowsum_depthwise(golden_dir, name, size):
    """the packed-fp16 row-sum depthwise mode (lp_set_dw_precision(1)) must stay inside the same tolerance"""
    from litepose_b200 import _lib
    lib = _lib.load()
    z = np.load(os.path.join(golden_dir, "model_%s_%d.npz" % (name, size)))
    cfg = get_cfg(input_size=size)
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(cfg, False, get_arch(name)), 1).cuda().eval()
    x = synth.make_frames(1, size, seed=11).cuda()
    lib.lp_set_dw_precision(1)
    try:
        with torch.no_grad():
            o = model(x)
    finally:
        lib.lp_set_dw_precision(-1)
    _tol(o[0].cpu().numpy(), z["out0"], name + " prec1 out0")
    _tol(o[1].cpu().numpy(), z["out1"], name + " prec1 out1")


def test_folded_checkpoint_engine_matches(tmp_path):
    """engine built from the offline folded checkpoint == engine built from the state_dict (bit for bit)"""
    from litepose_b200.engine import LitePoseEngine
    cfg = get_cfg(input_size=128)
    arch = get_arch("XS")
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(cfg, False, arch), 1).eval()
    x = synth.make_frames(2, 128, seed=11).cuda().half()
    a = LitePoseEngine(model.state_dict(), arch, "cuda")
    path = str(tmp_path / "m.folded.npz")
    LitePoseEngine(model.state_dict(), arch, "cpu").export_folded(path)       # converted without a GPU
    b = LitePoseEngine.from_folded(path, "cuda")
    for flip in (False, True):
        oa = a.run(x, flip=flip, out_fp32=True, clone=True)
        ob = b.run(x, flip=flip, out_fp32=True, clone=True)
        for u, v in zip(oa, ob):
            assert torch.equal(u, v)


def test_pipeline_final_preds_on_device():
    """valid.py:230-233 inside the step: keypoints mapped back to the original image by the device kernel equal the
    oracle parser's keypoints pushed through the host get_final_preds (reference arithmetic)."""
    from litepose_b200.lib.utils import transforms as T
    from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd
    cfg = get_cfg(input_size=128)
    arch = get_arch("XS")
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, arch), 1)).eval().cuda()
    n = 3
    frames = synth.make_frames(n, 128, seed=5).half().pin_memory()
    plant = PlantedCrowd(n, 14, 128, 128, 2, num_people=3, seed=4, device="cuda")
    pipe = LitePosePipeline(model, cfg, use_graphs=True)
    plain = pipe.step(frames, plant)                          # heat-map coordinates
    sizes = [(480, 640), (640, 427), (333, 500)]              # original (h, w) of the three images
    cs = [T.get_multi_scale_size(np.zeros((h, w, 3), np.uint8), 128, 1.0, 1.0)[1:] for h, w in sizes]
    pipe.set_final_preds([c for c, _ in cs], [s for _, s in cs])
    for _ in range(2):                                        # second call replays the captured graph
        mapped = pipe.step(frames, plant)
    for i in range(n):
        a, b = plain[i], mapped[i]
        assert a[2] == b[2] and a[2] > 0
        exp = T.get_final_preds([list(a[0])], cs[i][0], cs[i][1], [128, 128])
        assert np.array_equal(np.stack(exp), b[0])
    pipe.set_final_preds(None)
    again = pipe.step(frames, plant)
    assert all(np.array_equal(x[0], y[0]) for x, y in zip(plain, again))


def test_forward_from_a_fresh_thread():
    """nn.DataParallel (reference valid.py:165) calls forward from worker threads.  A thread that has made no CUDA
    runtime call yet has no driver context bound, and the first entry point of the forward (the fused stem) builds a
    tensor map through a driver call: the library binds the primary context itself.  One device is enough to see it."""
    import threading
    cfg = get_cfg(input_size=128)
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(cfg, False, get_arch("XS")), 1).cuda().eval()
    x = synth.make_frames(2, 128, seed=3).cuda()
    with torch.no_grad():
        ref = model(x)                         # engine and plan are built here: the thread's first CUDA work is the library's
    box = {}

    def work():
        try:
            with torch.no_grad():
                box["out"] = model(x)
            torch.cuda.synchronize()
        except Exception as e:                 # surfaced in the main thread below
            box["err"] = e

    t = threading.Thread(target=work)
    t.start()
    t.join()
    assert "err" not in box, box.get("err")
    for a, b in zip(ref, box["out"]):
        assert torch.equal(a, b)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (nn.DataParallel over device_ids (0, 1))")
def test_dataparallel_two_devices():
    """reference valid.py:165 wraps the model in nn.DataParallel: replicas run on threads and share the drop-in module's
    engine cache (one engine per device, lookups under a lock); outputs equal the single-device forward bit for bit."""
    cfg = get_cfg(input_size=128)
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(cfg, False, get_arch("XS")), 1).cuda(0).eval()
    x = synth.make_frames(6, 128, seed=3).cuda(0)
    with torch.no_grad():
        single = model(x)
        dp = torch.nn.DataParallel(model, device_ids=[0, 1])
        for _ in range(3):                      # replicas are re-created every call; engines are reused per device
            multi = dp(x)
    assert len(model._lp_cache.engines) == 2
    for a, b in zip(single, multi):
        assert b.device.index == 0 and torch.equal(a, b)
    # invalidation reaches the replicas: an in-place weight update on the master changes both halves of the batch
    with torch.no_grad():
        model.first[0][0].weight.mul_(1.5)
        again = dp(x)
        ref = model(x)
    for a, b, old in zip(ref, again, multi):
        assert torch.equal(a, b) and not torch.equal(b, old)
