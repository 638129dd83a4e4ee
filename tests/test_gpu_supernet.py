"""-m gpu: the LitePose super-network (pose_supermobilenet) on the sm_90a kernels.

(a) The engine of every golden architecture and of 20 seeded ArchManager.random_sample() draws (64-128 px, fp16 / fp32
    input, plain / mirrored) equals supernet_emul.forward (tests/net_emul.py's arithmetic with the supernet's residual
    and stride lists) on the derived state dict, bit for bit.
(b) The module's CUDA forward is within 2e-3 max|ref| + 1e-4 of the reference's fp32 goldens.
(c) infer_images on the supernet equals infer_images on the pose_mobilenet that subnet.extract_subnet builds for a
    [6, 7] architecture, bit for bit.
(d) The engine cache: switching search_arch between forwards never returns another architecture's engine, a forward
    without is_search runs the architecture it draws, and a train-mode pass followed by eval runs the new statistics.
(e) network_to_half, single-device nn.DataParallel and folded checkpoints; LitePosePipeline binds the search
    architecture and refuses a supernet without one."""
import copy
import json
import os
import random

import numpy as np
import pytest
import torch

import supernet_emul
from litepose_b200 import _lib, engine, subnet, synth
from litepose_b200.arch_manager import ArchManager
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models import pose_supermobilenet

pytestmark = pytest.mark.gpu

GOLDENS = ["search_XS", "search_S", "fixed_256_0.5", "random_seed1", "random_seed2", "mixed"]


@pytest.fixture(autouse=True)
def default_dw_precision():
    _lib.load().lp_set_dw_precision(-1)
    yield
    _lib.load().lp_set_dw_precision(-1)


def assert_equal_values(got, want, what):
    got = np.asarray(got)
    assert got.shape == np.shape(want), (what, got.shape, np.shape(want))
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    neq = got != want
    assert not neq.any(), "%s: %d of %d elements differ (first at %s: %r vs %r)" % (
        what, neq.sum(), neq.size, np.argwhere(neq)[0], got[neq][0], np.asarray(want)[neq][0])


_sd = {}


def _supernet_sd():
    if not _sd:
        torch.manual_seed(0)
        m = synth.randomize_bn_(pose_supermobilenet.get_pose_net(get_cfg(input_size=128)), 1)
        _sd.update({k: v.detach().clone() for k, v in m.state_dict().items()})
    return _sd


def _supernet(size=128):
    m = pose_supermobilenet.get_pose_net(get_cfg(input_size=size))
    m.load_state_dict(_supernet_sd(), strict=True)
    return m.eval()


def _golden_arch(golden_dir, name):
    z = np.load(os.path.join(golden_dir, "model_supernet_%s.npz" % name))
    return z, json.loads(str(z["arch"]))


def _draws():
    """20 seeded draws, each with an input size, input dtype and pass"""
    am = ArchManager(get_cfg())
    out = []
    for i in range(20):
        random.seed(100 + i)
        out.append((am.random_sample(), (64, 96, 128)[i % 3], ("fp16", "fp32")[i % 2], bool((i // 2) % 2)))
    return out


def _check_engine(arch, size, dt, flip, what, n=1):
    sub = subnet.derive_supernet_subnet(_supernet_sd(), arch)
    eng = engine.LitePoseEngine(sub.state_dict, sub.arch, "cuda", residual=sub.residual, strides=sub.strides)
    x = synth.make_frames(n, size, seed=size + n)
    x = x.half() if dt == "fp16" else x
    out_fp32 = dt == "fp32"
    got = eng.run(x.cuda(), flip=flip, out_fp32=out_fp32)
    want = supernet_emul.forward(sub.state_dict, sub.arch, x.numpy(), flip, out_fp32,
                                 residual=sub.residual, strides=sub.strides)
    for i, (g, w) in enumerate(zip(got, want)):
        g = g.cpu().numpy()
        assert g.dtype == (np.float32 if out_fp32 else np.float16)
        assert_equal_values(g, w, "%s output %d" % (what, i))
    return eng


@pytest.mark.parametrize("name", GOLDENS)
def test_engine_equals_emulation_on_golden_archs(golden_dir, name):
    _, arch = _golden_arch(golden_dir, name)
    _check_engine(arch, 128, "fp16", False, name)
    _check_engine(arch, 96, "fp32", True, name + " mirrored")


@pytest.mark.parametrize("i", range(20))
def test_engine_equals_emulation_on_random_draws(i):
    arch, size, dt, flip = _draws()[i]
    _check_engine(arch, size, dt, flip, "draw %d" % i)


@pytest.mark.parametrize("name", GOLDENS)
def test_module_within_tolerance_of_goldens(golden_dir, name):
    z, arch = _golden_arch(golden_dir, name)
    model = _supernet().cuda()
    x = synth.make_frames(1, 128, seed=11).cuda()
    if int(z["seed"]) >= 0:     # the forward's own draw
        random.seed(int(z["seed"]))
        with torch.no_grad():
            got = model(x.half())
        assert np.array_equal(np.array(random.getstate()[1], np.int64), z["random_state"])
    else:
        model.arch_manager.is_search, model.arch_manager.search_arch = True, arch
        with torch.no_grad():
            got = model(x.half())
    for g, k in zip(got, ("out0", "out1")):
        err = np.abs(g.float().cpu().numpy() - z[k]).max()
        assert err <= 2e-3 * np.abs(z[k]).max() + 1e-4, (name, k, err)


def test_infer_images_equals_extracted_pose_mobilenet():
    from litepose_b200.pipeline import LitePosePipeline
    cfg = get_cfg(input_size=128)
    arch = get_arch("XS")
    sup = _supernet().cuda()
    sup.arch_manager.is_search, sup.arch_manager.search_arch = True, arch
    lp = subnet.extract_subnet(_supernet_sd(), cfg, arch).cuda()
    rng = np.random.RandomState(3)
    imgs = torch.from_numpy(rng.randint(0, 256, (2, 150, 200, 3)).astype(np.uint8)).pin_memory()
    a = LitePosePipeline(sup, cfg).infer_images(imgs)
    b = LitePosePipeline(lp, cfg).infer_images(imgs)
    for (ra, sa, pa), (rb, sb, pb) in zip(a, b):
        assert pa == pb and np.array_equal(ra, rb) and np.array_equal(np.asarray(sa), np.asarray(sb))


def test_switching_search_arch_never_returns_a_stale_engine(golden_dir):
    model = _supernet().cuda()
    x = synth.make_frames(1, 64, seed=5).cuda().half()
    archs = [_golden_arch(golden_dir, n)[1] for n in ("search_XS", "mixed", "fixed_256_0.5", "search_S", "random_seed1",
                                                      "search_XS")]
    am = model.arch_manager
    am.is_search = True
    for arch in archs:
        am.search_arch = arch
        with torch.no_grad():
            got = model(x)
        want = model.lp_engine(x.device, copy.deepcopy(arch)).run(x, out_fp32=False)
        fresh = subnet.derive_supernet_subnet(model.state_dict(), arch)
        ref = engine.LitePoseEngine(fresh.state_dict, fresh.arch, "cuda", residual=fresh.residual,
                                    strides=fresh.strides).run(x, out_fp32=False)
        for g, w, r in zip(got, want, ref):
            assert torch.equal(g, w) and torch.equal(g, r)
    assert len(model._lp_cache.engines) <= pose_supermobilenet.ENGINE_LRU
    # without is_search every forward runs the architecture it draws
    am.is_search = False
    random.seed(7)
    drawn = ArchManager(get_cfg()).random_sample()
    random.seed(7)
    with torch.no_grad():
        got = model(x)
    want = model.lp_engine(x.device, drawn).run(x, out_fp32=False)
    assert all(torch.equal(g, w) for g, w in zip(got, want))


def test_train_pass_then_eval_equals_fresh_module():
    """the search's BN recalibration: train-mode forwards on synthetic batches update the prefix statistics, and the
    next eval forward runs them"""
    model = _supernet().cuda()
    arch = ArchManager(get_cfg()).fixed_sample(256, 0.75)
    model.arch_manager.is_search, model.arch_manager.search_arch = True, arch
    x = synth.make_frames(1, 64, seed=9).cuda()
    with torch.no_grad():
        before = model(x)
        model.train()
        for seed in (1, 2, 3):
            model(synth.make_frames(4, 64, seed=seed).cuda())
        model.eval()
        after = model(x)
    fresh = pose_supermobilenet.get_pose_net(get_cfg(input_size=64))
    fresh.load_state_dict(model.state_dict(), strict=True)
    fresh = fresh.cuda().eval()
    fresh.arch_manager.is_search, fresh.arch_manager.search_arch = True, arch
    with torch.no_grad():
        want = fresh(x)
    assert any(not torch.equal(a, b) for a, b in zip(before, after))
    assert all(torch.equal(a, b) for a, b in zip(after, want))


def test_network_to_half_data_parallel_and_folded(tmp_path, golden_dir):
    _, arch = _golden_arch(golden_dir, "mixed")
    model = _supernet().cuda()
    model.arch_manager.is_search, model.arch_manager.search_arch = True, arch
    x = synth.make_frames(2, 64, seed=4).cuda()
    with torch.no_grad():
        want = model(x.half())
    # network_to_half: fp16 module, fp32 BN, fp16 input (reference lib/fp16_utils/fp16util.py:87-91)
    half = copy.deepcopy(model).half()
    for m in half.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.float()
    wrapped = torch.nn.Sequential(half)
    with torch.no_grad():
        got = wrapped(x.half())
    err = max((a.float() - b.float()).abs().max().item() for a, b in zip(got, want))
    assert err <= 2e-3 * max(b.float().abs().max().item() for b in want) + 1e-4
    with torch.no_grad():
        dp = torch.nn.DataParallel(model, device_ids=[0])(x.half())
    assert all(torch.equal(a, b) for a, b in zip(dp, want))
    path = str(tmp_path / "super.folded.npz")
    eng = model.lp_engine(x.device)
    eng.export_folded(path)
    back = engine.LitePoseEngine.from_folded(path, "cuda")
    for a, b in zip(back.run(x.half(), out_fp32=False), want):
        assert torch.equal(a, b)


def test_pipeline_binds_the_search_arch_and_refuses_without_one(golden_dir):
    from litepose_b200.pipeline import LitePosePipeline
    cfg = get_cfg(input_size=128)
    model = _supernet().cuda()
    with pytest.raises(ValueError, match="is_search"):
        LitePosePipeline(model, cfg)
    _, arch = _golden_arch(golden_dir, "mixed")
    model.arch_manager.is_search, model.arch_manager.search_arch = True, arch
    pipe = LitePosePipeline(model, cfg)
    assert pipe.engine is model.lp_engine(torch.device("cuda"), arch)
    imgs = torch.from_numpy(np.random.RandomState(1).randint(0, 256, (1, 128, 128, 3)).astype(np.uint8))
    assert len(pipe.infer_images(imgs)) == 1
