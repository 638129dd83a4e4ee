"""CPU: the LitePose super-network drop-in (pose_supermobilenet) against the reference's own module through the committed
fixtures and, where the reference tree is present, directly; the restated ArchManager's draws; every rule of
subnet.derive_supernet_subnet; the engine's per-block residual / stride lists and folded export; and the drop-in's
resolution of ``models.pose_supermobilenet`` in both launch modes."""
import copy
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from litepose_b200 import engine, subnet, synth
from litepose_b200.arch_manager import ArchManager
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models import pose_mobilenet, pose_supermobilenet
from oracle import model_ref_supernet, refshim
from oracle.make_golden import sd_digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = ["search_XS", "search_S", "fixed_256_0.5", "random_seed1", "random_seed2", "mixed"]
MIXED_JSON = {"img_size": 256, "input_channel": 16, "deconv_setting": [48, 24, 16], "backbone_setting": [
    {"num_blocks": 2, "stride": 2, "channel": 24, "block_setting": [[4, 5], [3, 3]]},
    {"num_blocks": 3, "stride": 2, "channel": 32, "block_setting": [[6, 5], [6, 7], [3, 7]]},
    {"num_blocks": 2, "stride": 2, "channel": 80, "block_setting": [[6, 7], [4, 5]]},
    {"num_blocks": 3, "stride": 1, "channel": 80, "block_setting": [[6, 7], [3, 3], [6, 5]]}]}


def _supernet(size=128):
    torch.manual_seed(0)
    return synth.randomize_bn_(pose_supermobilenet.get_pose_net(get_cfg(input_size=size)), 1).eval()


def _golden(golden_dir, name):
    z = np.load(os.path.join(golden_dir, "model_supernet_%s.npz" % name))
    return z, json.loads(str(z["arch"]))


def _fwd(model, arch, x):
    model.arch_manager.is_search, model.arch_manager.search_arch = True, arch
    with torch.no_grad():
        return model(x)


def test_names_shapes_and_digest(golden_dir):
    sd = _supernet().state_dict()
    assert len(sd) == 815 and sum(".Linear5x5." in k or ".Linear3x3." in k for k in sd) == 136
    for name in GOLDENS:
        assert sd_digest(sd) == str(_golden(golden_dir, name)[0]["digest"]), name


@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_and_module_tree_equal_reference_golden(golden_dir, name):
    z, arch = _golden(golden_dir, name)
    model = _supernet()
    x = synth.make_frames(1, 128, seed=11)
    with torch.no_grad():
        outs = model_ref_supernet.forward(model.state_dict(), arch, x)
    if int(z["seed"]) >= 0:     # the forward's own draw (CPU tensor: the module tree), and the random state it leaves
        model.arch_manager.is_search = False
        random.seed(int(z["seed"]))
        with torch.no_grad():
            mods = model(x)
        assert np.array_equal(np.array(random.getstate()[1], np.int64), z["random_state"])
    else:
        mods = _fwd(model, arch, x)
    for a, m, k in zip(outs, mods, ("out0", "out1")):
        assert np.abs(a.numpy() - z[k]).max() <= 1e-5
        assert np.abs(m.numpy() - z[k]).max() <= 1e-5
        tol = 2e-3 * np.abs(z[k]).max() + 1e-4
        assert np.abs(z[k + "_fp16eager"] - z[k]).max() <= tol


@pytest.mark.skipif(not refshim.available(), reason="reference tree not present")
def test_oracle_and_module_equal_unmodified_reference():
    cfg = get_cfg(input_size=64)
    ref = model_ref_supernet.build_reference(cfg)
    ours = _supernet(64)
    assert [(k, tuple(v.shape)) for k, v in ref.state_dict().items()] == \
        [(k, tuple(v.shape)) for k, v in ours.state_dict().items()]
    assert sd_digest(ref.state_dict()) == sd_digest(ours.state_dict())
    x = synth.make_frames(2, 64, seed=3)
    random.seed(5)
    for arch in (MIXED_JSON, ArchManager(cfg).random_sample(), ArchManager(cfg).fixed_sample(320, 0.75)):
        want = _fwd(ref, arch, x)
        got = model_ref_supernet.forward(ref.state_dict(), arch, x)
        mods = _fwd(ours, arch, x)
        for a, b, c in zip(got, want, mods):
            assert (a - b).abs().max().item() == 0.0 and (c - b).abs().max().item() == 0.0


@pytest.mark.skipif(not refshim.available(), reason="reference tree not present")
def test_train_pass_and_pretrained_init_equal_reference(tmp_path):
    """the BN recalibration pass (training mode, prefix statistics) and is_train with INIT_WEIGHTS
    (re_organize_weights) leave the same tensors as the reference module"""
    cfg = get_cfg(input_size=64)
    ref = model_ref_supernet.build_reference(cfg).train()
    ours = _supernet(64).train()
    for seed in (1, 2):
        x = synth.make_frames(2, 64, seed=seed)
        random.seed(seed)
        with torch.no_grad():
            ref(x)
        random.seed(seed)
        with torch.no_grad():
            ours(x)
    for (k, a), b in zip(ref.state_dict().items(), ours.state_dict().values()):
        assert torch.equal(a, b), k
    path = str(tmp_path / "pretrained.pth")
    torch.save({"module." + k: v for k, v in ref.state_dict().items()}, path)
    cfg.MODEL.PRETRAINED = path
    psm, _ = model_ref_supernet.load_reference()
    torch.manual_seed(4)
    want = psm.get_pose_net(cfg, True).state_dict()
    torch.manual_seed(4)
    got = pose_supermobilenet.get_pose_net(cfg, True).state_dict()
    for (k, a), b in zip(want.items(), got.values()):
        assert torch.equal(a, b), k


def test_arch_manager_draws(golden_dir):
    cfg = get_cfg(input_size=128)
    am = ArchManager(cfg)
    assert (am.expansion, am.kernel_size, am.width_mult, am.is_search, am.search_arch) == \
        ([6], [7], [1.0, 0.75, 0.5, 0.25], False, None)
    assert am.arch_setting == [[32, 4, 2], [64, 6, 2], [96, 8, 2], [160, 8, 1]]
    for name in ("random_seed1", "random_seed2"):
        z, arch = _golden(golden_dir, name)
        random.seed(int(z["seed"]))
        assert am.random_sample() == arch
        assert np.array_equal(np.array(random.getstate()[1], np.int64), z["random_state"])
    assert am.fixed_sample(256, 0.5) == _golden(golden_dir, "fixed_256_0.5")[1]
    am.is_search, am.search_arch = True, {"x": 1}
    state = random.getstate()
    assert am.random_sample() == {"x": 1} and random.getstate() == state
    if refshim.available():
        _, ref_am = model_ref_supernet.load_reference()
        ref = ref_am.ArchManager(cfg)
        for seed in range(40):
            random.seed(seed)
            a = ArchManager(cfg).random_sample()
            sa = random.getstate()
            random.seed(seed)
            assert ref.random_sample() == a and random.getstate() == sa
            assert ref.rand_kernel_size() == ArchManager(cfg).rand_kernel_size() == 7
        for reso, ratio in ((256, 0.5), (512, 1.0), (384, 0.25), (448, 0.75)):
            assert ref.fixed_sample(reso, ratio) == ArchManager(cfg).fixed_sample(reso, ratio)


def test_k7_subnet_is_the_extracted_litepose():
    """at [6, 7] everywhere and unequal stage-2/3 widths the supernet's rules are LitePose's: the derived state dict
    equals the prefix extraction of subnet.extract_subnet_state_dict, and the residual / stride lists LitePose's rule"""
    sd = _supernet().state_dict()
    for arch in (get_arch("XS"), get_arch("S"), ArchManager(get_cfg()).fixed_sample(512, 1.0)):
        sub = subnet.derive_supernet_subnet(sd, arch)
        lp = pose_mobilenet.get_pose_net(get_cfg(input_size=128), False, arch)
        ext = subnet.extract_subnet_state_dict(sd, lp.state_dict())
        assert sorted(sub.state_dict) == sorted(ext)
        for k in ext:
            assert torch.equal(sub.state_dict[k], ext[k]), k
        blocks = [b for st in lp.stage for b in st]
        assert sub.residual == [b.use_residual_connection for b in blocks]
        assert sub.strides == [b.stride for b in blocks]
        lp.load_state_dict(sub.state_dict, strict=True)


def test_mixed_subnet_rules():
    sd = _supernet().state_dict()
    sub = subnet.derive_supernet_subnet(sd, MIXED_JSON)
    # point 4 of the supernet's rules: stage 3 block 0 (stride 1, 80 -> 80) adds no identity, LitePose's rule would
    assert sub.residual == [False, True, False, True, True, False, True, False, True, True]
    assert sub.strides == [2, 1, 2, 1, 1, 2, 1, 1, 1, 1]
    lp = pose_mobilenet.get_pose_net(get_cfg(input_size=64), False, MIXED_JSON).eval()
    assert lp.stage[3][0].use_residual_connection
    # the k = 5 / 3 transform: the block's Linear over the centre taps
    w = sd["stage.0.1.depth_conv.0.weight"][:72, :, 2:5, 2:5].reshape(72, 1, 9)
    want = torch.nn.functional.linear(w, sd["stage.0.1.Linear3x3.weight"], sd["stage.0.1.Linear3x3.bias"])
    assert torch.equal(sub.state_dict["stage.0.1.depth_conv.0.weight"], want.reshape(72, 1, 3, 3))
    assert sub.state_dict["stage.1.0.depth_conv.0.weight"].shape == (144, 1, 5, 5)
    # LitePose with the derived weights and the supernet's residual equals the supernet; with its own rule it does not
    lp.load_state_dict(sub.state_dict, strict=True)
    x = synth.make_frames(1, 64, seed=2)
    want = model_ref_supernet.forward(sd, MIXED_JSON, x)
    with torch.no_grad():
        own = lp(x)
        lp.stage[3][0].use_residual_connection = False
        fixed = lp(x)
    assert all((a - b).abs().max() == 0 for a, b in zip(fixed, want))
    assert all((a - b).abs().max() > 1e-4 for a, b in zip(own, want))
    # the arch's stride keys are ignored; the '1.' prefix of network_to_half is accepted
    moved = copy.deepcopy(MIXED_JSON)
    for st in moved["backbone_setting"]:
        st["stride"] = 1
    again = subnet.derive_supernet_subnet({"1." + k: v.half() if v.is_floating_point() else v for k, v in sd.items()},
                                          moved)
    assert again.strides == sub.strides and again.residual == sub.residual and again.arch == sub.arch
    assert all(again.state_dict[k].dtype == torch.float32 for k in again.state_dict if "num_batches" not in k)


@pytest.mark.parametrize("change, match", [
    (lambda a: a["backbone_setting"][0]["block_setting"].__setitem__(0, [2.25, 7]), "not a multiple of 8"),
    (lambda a: a["backbone_setting"][2].__setitem__("num_blocks", 11), "supernet holds 10"),
    (lambda a: a["backbone_setting"][3]["block_setting"].__setitem__(1, [6, 9]), "kernel size"),
    (lambda a: a.__setitem__("input_channel", 32), "leading"),
    (lambda a: a["backbone_setting"].pop(), "4 stages"),
])
def test_derivation_refuses_with_the_reason(change, match):
    arch = copy.deepcopy(MIXED_JSON)
    change(arch)
    with pytest.raises(ValueError, match=match):
        subnet.derive_supernet_subnet(_supernet(64).state_dict(), arch)


def test_engine_plan_of_a_supernet_subnet(tmp_path):
    sub = subnet.derive_supernet_subnet(_supernet().state_dict(), MIXED_JSON)
    eng = engine.LitePoseEngine(sub.state_dict, sub.arch, "cpu", residual=sub.residual, strides=sub.strides)
    assert [b["res"] for b in eng.P["blocks"]] == sub.residual
    assert [b["stride"] for b in eng.P["blocks"]] == sub.strides
    assert [b["dw"]["k"] for b in eng.P["blocks"]] == [5, 3, 5, 7, 7, 7, 5, 7, 3, 5]
    ops = eng._build_plan(2, 128, 128, torch.float16, True, alloc=engine._Bump())["ops"]
    dws = [o for o in ops if o.name == "dw7"]
    assert [o.args[8] for o in dws if o.args[8] != 7] == [5, 3, 5, 5, 3, 5]     # k = 5 / 3: unfused dwconv
    # stage 3 block 0 (stride 1, 80 -> 80, no identity): no residual pointer whichever kernel runs it
    blk = [o for o in ops if o.name in ("block_s1", "block_s2", "dw7_project", "pc")]
    assert len(blk) == 10
    s3b0 = blk[7]
    assert (s3b0.args[7] == 0) if s3b0.name == "block_s1" else (s3b0.args[5 if s3b0.name == "dw7_project" else 3]
                                                                 is None)
    default = engine.LitePoseEngine(sub.state_dict, sub.arch, "cpu")
    assert default.P["blocks"][7]["res"] and not eng.P["blocks"][7]["res"]
    path = str(tmp_path / "super.folded.npz")
    eng.export_folded(path)
    back = engine.LitePoseEngine.from_folded(path, "cpu")
    assert [(b["res"], b["stride"]) for b in back.P["blocks"]] == [(b["res"], b["stride"]) for b in eng.P["blocks"]]
    with pytest.raises(ValueError, match="lists 9 blocks"):
        engine.LitePoseEngine(sub.state_dict, sub.arch, "cpu", residual=sub.residual[:-1])
    bad = list(sub.residual)
    bad[0] = True
    with pytest.raises(ValueError, match="identity add"):
        engine.LitePoseEngine(sub.state_dict, sub.arch, "cpu", residual=bad)


def test_module_behaves_like_the_reference_module():
    model = _supernet(64)
    m2 = copy.deepcopy(model)
    assert m2._lp_cache is not model._lp_cache and m2.arch_manager is not model.arch_manager
    m2.load_state_dict(model.state_dict(), strict=True)
    assert model.channel == [24, 32, 64, 96, 160] and model.final_channel == [28, 14]
    assert [len(s) for s in model.stage] == [6, 8, 10, 10]
    assert not model.stage[3][0].use_residual_connection and model.stage[3][1].use_residual_connection
    half = torch.nn.Sequential(m2.half())
    assert next(half.parameters()).dtype == torch.float16
    model.arch_manager.is_search = False
    with pytest.raises(ValueError, match="is_search"):
        model.lp_engine("cuda:0")
    cfg = get_cfg(input_size=64)
    cfg.MODEL.EXTRA.NUM_DECONV_KERNELS = [4, 3, 4]
    with pytest.raises(ValueError, match="4x4 stride-2"):
        pose_supermobilenet.get_pose_net(cfg)


def test_module_tree_runs_after_deconv_output_padding_fix():
    """the one deviation from the reference: its SuperConvTranspose2d raises on torch >= 2; this one returns the
    layer's output_padding and honours output_size"""
    m = _supernet(64).deconv_refined[0]
    x = torch.randn(1, 160, 4, 4)
    assert m(x, 64).shape == (1, 64, 8, 8)
    assert m(x, 64, output_size=[9, 9]).shape == (1, 64, 9, 9)


STUBS = {
    "_init_paths.py": "import os, sys\n"
                      "sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'lib'))\n",
    "lib/models/__init__.py": "",
    "lib/models/pose_mobilenet.py": "STOCK_REFERENCE_MODEL = True\n",
    "lib/models/pose_supermobilenet.py": "STOCK_REFERENCE_MODEL = True\n",
    "lib/models/pose_superresnet.py": "REFERENCE_ZOO = True\n",
    "lib/core/__init__.py": "",
    "lib/utils/__init__.py": "",
    "mobile_configs/search-XS.json": json.dumps(get_arch("XS")),
}

# what valid.py:95-145 does with --cfg supermobile.yaml --superconfig search-XS.json, up to its CPU summary forward
VALID = r'''
import argparse, json, sys
import _init_paths
assert sys.path[0].endswith("lib"), sys.path[:3]
import models
from litepose_b200.config import load_experiment
p = argparse.ArgumentParser()
p.add_argument("--cfg"); p.add_argument("--superconfig")
args = p.parse_args()
cfg, _ = load_experiment(args.cfg, args.superconfig)
cfg.DATASET.INPUT_SIZE = 64
assert models.pose_supermobilenet.__file__.startswith("%(root)s"), models.pose_supermobilenet.__file__
model = eval("models." + cfg.MODEL.NAME + ".get_pose_net")(cfg, is_train=True)
model.arch_manager.is_search = True
with open(args.superconfig) as f:
    model.arch_manager.search_arch = json.load(f)
import torch
outs = model(torch.rand(1, 3, cfg.DATASET.INPUT_SIZE, cfg.DATASET.INPUT_SIZE))
assert [tuple(o.shape) for o in outs] == [(1, 28, 16, 16), (1, 14, 32, 32)]
import models.pose_superresnet as sr
assert sr.__file__.startswith("%(ref)s")
print("supernet dropin ok")
'''


@pytest.mark.parametrize("how", ["sitecustomize", "runner"])
def test_dropin_resolves_pose_supermobilenet(tmp_path, how):
    ref = tmp_path / "reference"
    for name, text in STUBS.items():
        f = ref / name
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_text(text)
    with open(os.path.join(ROOT, "tests", "golden", "mobile.yaml")) as f:       # the experiment file, as supermobile
        yaml_text = f.read().replace("NAME: pose_mobilenet", "NAME: pose_supermobilenet")
    (ref / "experiments" / "crowd_pose" / "mobilenet").mkdir(parents=True)
    (ref / "experiments" / "crowd_pose" / "mobilenet" / "supermobile.yaml").write_text(yaml_text)
    ref = str(ref)
    (tmp_path / "reference" / "valid.py").write_text(VALID % {"ref": ref, "root": ROOT})
    argv = ["--cfg", "experiments/crowd_pose/mobilenet/supermobile.yaml", "--superconfig",
            "mobile_configs/search-XS.json"]
    env = dict(os.environ)
    if how == "sitecustomize":
        env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "litepose_b200", "dropin_site"), ROOT])
        cmd = [sys.executable, os.path.join(ref, "valid.py")] + argv
    else:
        env["PYTHONPATH"] = ROOT
        cmd = [sys.executable, "-m", "litepose_b200.dropin", os.path.join(ref, "valid.py")] + argv
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ref)
    assert r.returncode == 0 and "supernet dropin ok" in r.stdout, r.stdout + r.stderr
