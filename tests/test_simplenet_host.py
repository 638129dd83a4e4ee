"""CPU: the pose_simplenet drop-in (LitePose without the fusion head) against the reference's own module through the
committed fixtures, the oracle forward against them, the engine's recognition of the single-branch state dict, its
folded export, and the drop-in's resolution of ``models.pose_simplenet`` in both launch modes."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from litepose_b200 import engine, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models import pose_mobilenet, pose_simplenet
from oracle import model_ref_simplenet, refshim
from oracle.make_golden import sd_digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(name, size, mod=pose_simplenet):
    torch.manual_seed(0)
    return synth.randomize_bn_(mod.get_pose_net(get_cfg(input_size=size), False, get_arch(name)), 1).eval()


@pytest.mark.parametrize("name", ["XS", "S"])
def test_state_dict_and_oracle_equal_reference_golden(golden_dir, name):
    z = np.load(os.path.join(golden_dir, "model_simplenet_%s_128.npz" % name))
    model = _model(name, 128)
    sd = model.state_dict()
    assert sd_digest(sd) == str(z["digest"]), "drop-in must create the reference's keys, shapes and seeded weights"
    assert not any(k.startswith(("deconv_raw.", "final_raw.")) for k in sd)
    full = pose_mobilenet.get_pose_net(get_cfg(input_size=128), False, get_arch(name)).state_dict()
    assert list(sd) == [k for k in full if not k.startswith(("deconv_raw.", "final_raw."))]
    x = synth.make_frames(1, 128, seed=11)
    with torch.no_grad():
        outs = model_ref_simplenet.forward(sd, get_arch(name), x)
        mods = model(x)                        # CPU tensor: the module tree
    for a, m, k in zip(outs, mods, ("out0", "out1")):
        assert np.allclose(a.numpy(), z[k], atol=1e-5)
        assert np.allclose(m.numpy(), z[k], atol=1e-5)
        tol = 2e-3 * np.abs(z[k]).max() + 1e-4
        assert np.abs(z[k + "_fp16eager"] - z[k]).max() <= tol


@pytest.mark.skipif(not refshim.available(), reason="reference tree not present")
def test_oracle_equals_unmodified_reference():
    cfg, arch = get_cfg(input_size=64), get_arch("XS")
    ref = model_ref_simplenet.build_reference(cfg, arch)
    x = synth.make_frames(2, 64, seed=3)
    with torch.no_grad():
        want = ref(x)
        got = model_ref_simplenet.forward(ref.state_dict(), arch, x)
    for a, b in zip(got, want):
        assert (a - b).abs().max().item() == 0.0


def test_module_behaves_like_the_reference_module():
    model = _model("XS", 64)
    m2 = copy.deepcopy(model)
    assert m2._lp_cache is not model._lp_cache
    m2.load_state_dict(model.state_dict(), strict=True)
    assert model.channel == [16, 16, 32, 48, 80] and model.final_channel == [28, 14]
    half = torch.nn.Sequential(m2.half())
    assert next(half.parameters()).dtype == torch.float16
    cfg = get_cfg(input_size=64)
    cfg.MODEL.EXTRA.NUM_DECONV_KERNELS = [4, 3, 4]
    with pytest.raises(ValueError, match="4x4 stride-2"):
        pose_simplenet.get_pose_net(cfg, False, get_arch("XS"))


def test_engine_recognises_simplenet_on_cpu():
    sd = _model("S", 128).state_dict()
    eng = engine.LitePoseEngine(sd, get_arch("S"), "cpu")
    assert eng.topology == engine.SIMPLE
    assert all(d["Cw"] == 0 for d in eng.P["deconv"]) and all(h["C2"] == 0 for h in eng.P["heads"])
    assert not any("final_raw_dw" in h for h in eng.P["heads"])
    ops = eng._build_plan(2, 512, 512, torch.float16, True, alloc=engine._Bump())["ops"]
    for op in ops:
        if op.name == "deconv":
            assert op.args[1] is None and op.args[9] == 0
        if op.name == "head_fused":
            assert op.args[1] is None and op.args[11] == 0
    full = engine.LitePoseEngine(_model("S", 128, pose_mobilenet).state_dict(), get_arch("S"), "cpu")
    assert full.topology == engine.FUSION


@pytest.mark.parametrize("drop", ["deconv_raw.1.", "final_raw.0.", "final_raw."])
def test_engine_refuses_a_half_raw_state_dict(drop):
    sd = _model("XS", 64, pose_mobilenet).state_dict()
    sd = {k: v for k, v in sd.items() if not k.startswith(drop)}
    with pytest.raises(ValueError, match="some levels only"):
        engine.LitePoseEngine(sd, get_arch("XS"), "cpu")


def test_folded_export_round_trips_on_cpu(tmp_path):
    sd = _model("XS", 128).state_dict()
    a = engine.LitePoseEngine(sd, get_arch("XS"), "cpu")
    path = str(tmp_path / "simple.folded.npz")
    a.export_folded(path)
    b = engine.LitePoseEngine.from_folded(path, "cpu")
    assert b.topology == engine.SIMPLE
    pa = a._build_plan(1, 128, 128, torch.float16, True, alloc=engine._Bump())["ops"]
    pb = b._build_plan(1, 128, 128, torch.float16, True, alloc=engine._Bump())["ops"]

    def shapes(ops):       # op names, NULL pointers and the shape arguments (weight pointers differ between engines)
        return [(o.name, [a for a in o.args if a is None or (isinstance(a, int) and a < 4096)]) for o in ops]

    assert shapes(pa) == shapes(pb)
    for i in range(3):
        assert torch.equal(a.P["deconv"][i]["w"], b.P["deconv"][i]["w"])
    for i in range(2):
        for k in ("dw_cat", "bdw_cat", "pw_cat"):
            assert torch.equal(a.P["heads"][i][k], b.P["heads"][i][k])


def test_folded_file_without_topology_loads_as_fusion(tmp_path):
    """files written before the header recorded the head topology are fusion-head files"""
    import json
    a = engine.LitePoseEngine(_model("XS", 64, pose_mobilenet).state_dict(), get_arch("XS"), "cpu")
    path = str(tmp_path / "old.npz")
    a.export_folded(path)
    z = dict(np.load(path))
    header = json.loads(bytes(z["__header__"]).decode())
    del header["topology"]
    z["__header__"] = np.frombuffer(json.dumps(header).encode(), dtype=np.uint8)
    np.savez(path, **z)
    b = engine.LitePoseEngine.from_folded(path, "cpu")
    assert b.topology == engine.FUSION and all(d["Cw"] > 0 for d in b.P["deconv"])


STUBS = {
    "_init_paths.py": "import os, sys\n"
                      "sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'lib'))\n",
    "lib/models/__init__.py": "",
    "lib/models/pose_mobilenet.py": "STOCK_REFERENCE_MODEL = True\n",
    "lib/models/pose_simplenet.py": "STOCK_REFERENCE_MODEL = True\n",
    "lib/models/pose_higher_hrnet.py": "REFERENCE_ZOO = True\n",
    "lib/core/__init__.py": "",
    "lib/utils/__init__.py": "",
}

CHECK = r'''
import sys
import _init_paths
assert sys.path[0].endswith("lib"), sys.path[:3]
import models
repo = "%(root)s"
assert models.pose_simplenet.__file__.startswith(repo), models.pose_simplenet.__file__
from litepose_b200.config import get_cfg, get_arch
m = eval("models.pose_simplenet.get_pose_net")(get_cfg(input_size=64), is_train=False, cfg_arch=get_arch("XS"))
assert hasattr(m, "lp_engine") and not hasattr(m, "deconv_raw")
import models.pose_higher_hrnet as hr
assert hr.__file__.startswith("%(ref)s")
print("simplenet dropin ok")
'''


@pytest.mark.parametrize("how", ["sitecustomize", "runner"])
def test_dropin_resolves_pose_simplenet(tmp_path, how):
    ref = tmp_path / "reference"
    for name, text in STUBS.items():
        f = ref / name
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_text(text)
    ref = str(ref)
    body = CHECK % {"ref": ref, "root": ROOT}
    env = dict(os.environ)
    if how == "sitecustomize":
        env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "litepose_b200", "dropin_site"), ROOT])
        script = tmp_path / "check.py"
        script.write_text(body)
        cmd = [sys.executable, "-c", "import sys; sys.path.insert(0, %r); exec(open(%r).read())" % (ref, str(script))]
    else:
        env["PYTHONPATH"] = ROOT
        script = tmp_path / "run_in_ref.py"
        script.write_text("import sys; sys.path.insert(0, %r)\n" % ref + body)
        cmd = [sys.executable, "-m", "litepose_b200.dropin", str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ref)
    assert r.returncode == 0 and "simplenet dropin ok" in r.stdout, r.stdout + r.stderr
