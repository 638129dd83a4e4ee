"""CPU: the super-network's BN recalibration pass (SuperLitePose.lp_recalibrate_bn) against the reference's goldens.

(a) The package's SuperLitePose module tree in training mode reproduces tests/golden/supernet_recal_*.npz: every
    BatchNorm buffer after each of three batches, num_batches_tracked, and the last batch's outputs, within fp32
    round-off.  This pins the train-mode semantics (slices, unbiased running variance, which BatchNorm counts batches).
(b) tests/bn_train_emul.py, the bit-exact restatement of the kernel path, is within
    recal_cases.TOL_FACTOR times the model tolerance 2e-3 max|ref| + 1e-4 of the goldens, per output and per BatchNorm
    tensor (the fp16 raw tensors; see there); the fraction used is printed.  The goldens'
    untouched suffixes of every BatchNorm equal the start state.
(c) lp_recalibrate_bn's refusals, and its random_sample() draw, which is forward's."""
import random

import numpy as np
import pytest
import torch

import bn_train_emul
import recal_cases as rc
from oracle.make_golden import sd_digest
from litepose_b200.config import get_cfg
from litepose_b200.lib.models import pose_supermobilenet
from litepose_b200.subnet import derive_supernet_subnet


@pytest.mark.parametrize("name", rc.ARCHS)
def test_module_tree_reproduces_golden(golden_dir, name):
    z, arch = rc.golden(golden_dir, name)
    inp = rc.inputs(golden_dir)
    model = rc.supernet(golden_dir, arch).train()
    with torch.no_grad():
        for i in range(3):
            outs = model(torch.from_numpy(inp["batches"][i]).float())
            rm, rv, nbt = rc.state(model)
            for got, want, what in ((rm, z["running_mean"][i], "running_mean"), (rv, z["running_var"][i], "running_var")):
                err = np.abs(got - want).max()
                assert err <= 1e-5 * np.abs(want).max() + 1e-6, (name, i, what, err)
            assert np.array_equal(nbt, z["num_batches_tracked"][i]), (name, i)
    for k, o in zip(("out0", "out1"), outs):
        err = np.abs(o.numpy() - z[k]).max()
        assert err <= 1e-4 * np.abs(z[k]).max() + 1e-6, (name, k, err)


def test_golden_digest_and_counts(golden_dir):
    """the goldens were made from the seeded weights this package builds, and only first.0.1 / first.1.1 count"""
    inp = rc.inputs(golden_dir)
    z, arch = rc.golden(golden_dir, "search_XS")
    torch.manual_seed(0)
    from litepose_b200 import synth
    m = synth.randomize_bn_(pose_supermobilenet.get_pose_net(get_cfg(input_size=rc.SIZE)), 1)
    assert sd_digest(m.state_dict()) == str(inp["digest"])
    names = [n for n, _ in rc.bn_modules(m)]
    grew = {n for n, a, b in zip(names, inp["num_batches_tracked"], z["num_batches_tracked"][-1]) if b != a}
    assert grew == {"first.0.1", "first.1.1"}
    assert all(z["num_batches_tracked"][-1][names.index(n)] == inp["num_batches_tracked"][names.index(n)] + 3
               for n in grew)


@pytest.mark.parametrize("name", rc.ARCHS)
def test_emulation_within_golden_tolerance(golden_dir, name):
    z, arch = rc.golden(golden_dir, name)
    inp = rc.inputs(golden_dir)
    model = rc.supernet(golden_dir, arch)
    used = rc.used(model, arch)
    sub = derive_supernet_subnet(model.state_dict(), arch)
    params = {n: (0.1, 1e-5) for n in used}
    rm0, rv0 = np.asarray(inp["running_mean"]), np.asarray(inp["running_var"])
    running = {n: (rm0[o:o + c], rv0[o:o + c]) for n, (o, c) in used.items()}
    worst = 0.0
    for i in range(3):
        outs, new, bad = bn_train_emul.forward(sub, inp["batches"][i].astype(np.float32), running, params)
        assert not bad
        running = new
        for n, (o, c) in used.items():
            for j, key in enumerate(("running_mean", "running_var")):
                want = z[key][i][o:o + c]
                used_ = rc.tol_used(new[n][j], want)
                worst = max(worst, used_)
                assert used_ <= rc.TOL_FACTOR, (name, i, n, key, used_)
    for k, o in zip(("out0", "out1"), outs):
        u = rc.tol_used(o, z[k])
        print("%s %s: %.3f of the tolerance" % (name, k, u))
        assert u <= rc.TOL_FACTOR, (name, k, u)
    print("%s BN buffers: at most %.3f of the tolerance" % (name, worst))
    # the reference leaves the suffix past each slice (and every BatchNorm the sub-network skips) untouched
    mask = np.ones(rm0.shape, bool)
    for n, (o, c) in used.items():
        mask[o:o + c] = False
    for i in range(3):
        assert np.array_equal(z["running_mean"][i][mask], rm0[mask])
        assert np.array_equal(z["running_var"][i][mask], rv0[mask])


def _model():
    torch.manual_seed(0)
    return pose_supermobilenet.get_pose_net(get_cfg(input_size=64))


def test_refusals():
    m = _model()
    with pytest.raises(ValueError, match="CUDA tensor"):
        m.lp_recalibrate_bn(torch.zeros(2, 3, 64, 64))
    with pytest.raises(ValueError, match="NCHW"):
        m.lp_recalibrate_bn(torch.zeros(2, 3, 64, 64, dtype=torch.float64))
    with pytest.raises(ValueError, match="multiples of 16"):
        m.lp_recalibrate_bn(torch.zeros(2, 3, 72, 64))
    with pytest.raises(ValueError, match="more than one"):
        m.lp_recalibrate_bn(torch.zeros(1, 3, 16, 16))
    m.stage[0][0].depth_conv[1].momentum = None
    with pytest.raises(ValueError, match="momentum None"):
        m.lp_recalibrate_bn(torch.zeros(2, 3, 64, 64))


def test_draws_like_forward():
    """lp_recalibrate_bn consumes random_sample() exactly as forward does (one draw per call)"""
    m = _model().eval()
    x = torch.zeros(1, 3, 64, 64)
    random.seed(7)
    with pytest.raises(ValueError):
        m.lp_recalibrate_bn(x)
    after_recal = random.getstate()
    random.seed(7)
    with torch.no_grad():
        m(x)
    assert random.getstate() == after_recal
