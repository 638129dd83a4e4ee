"""CPU: tests/supernet_emul.py, the bit-exact restatement the GPU tests hold the supernet engine to.  With LitePose's own
residual / stride lists it equals tests/net_emul.py bit for bit (so it does the arithmetic net_emul pins); with the
supernet's lists, on a sub-network where the two rules differ, it follows the supernet (within fp16 tolerance of the
fp32 oracle) and no longer equals net_emul."""
import numpy as np
import torch

import net_emul
import supernet_emul
from litepose_b200 import subnet, synth
from litepose_b200.config import get_cfg
from litepose_b200.lib.models import pose_supermobilenet
from oracle import model_ref_supernet

# equal stage-2 / stage-3 widths: LitePose's rule adds an identity on stage 3 block 0, the supernet does not
ARCH = {"img_size": 256, "input_channel": 16, "deconv_setting": [32, 24, 16], "backbone_setting": [
    {"num_blocks": 2, "stride": 2, "channel": 16, "block_setting": [[6, 7], [3, 5]]},
    {"num_blocks": 2, "stride": 2, "channel": 32, "block_setting": [[6, 7], [4, 3]]},
    {"num_blocks": 2, "stride": 2, "channel": 48, "block_setting": [[6, 5], [6, 7]]},
    {"num_blocks": 2, "stride": 1, "channel": 48, "block_setting": [[6, 7], [3, 7]]}]}


def _sub():
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_supermobilenet.get_pose_net(get_cfg(input_size=64)), 1)
    sd = model.state_dict()
    return sd, subnet.derive_supernet_subnet(sd, ARCH)


def _litepose_lists(arch):
    res, strides, c = [], [], arch["input_channel"]
    for st in arch["backbone_setting"]:
        for bi in range(st["num_blocks"]):
            s = st["stride"] if bi == 0 else 1
            res.append(s == 1 and c == st["channel"])
            strides.append(s)
            c = st["channel"]
    return res, strides


def test_equals_net_emul_with_litepose_lists():
    _, sub = _sub()
    res, strides = _litepose_lists(sub.arch)
    assert res != sub.residual and strides == sub.strides
    x = synth.make_frames(1, 64, seed=4)
    for xin, flip, out_fp32 in ((x.half().numpy(), False, False), (x.numpy(), True, True)):
        got = supernet_emul.forward(sub.state_dict, sub.arch, xin, flip, out_fp32, residual=res, strides=strides)
        want = net_emul.forward(sub.state_dict, sub.arch, xin, flip, out_fp32)
        for g, w in zip(got, want):
            assert g.dtype == w.dtype and np.array_equal(g, w)


def test_follows_the_supernet_lists():
    sd, sub = _sub()
    x = synth.make_frames(1, 64, seed=4)
    got = supernet_emul.forward(sub.state_dict, sub.arch, x.half().numpy(), residual=sub.residual,
                                strides=sub.strides)
    lite = net_emul.forward(sub.state_dict, sub.arch, x.half().numpy())
    with torch.no_grad():
        ref = model_ref_supernet.forward(sd, ARCH, x)
    for g, l_, r in zip(got, lite, ref):
        r = r.numpy()
        tol = 2e-3 * np.abs(r).max() + 1e-4
        assert np.abs(g - r).max() <= tol
        assert np.abs(l_ - r).max() > np.abs(g - r).max()
