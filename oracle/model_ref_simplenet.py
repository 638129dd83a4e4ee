"""ORACLE (test infrastructure, not product code).

CPU fp32 restatement of the reference's ``pose_simplenet`` forward (LitePose without the Fusion Deconv Head) as a pure
function of a state_dict carrying the reference's parameter names, in the style of oracle/model_ref.py and with its
conv / BN helpers:
  * stem and inverted-residual stages   reference lib/models/pose_simplenet.py:35-59,124-128
  * deconv levels and output heads      reference lib/models/pose_simplenet.py:129-138 - every level on the refined
                                        tensor alone, every output ``final_refined[i-1]`` alone

build_reference() builds the UNMODIFIED reference module (imported in place through oracle/refshim.py) with the seeded
weights of refshim.build_reference_model.  Pinned against it in tests/test_simplenet_host.py (0.0 max difference where
the reference tree is present) and through tests/golden/model_simplenet_*.npz (oracle/make_golden_simplenet.py).
"""
import torch.nn.functional as F

from oracle.model_ref import _bn, _conv


def forward(sd, arch, x, capture=None):
    """Reference-order forward; ``capture`` (dict) receives named activations."""
    def cap(name, t):
        if capture is not None:
            capture[name] = t
        return t

    x = x.float()
    x = F.relu6(_bn(_conv(x, sd["first.0.0.weight"], 2), sd, "first.0.1"))
    x = F.relu6(_bn(_conv(x, sd["first.1.0.weight"], 1, x.shape[1]), sd, "first.1.1"))
    x = cap("first", _bn(_conv(x, sd["first.2.weight"]), sd, "first.3"))
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            p = "stage.%d.%d." % (si, bi)
            stride = st["stride"] if bi == 0 else 1
            y = F.relu6(_bn(_conv(x, sd[p + "inv.0.weight"]), sd, p + "inv.1"))
            y = F.relu6(_bn(_conv(y, sd[p + "depth_conv.0.weight"], stride, y.shape[1]), sd, p + "depth_conv.1"))
            y = _bn(_conv(y, sd[p + "point_conv.0.weight"]), sd, p + "point_conv.1")
            if stride == 1 and x.shape[1] == y.shape[1]:
                y = y + x
            x = cap(p + "out", y)
    refined = x
    outs = []
    for i in range(3):
        a = F.conv_transpose2d(refined, sd["deconv_refined.%d.weight" % i].float(), None, 2, 1)
        refined = cap("deconv.%d" % i, F.relu(_bn(a, sd, "deconv_bnrelu.%d.0" % i)))
        if i > 0:
            p = "final_refined.%d.conv." % (i - 1)
            t = F.relu(_bn(_conv(refined, sd[p + "0.weight"], 1, refined.shape[1]), sd, p + "1"))
            outs.append(cap("out.%d" % (i - 1), _conv(t, sd[p + "3.weight"])))
    return outs


def build_reference(cfg, arch, seed=0, bn_seed=1):
    """The reference's lib/models/pose_simplenet.py, seeded as refshim.build_reference_model seeds pose_mobilenet."""
    import importlib
    import torch
    from litepose_b200.synth import randomize_bn_
    from oracle import refshim
    refshim.load()
    ps = importlib.import_module("lib.models.pose_simplenet")
    torch.manual_seed(seed)
    model = ps.get_pose_net(cfg, False, arch)
    randomize_bn_(model, bn_seed)
    return model.eval()
