"""ORACLE (test infrastructure, not product code).

CPU fp32 restatement of the reference's ``SuperLitePose.forward`` (the LitePose super-network) as a pure function of
(super state dict, arch), in the style of oracle/model_ref.py and with its conv / BN helpers.  It slices the supernet's
tensors where the reference's super layers do, and shares no code with litepose_b200/subnet.py:
  * stem                          reference lib/models/pose_supermobilenet.py:36-41,135-138 (first.2 [:c0], first.3 [:c0])
  * SuperInvBottleneck.forward    reference lib/models/layers/super_layers.py:165-191: round(cin*t) wide, centre k x k of
                                  the 7x7 depthwise through Linear5x5 / Linear3x3 for k = 5 / 3, identity add fixed by the
                                  supernet's widest widths and strides (2, 2, 2, 1 on block 0 of the stages)
  * deconv levels and heads       reference lib/models/pose_supermobilenet.py:151-162, super_layers.py:31-86

build_reference() builds the UNMODIFIED reference module (imported in place through oracle/refshim.py) with the seeded
weights of refshim.build_reference_model and one shim: ``SuperConvTranspose2d._output_padding`` accepts the torch-1 call
the reference makes (super_layers.py:40) and returns the layer's ``output_padding``, what that call means when
``output_size`` is None.  Without it the reference raises on torch >= 2.0.  Pinned against it in
tests/test_supernet_host.py (0.0 max difference where the reference tree is present) and through
tests/golden/model_supernet_*.npz (oracle/make_golden_supernet.py).
"""
import torch
import torch.nn.functional as F

from oracle.model_ref import _conv

EPS = 1e-5
STRIDES = (2, 2, 2, 1)


def _sbn(x, sd, p):
    """BatchNorm over the input's channels: the leading slice of every vector"""
    c = x.shape[1]
    return F.batch_norm(x, sd[p + ".running_mean"][:c].float(), sd[p + ".running_var"][:c].float(),
                        sd[p + ".weight"][:c].float(), sd[p + ".bias"][:c].float(), False, 0.0, EPS)


def forward(sd, arch, x, capture=None):
    """Reference-order forward of sub-architecture ``arch``; ``capture`` (dict) receives named activations."""
    def cap(name, t):
        if capture is not None:
            capture[name] = t
        return t

    sd = {(k[2:] if k.startswith("1.") else k): v for k, v in sd.items()}
    x = x.float()
    x = F.relu6(_sbn(_conv(x, sd["first.0.0.weight"], 2), sd, "first.0.1"))
    x = F.relu6(_sbn(_conv(x, sd["first.1.0.weight"], 1, x.shape[1]), sd, "first.1.1"))
    x = _conv(x, sd["first.2.weight"][:arch["input_channel"], :x.shape[1]])
    x = cap("first", _sbn(x, sd, "first.3"))
    feats = [x]
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            p = "stage.%d.%d." % (si, bi)
            t, k = st["block_setting"][bi]
            stride = STRIDES[si] if bi == 0 else 1
            wi, wp = sd[p + "inv.0.weight"], sd[p + "point_conv.0.weight"]
            mid = round(x.shape[1] * t)
            y = F.relu6(_sbn(_conv(x, wi[:mid, :x.shape[1]]), sd, p + "inv.1"))
            lo = 3 - k // 2
            w = sd[p + "depth_conv.0.weight"][:mid, :, lo:lo + k, lo:lo + k].float()
            if k != 7:
                lin = "%sLinear%dx%d." % (p, k, k)
                w = F.linear(w.reshape(mid, 1, k * k), sd[lin + "weight"].float(),
                             sd[lin + "bias"].float()).reshape(mid, 1, k, k)
            y = F.relu6(_sbn(F.conv2d(y, w, None, stride, k // 2, 1, mid), sd, p + "depth_conv.1"))
            y = _sbn(_conv(y, wp[:st["channel"], :mid]), sd, p + "point_conv.1")
            if stride == 1 and wi.shape[1] == wp.shape[0]:       # the supernet's widest widths decide
                y = y + x
            x = cap(p + "out", y)
        feats.append(x)
    outs = []
    refined, raw = feats[-1], feats[-2]
    for i, f in enumerate(arch["deconv_setting"]):
        a = F.conv_transpose2d(refined, sd["deconv_refined.%d.weight" % i][:refined.shape[1], :f].float(), None, 2, 1)
        b = F.conv_transpose2d(raw, sd["deconv_raw.%d.weight" % i][:raw.shape[1], :f].float(), None, 2, 1)
        refined = cap("deconv.%d" % i, F.relu(_sbn(a + b, sd, "deconv_bnrelu.%d.0" % i)))
        raw = feats[-i - 3]
        if i > 0:
            o = 0
            for nm, src in (("final_refined", refined), ("final_raw", raw)):
                p = "%s.%d.conv." % (nm, i - 1)
                c = src.shape[1]
                h = F.relu(_sbn(_conv(src, sd[p + "0.weight"][:c], 1, c), sd, p + "1"))
                o = o + _conv(h, sd[p + "3.weight"][:, :c])
            outs.append(cap("out.%d" % (i - 1), o))
    return outs


def _shim(sl):
    """the one change to the reference: its torch-1 ``_output_padding`` call made valid on torch >= 2.0"""
    base = torch.nn.ConvTranspose2d._output_padding

    def output_padding(self, input, output_size, stride, padding, kernel_size, num_spatial_dims=2, dilation=None):
        return base(self, input, output_size, stride, padding, kernel_size, num_spatial_dims, dilation)

    sl.SuperConvTranspose2d._output_padding = output_padding


def load_reference():
    """the reference's pose_supermobilenet and arch_manager modules, imported in place (plus the shim)"""
    import importlib
    from oracle import refshim
    refshim.load()
    sl = importlib.import_module("lib.models.layers.super_layers")
    if not getattr(sl.SuperConvTranspose2d, "_lp_shimmed", False):
        _shim(sl)
        sl.SuperConvTranspose2d._lp_shimmed = True
    return importlib.import_module("lib.models.pose_supermobilenet"), importlib.import_module("arch_manager")


def build_reference(cfg, seed=0, bn_seed=1):
    """The reference's SuperLitePose, seeded as refshim.build_reference_model seeds pose_mobilenet."""
    from litepose_b200.synth import randomize_bn_
    psm, _ = load_reference()
    torch.manual_seed(seed)
    model = psm.get_pose_net(cfg, False)
    randomize_bn_(model, bn_seed)
    return model.eval()
