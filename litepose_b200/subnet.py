"""Sub-network extraction from a (super)network checkpoint (SURVEY.md 8(f) row 4).

The reference trains one supernet and obtains LitePose-XS...L by weight transfer (weight_transfer.py:75-146): every
tensor of the sub-network is the leading slice of the same-named supernet tensor - conv [:out, :in], transposed conv
[:in, :out], depthwise [:mid], BatchNorm vectors [:n] - and blocks beyond the sub-network's depth are dropped.  Because
all of those are prefix slices in every dimension, one rule covers them."""
import torch


def extract_subnet_state_dict(super_state_dict, sub_state_dict_like):
    """super_state_dict: checkpoint of the larger network (keys optionally prefixed '1.' by network_to_half);
    sub_state_dict_like: state_dict (or {name: shape}) of the target architecture.  Returns a state_dict for the target:
    floating-point tensors as float32 clones (weight_transfer.py does .float().clone()), counters unchanged."""
    sup = {(k[2:] if k.startswith("1.") else k): v for k, v in super_state_dict.items()}
    out = {}
    for name, like in sub_state_dict_like.items():
        shape = tuple(like.shape) if hasattr(like, "shape") else tuple(like)
        if name not in sup:
            raise KeyError("supernet checkpoint has no tensor %r" % name)
        src = sup[name]
        if src.dim() != len(shape) or any(s < d for s, d in zip(src.shape, shape)):
            raise ValueError("%s: supernet tensor %s cannot provide %s" % (name, tuple(src.shape), shape))
        piece = src[tuple(slice(0, d) for d in shape)]
        out[name] = piece.float().clone() if piece.is_floating_point() else piece.clone()
    return out


def extract_subnet(super_state_dict, cfg, arch):
    """Builds the target LitePose (litepose_b200 drop-in module) for ``arch`` and loads the extracted weights."""
    from litepose_b200.lib.models.pose_mobilenet import get_pose_net
    net = get_pose_net(cfg, False, arch)
    net.load_state_dict(extract_subnet_state_dict(super_state_dict, net.state_dict()), strict=True)
    return net.eval()


# The super-network (reference lib/models/pose_supermobilenet.py) evaluates a sub-architecture without extracting it:
# its forward slices the same tensors on the fly, with rules of its own that differ from a LitePose built for that
# architecture in three places:
#   * a block's depthwise kernel is the centre k x k of the 7x7 weight, and for k = 5 / 3 that block's own
#     Linear5x5 / Linear3x3 maps the k*k taps of every channel (W . L^T + b) before use (super_layers.py:165-191);
#   * a block's stride and identity add are fixed by the supernet's construction, from its widest channel counts
#     (super_layers.py:163): block 0 of every stage never adds its input, not even where the sub-network's widths are
#     equal (stage 3 block 0 with equal stage-2 and stage-3 widths), where a LitePose would;
#   * the arch dict's ``stride`` keys are ignored; the supernet's stages have strides 2, 2, 2, 1.
SUPER_STRIDES = (2, 2, 2, 1)      # the supernet's stage strides (pose_supermobilenet.py:26-31)
SUPER_KERNEL = 7                  # widest depthwise kernel of a super block


class SupernetSub(object):
    """One sub-network of a super-network: ``state_dict`` with LitePose (pose_mobilenet) names and shapes, ``arch`` the
    cfg_arch with the supernet's strides, and per block (stage-major) ``residual`` and ``strides``, the rules the
    supernet applies (LitePoseEngine(state_dict, arch, device, residual=..., strides=...))."""

    def __init__(self, state_dict, arch, residual, strides):
        self.state_dict, self.arch, self.residual, self.strides = state_dict, arch, residual, strides


def _super_blocks(sup, stage):
    n = 0
    while "stage.%d.%d.inv.0.weight" % (stage, n) in sup:
        n += 1
    return n


def derive_supernet_subnet(super_state_dict, cfg_arch):
    """The sub-network ``cfg_arch`` of a super-network checkpoint (keys optionally prefixed '1.' by network_to_half)
    as a SupernetSub.  Every tensor is a leading slice of the supernet's (SuperConv2d [:out, :in], SuperBatchNorm2d
    [:n], SuperConvTranspose2d [:in, :out], SuperSepConv2d depthwise [:in] and 1x1 [:, :in]); the first ``num_blocks``
    blocks of each stage are kept; a block's expansion width is round(cin * t), refused unless a multiple of 8 (the
    kernels' channel granularity); the k = 5 / 3 depthwise transform is computed in fp32 on the CPU.  Floating-point
    tensors come out as fp32 CPU tensors, counters unchanged."""
    sup = {(k[2:] if k.startswith("1.") else k): v.detach().cpu() for k, v in super_state_dict.items()}
    out = {}

    def take(name, *sizes):
        src = sup[name]
        if any(s > d for s, d in zip(sizes, src.shape)):
            raise ValueError("%s: the supernet tensor %s has no leading %s slice" % (name, tuple(src.shape), sizes))
        piece = src[tuple(slice(0, s) for s in sizes)]
        out[name] = piece.float().clone() if piece.is_floating_point() else piece.clone()

    def bn(prefix, n):
        for leaf in ("weight", "bias", "running_mean", "running_var"):
            take(prefix + "." + leaf, n)
        if prefix + ".num_batches_tracked" in sup:
            take(prefix + ".num_batches_tracked")

    for name in sup:
        if name.startswith(("first.0.", "first.1.")):
            take(name)
    c = int(cfg_arch["input_channel"])
    take("first.2.weight", c)
    bn("first.3", c)
    channels = [c]
    stages = cfg_arch["backbone_setting"]
    if len(stages) != len(SUPER_STRIDES):
        raise ValueError("the supernet has %d stages, the architecture %d" % (len(SUPER_STRIDES), len(stages)))
    residual, strides = [], []
    for si, st in enumerate(stages):
        n, cout = int(st["num_blocks"]), int(st["channel"])
        have = _super_blocks(sup, si)
        if not 1 <= n <= have:
            raise ValueError("stage %d: %d blocks asked, the supernet holds %d" % (si, n, have))
        if len(st["block_setting"]) < n:
            raise ValueError("stage %d: block_setting lists %d blocks for num_blocks %d"
                             % (si, len(st["block_setting"]), n))
        for bi in range(n):
            p = "stage.%d.%d." % (si, bi)
            t, k = st["block_setting"][bi]
            mid = round(c * t)
            if mid % 8:
                raise ValueError("stage %d block %d: expansion width round(%d * %s) = %d is not a multiple of 8, which "
                                 "the kernels' channel tiling needs" % (si, bi, c, t, mid))
            if k not in (3, 5, 7):
                raise ValueError("stage %d block %d: kernel size %r; the supernet has 3, 5 and 7" % (si, bi, k))
            take(p + "inv.0.weight", mid, c)
            bn(p + "inv.1", mid)
            w = sup[p + "depth_conv.0.weight"]
            if mid > w.shape[0]:
                raise ValueError("%sdepth_conv: expansion width %d, the supernet has %d" % (p, mid, w.shape[0]))
            lo = SUPER_KERNEL // 2 - k // 2
            w = w[:mid, :, lo:lo + k, lo:lo + k].float()
            if k != SUPER_KERNEL:
                lin = "%sLinear%dx%d." % (p, k, k)
                w = torch.nn.functional.linear(w.reshape(mid, 1, k * k), sup[lin + "weight"].float(),
                                               sup[lin + "bias"].float()).reshape(mid, 1, k, k)
            out[p + "depth_conv.0.weight"] = w.clone()
            bn(p + "depth_conv.1", mid)
            take(p + "point_conv.0.weight", cout, mid)
            bn(p + "point_conv.1", cout)
            stride = SUPER_STRIDES[si] if bi == 0 else 1
            sup_in = sup[p + "inv.0.weight"].shape[1]
            sup_out = sup[p + "point_conv.0.weight"].shape[0]
            res = stride == 1 and sup_in == sup_out
            if res and c != cout:
                raise ValueError("stage %d block %d adds its input in the supernet, but the architecture changes its "
                                 "width (%d -> %d)" % (si, bi, c, cout))
            residual.append(res)
            strides.append(stride)
            c = cout
        channels.append(c)
    filters = [int(f) for f in cfg_arch["deconv_setting"]]
    refined = channels[-1]
    for i, f in enumerate(filters):
        take("deconv_refined.%d.weight" % i, refined, f)
        take("deconv_raw.%d.weight" % i, channels[-i - 2], f)
        bn("deconv_bnrelu.%d.0" % i, f)
        refined = f
    for i in range(1, len(filters)):
        for nm, cin in (("final_refined", filters[i]), ("final_raw", channels[-i - 3])):
            p = "%s.%d.conv." % (nm, i - 1)
            take(p + "0.weight", cin)
            bn(p + "1", cin)
            take(p + "3.weight", sup[p + "3.weight"].shape[0], cin)
    arch = {"img_size": cfg_arch.get("img_size"), "input_channel": channels[0], "deconv_setting": filters,
            "backbone_setting": [{"num_blocks": int(st["num_blocks"]), "stride": SUPER_STRIDES[si],
                                  "channel": int(st["channel"]),
                                  "block_setting": [list(b) for b in st["block_setting"][:int(st["num_blocks"])]]}
                                 for si, st in enumerate(stages)]}
    return SupernetSub(out, arch, residual, strides)
