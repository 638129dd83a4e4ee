"""Drop-in replacement of the reference's ``lib/models/pose_mobilenet.py``.

``get_pose_net(cfg, is_train=False, cfg_arch=None)`` returns an ``nn.Module`` whose
parameter/buffer names, shapes and creation order equal the reference's
(reference lib/models/pose_mobilenet.py:21-176, lib/models/layers/layers.py:18-24,
90-133), so ``load_state_dict(strict=True)`` (valid.py:157), ``network_to_half``
(lib/fp16_utils/fp16util.py:87-91), ``copy.deepcopy`` and seeded initialisation behave
identically.  What differs is ``forward``: in eval mode on a CUDA tensor it runs the
hand-written sm_90a kernels through the C ABI (litepose_b200.engine); the module
tree itself is only executed for CPU tensors (the parameter-count/summary call of
valid.py:147-150) and in training mode (autograd), never for CUDA inference.
"""
import os

import torch
import torch.nn as nn

from ._engine_module import EngineModule, _EngineCache


def _make_divisible(v, divisor, min_value=None):
    floor = divisor if min_value is None else min_value
    out = max(floor, (int(v + divisor / 2) // divisor) * divisor)
    return out + divisor if out < 0.9 * v else out


def _conv_bn(cin, cout, k, stride, groups, act):
    layers = [nn.Conv2d(cin, cout, k, stride, k // 2, groups=groups, bias=False), nn.BatchNorm2d(cout)]
    if act is not None:
        layers.append(act(inplace=True))
    return layers


class convbnrelu(nn.Sequential):
    """conv k x k + BN + ReLU6 (children 0,1,2 like the reference block)."""

    def __init__(self, inp, oup, ker=3, stride=1, groups=1):
        super().__init__(*_conv_bn(inp, oup, ker, stride, groups, nn.ReLU6))


class InvBottleneck(nn.Module):
    """1x1 expand -> k x k depthwise -> 1x1 project (+ identity when shapes allow)."""

    def __init__(self, inplanes, planes, stride=1, ker=3, exp=6):
        super().__init__()
        mid = _make_divisible(round(inplanes * exp), 8)
        self.inv = nn.Sequential(*_conv_bn(inplanes, mid, 1, 1, 1, nn.ReLU6))
        self.depth_conv = nn.Sequential(*_conv_bn(mid, mid, ker, stride, mid, nn.ReLU6))
        self.point_conv = nn.Sequential(*_conv_bn(mid, planes, 1, 1, 1, None))
        self.stride = stride
        self.use_residual_connection = stride == 1 and inplanes == planes

    def forward(self, x):
        y = self.point_conv(self.depth_conv(self.inv(x)))
        return y + x if self.use_residual_connection else y


class SepConv2d(nn.Module):
    """k x k depthwise + BN + ReLU, then a bias-free 1x1."""

    def __init__(self, inp, oup, ker=3, stride=1):
        super().__init__()
        self.conv = nn.Sequential(*(_conv_bn(inp, inp, ker, stride, inp, nn.ReLU)
                                    + [nn.Conv2d(inp, oup, 1, 1, 0, bias=False)]))

    def forward(self, x):
        return self.conv(x)


class LitePose(EngineModule):
    def __init__(self, cfg, width_mult=1.0, round_nearest=8, cfg_arch=None):
        super().__init__()
        self.cfg_arch = cfg_arch
        c = _make_divisible(cfg_arch['input_channel'] * width_mult, round_nearest)
        self.first = nn.Sequential(convbnrelu(3, 32, ker=3, stride=2),
                                   convbnrelu(32, 32, ker=3, stride=1, groups=32),
                                   nn.Conv2d(32, c, 1, 1, 0, bias=False),
                                   nn.BatchNorm2d(c))
        self.channel = [c]
        stages = []
        for st in cfg_arch['backbone_setting']:
            cout = _make_divisible(st['channel'] * width_mult, round_nearest)
            blocks = []
            for b in range(st['num_blocks']):
                t, k = st['block_setting'][b]
                blocks.append(InvBottleneck(c, cout, st['stride'] if b == 0 else 1, ker=k, exp=t))
                c = cout
            stages.append(nn.Sequential(*blocks))
            self.channel.append(cout)
        self.stage = nn.ModuleList(stages)
        extra = cfg.MODEL.EXTRA
        self.filters = cfg_arch['deconv_setting']
        self.inplanes = self.channel[-1]
        self.num_deconv_layers = extra.NUM_DECONV_LAYERS
        refined, raw, bnrelu = [], [], []
        for i in range(self.num_deconv_layers):
            k = extra.NUM_DECONV_KERNELS[i]
            if k != 4:
                raise ValueError("LitePose fusion deconv uses 4x4 stride-2 kernels (got %d)" % k)
            planes = self.filters[i]
            refined.append(nn.ConvTranspose2d(self.inplanes, planes, 4, 2, 1, 0, bias=False))
            raw.append(nn.ConvTranspose2d(self.channel[-i - 2], planes, 4, 2, 1, 0, bias=False))
            bnrelu.append(nn.Sequential(nn.BatchNorm2d(planes), nn.ReLU(inplace=True)))
            self.inplanes = planes
        self.deconv_refined, self.deconv_raw = nn.ModuleList(refined), nn.ModuleList(raw)
        self.deconv_bnrelu = nn.ModuleList(bnrelu)
        dim_tag = cfg.MODEL.NUM_JOINTS if cfg.MODEL.TAG_PER_JOINT else 1
        f_ref, f_raw, self.final_channel = [], [], []
        for i in range(1, self.num_deconv_layers):
            oup = (cfg.MODEL.NUM_JOINTS if cfg.LOSS.WITH_HEATMAPS_LOSS[i - 1] else 0) + \
                  (dim_tag if cfg.LOSS.WITH_AE_LOSS[i - 1] else 0)
            f_ref.append(SepConv2d(self.filters[i], oup, ker=5))
            f_raw.append(SepConv2d(self.channel[-i - 3], oup, ker=5))
            self.final_channel.append(oup)
        self.final_refined, self.final_raw = nn.ModuleList(f_ref), nn.ModuleList(f_raw)
        self.loss_config = cfg.LOSS
        self._lp_cache = _EngineCache()

    # -- forward -------------------------------------------------------------
    def _forward_modules(self, x):
        x = self.first(x)
        feats = [x]
        for st in self.stage:
            feats.append(st(feats[-1]))
        outs = []
        refined, raw = feats[-1], feats[-2]
        for i in range(self.num_deconv_layers):
            refined = self.deconv_bnrelu[i](self.deconv_refined[i](refined) + self.deconv_raw[i](raw))
            raw = feats[-i - 3]
            if i > 0:
                outs.append(self.final_refined[i - 1](refined) + self.final_raw[i - 1](raw))
        return outs


def get_pose_net(cfg, is_train=False, cfg_arch=None):
    model = LitePose(cfg, cfg_arch=cfg_arch)
    if is_train and cfg.MODEL.INIT_WEIGHTS:
        print(cfg.MODEL.PRETRAINED)
        if os.path.isfile(cfg.MODEL.PRETRAINED):
            print("load pre-train model")
            state = torch.load(cfg.MODEL.PRETRAINED, map_location=torch.device('cpu'))
            keep = {k: v for k, v in state.items() if 'deconv' not in k and 'final' not in k}
            try:
                model.load_state_dict(keep, strict=False)
            except Exception:
                print("Error load!")
    return model
