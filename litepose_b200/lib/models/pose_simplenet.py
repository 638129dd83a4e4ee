"""Drop-in replacement of the reference's ``lib/models/pose_simplenet.py``: LitePose without the Fusion Deconv Head.

The paper's head ablation: the stem and inverted-residual stages of ``pose_mobilenet``, but every deconv level is
``deconv_bnrelu[i](deconv_refined[i](refined))`` and every output ``final_refined[i-1](refined)`` alone - no
``deconv_raw`` / ``final_raw`` modules (reference lib/models/pose_simplenet.py:20-155).  Parameter/buffer names,
shapes and creation order equal the reference's, so ``load_state_dict(strict=True)``, ``network_to_half``,
``copy.deepcopy`` and seeded initialisation behave as there.  As for ``pose_mobilenet``, eval-mode forward on a CUDA
tensor runs the sm_90a kernels (litepose_b200.engine recognises the single-branch state_dict); CPU tensors and
training run the module tree.
"""
import os

import torch
import torch.nn as nn

from ._engine_module import EngineModule, _EngineCache
from .pose_mobilenet import InvBottleneck, SepConv2d, _make_divisible, convbnrelu


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
        refined, bnrelu = [], []
        for i in range(extra.NUM_DECONV_LAYERS):
            k = extra.NUM_DECONV_KERNELS[i]
            if k != 4:
                raise ValueError("LitePose fusion deconv uses 4x4 stride-2 kernels (got %d)" % k)
            planes = self.filters[i]
            refined.append(nn.ConvTranspose2d(self.inplanes, planes, 4, 2, 1, 0, bias=False))
            bnrelu.append(nn.Sequential(nn.BatchNorm2d(planes), nn.ReLU(inplace=True)))
            self.inplanes = planes
        self.deconv_refined, self.deconv_bnrelu = nn.ModuleList(refined), nn.ModuleList(bnrelu)
        dim_tag = cfg.MODEL.NUM_JOINTS if cfg.MODEL.TAG_PER_JOINT else 1
        f_ref, self.final_channel = [], []
        for i in range(1, extra.NUM_DECONV_LAYERS):
            oup = (cfg.MODEL.NUM_JOINTS if cfg.LOSS.WITH_HEATMAPS_LOSS[i - 1] else 0) + \
                  (dim_tag if cfg.LOSS.WITH_AE_LOSS[i - 1] else 0)
            f_ref.append(SepConv2d(self.filters[i], oup, ker=5))
            self.final_channel.append(oup)
        self.final_refined = nn.ModuleList(f_ref)
        self.num_deconv_layers = extra.NUM_DECONV_LAYERS
        self.loss_config = cfg.LOSS
        self._lp_cache = _EngineCache()

    def _forward_modules(self, x):
        x = self.first(x)
        feats = [x]
        for st in self.stage:
            feats.append(st(feats[-1]))
        outs = []
        refined = feats[-1]
        for i in range(self.num_deconv_layers):
            refined = self.deconv_bnrelu[i](self.deconv_refined[i](refined))
            if i > 0:
                outs.append(self.final_refined[i - 1](refined))
        return outs


def get_pose_net(cfg, is_train=False, cfg_arch=None):
    model = LitePose(cfg, cfg_arch=cfg_arch)
    if is_train and cfg.MODEL.INIT_WEIGHTS:
        print(cfg.MODEL.PRETRAINED)
        if os.path.isfile(cfg.MODEL.PRETRAINED):
            print("load pre-train model")
            state = torch.load(cfg.MODEL.PRETRAINED)
            keep = {k: v for k, v in state.items() if 'deconv' not in k and 'final' not in k}
            model.load_state_dict(keep, strict=False)
    return model
