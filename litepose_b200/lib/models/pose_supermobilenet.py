"""Drop-in replacement of the reference's ``lib/models/pose_supermobilenet.py``: the LitePose super-network.

LitePose-XS...L are sub-networks of one weight-sharing super-network; the reference evaluates a sub-architecture
straight from the supernet checkpoint (valid.py --cfg supermobile.yaml --superconfig <arch>.json, calibrate_test.py's
architecture search).  ``get_pose_net(cfg, is_train=False)`` returns a ``SuperLitePose`` whose parameter/buffer names,
shapes and creation order equal the reference's (pose_supermobilenet.py:23-63, layers/super_layers.py:19-191), so
``load_state_dict(strict=True)``, ``network_to_half``, ``copy.deepcopy`` and seeded initialisation behave as there.
``model.arch_manager`` is the package's restatement of the reference's ``ArchManager`` (litepose_b200.arch_manager).

``forward`` asks ``arch_manager.random_sample()`` for the architecture once per call, as the reference does (its
``search_arch`` when ``is_search`` is set).  In eval mode on a CUDA tensor it then runs that sub-network on the sm_90a
kernels: ``litepose_b200.subnet.derive_supernet_subnet`` applies the supernet's rules (prefix slices, the k = 5 / 3
depthwise transform, its own strides and identity adds) and a ``LitePoseEngine`` runs the result; engines are cached
per (device, architecture), a few at a time.  CPU tensors and training mode run the module tree; after
``litepose_b200.train_dw.convert_depthwise`` its depthwise convolutions, the functional ones of ``SuperSepConv2d`` and
``SuperInvBottleneck`` included, run on the training kernels for CUDA tensors.

``lp_recalibrate_bn(x)`` is the search's BN recalibration pass (calibrate_test.py: ``model.train(); model(images)``) on
the kernels: it does to the module's BatchNorm buffers what a train-mode forward does, without autograd, and returns
what that forward returns (litepose_b200.bn_train).

One deviation: the reference's ``SuperConvTranspose2d.forward`` calls ``_output_padding`` with the argument list of
torch 1.x, which raises ``TypeError`` on torch >= 2.0 (the method gained ``num_spatial_dims``), so the reference module
cannot run a forward at all there.  This module passes the new arguments and gets the value the call was written for:
the layer's own ``output_padding`` (0) when no ``output_size`` is given.
"""
import json
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from litepose_b200.arch_manager import ArchManager, _make_divisible
from litepose_b200.train_dw import DepthwiseConv2d
from ._engine_module import EngineModule, _EngineCache
from .pose_mobilenet import convbnrelu

# engines kept per module: a search evaluates one candidate after another, a training run draws a new one per step
ENGINE_LRU = 4
# train-mode plans kept per module (BN recalibration): one per (device, architecture, input shape)
TRAIN_PLAN_LRU = 4


class SuperBatchNorm2d(nn.BatchNorm2d):
    """BatchNorm over the leading channels of its parameters and statistics (those the input has)"""

    def forward(self, x):
        c = x.shape[1]
        return F.batch_norm(x, self.running_mean[:c], self.running_var[:c], self.weight[:c], self.bias[:c],
                            self.training, self.momentum, self.eps)


class SuperConv2d(nn.Conv2d):
    """Conv2d with weight[:num_channel, :in]"""

    def forward(self, x, num_channel):
        w = self.weight[:num_channel, :x.shape[1]]
        b = None if self.bias is None else self.bias[:num_channel]
        return F.conv2d(x, w, b, self.stride, self.padding, self.dilation, self.groups)


class SuperConvTranspose2d(nn.ConvTranspose2d):
    """ConvTranspose2d with weight[:in, :num_channel] (the module-docstring deviation is here)"""

    def forward(self, x, num_channel, output_size=None):
        pad = self._output_padding(x, output_size, self.stride, self.padding, self.kernel_size, 2, self.dilation)
        w = self.weight[:x.shape[1], :num_channel]
        b = None if self.bias is None else self.bias[:num_channel]
        return F.conv_transpose2d(x, w, b, self.stride, self.padding, pad, self.groups, self.dilation)


class SuperSepConv2d(nn.Module):
    """k x k depthwise on the input's channels + BN + ReLU, then a bias-free 1x1 to ``num_channel``"""

    def __init__(self, inp, oup, ker=3, stride=1):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(inp, inp, ker, stride, ker // 2, groups=inp, bias=False),
                                  SuperBatchNorm2d(inp), nn.ReLU(inplace=True),
                                  nn.Conv2d(inp, oup, 1, 1, 0, bias=False))

    def forward(self, x, num_channel):
        c = x.shape[1]
        dw, pw = self.conv[0], self.conv[3]
        if isinstance(dw, DepthwiseConv2d):     # convert_depthwise: the training kernels on CUDA tensors
            x = dw.forward_weight(x, dw.weight[:c])
        else:
            x = F.conv2d(x, dw.weight[:c], None if dw.bias is None else dw.bias[:c], dw.stride, dw.padding, dw.dilation,
                         c)
        x = self.conv[2](self.conv[1](x))
        return F.conv2d(x, pw.weight[:num_channel, :c], None if pw.bias is None else pw.bias[:num_channel],
                        pw.stride, pw.padding, pw.dilation, pw.groups)


class SuperInvBottleneck(nn.Module):
    """Inverted residual at expansion <= 6 and depthwise kernel 7, 5 or 3.  Smaller kernels take the centre of the 7x7
    weight through this block's Linear5x5 / Linear3x3.  Stride and identity add are fixed here, from the widest
    channel counts."""
    expansion = 6
    ker_size = 7

    def __init__(self, inplanes, planes, stride=1):
        super().__init__()
        mid = round(inplanes * self.expansion)
        self.inv = nn.Sequential(SuperConv2d(inplanes, mid, 1, 1, 0, bias=False), SuperBatchNorm2d(mid),
                                 nn.ReLU6(inplace=True))
        self.depth_conv = nn.Sequential(nn.Conv2d(mid, mid, self.ker_size, stride, self.ker_size // 2, groups=mid,
                                                  bias=False),
                                        SuperBatchNorm2d(mid), nn.ReLU6(inplace=True))
        self.point_conv = nn.Sequential(SuperConv2d(mid, planes, 1, 1, 0, bias=False), SuperBatchNorm2d(planes))
        self.stride = stride
        self.Linear5x5 = nn.Linear(25, 25)
        self.Linear3x3 = nn.Linear(9, 9)
        self.use_residual_connection = stride == 1 and inplanes == planes

    def forward(self, x, out_nc, ker_size, expansion):
        mid = round(int(x.shape[1]) * expansion)
        y = self.inv[2](self.inv[1](self.inv[0](x, mid)))
        conv = self.depth_conv[0]
        lo = self.ker_size // 2 - ker_size // 2
        w = conv.weight[:mid, :, lo:lo + ker_size, lo:lo + ker_size]
        lin = {5: self.Linear5x5, 3: self.Linear3x3}.get(ker_size)
        if lin is not None:
            w = lin(w.reshape(w.shape[0], w.shape[1], -1)).reshape(w.shape[0], w.shape[1], ker_size, ker_size)
        if isinstance(conv, DepthwiseConv2d):   # convert_depthwise: the training kernels on CUDA tensors
            y = conv.forward_weight(y, w)
        else:
            b = None if conv.bias is None else conv.bias[:mid]
            y = F.conv2d(y, w, b, conv.stride, ker_size // 2, conv.dilation, mid)
        y = self.depth_conv[2](self.depth_conv[1](y))
        y = self.point_conv[1](self.point_conv[0](y, out_nc))
        return y + x if self.use_residual_connection else y


def _arch_key(cfg_arch):
    """what selects a sub-network: widths, depths and block settings (image size and stride keys do not)"""
    return json.dumps([cfg_arch["input_channel"], list(cfg_arch["deconv_setting"])] +
                      [[st["num_blocks"], st["channel"], st["block_setting"][:st["num_blocks"]]]
                       for st in cfg_arch["backbone_setting"]])


class SuperLitePose(EngineModule):
    def __init__(self, cfg, width_mult=1.0, round_nearest=8):
        super().__init__()
        # t, c, n, s of the widest stages
        setting = [[6, 32, 6, 2], [6, 64, 8, 2], [6, 96, 10, 2], [6, 160, 10, 1]]
        c = _make_divisible(24 * width_mult, round_nearest)
        self.arch_manager = ArchManager(cfg)
        self.first = nn.Sequential(convbnrelu(3, 32, ker=3, stride=2),
                                   convbnrelu(32, 32, ker=3, stride=1, groups=32),
                                   SuperConv2d(32, c, 1, 1, 0, bias=False),
                                   SuperBatchNorm2d(c))
        self.channel = [c]
        stages = []
        for _, ch, n, s in setting:
            cout = _make_divisible(ch * width_mult, round_nearest)
            blocks = []
            for b in range(n):
                blocks.append(SuperInvBottleneck(c, cout, s if b == 0 else 1))
                c = cout
            stages.append(nn.Sequential(*blocks))
            self.channel.append(cout)
        self.stage = nn.ModuleList(stages)
        extra = cfg.MODEL.EXTRA
        self.inplanes = self.channel[-1]
        refined, raw, bnrelu = [], [], []
        for i in range(extra.NUM_DECONV_LAYERS):
            k = extra.NUM_DECONV_KERNELS[i]
            if k != 4:
                raise ValueError("LitePose fusion deconv uses 4x4 stride-2 kernels (got %d)" % k)
            planes = extra.NUM_DECONV_FILTERS[i]
            refined.append(SuperConvTranspose2d(self.inplanes, planes, 4, 2, 1, 0, bias=False))
            raw.append(SuperConvTranspose2d(self.channel[-i - 2], planes, 4, 2, 1, 0, bias=False))
            bnrelu.append(nn.Sequential(SuperBatchNorm2d(planes), nn.ReLU(inplace=True)))
            self.inplanes = planes
        self.deconv_refined, self.deconv_raw = nn.ModuleList(refined), nn.ModuleList(raw)
        self.deconv_bnrelu = nn.ModuleList(bnrelu)
        dim_tag = cfg.MODEL.NUM_JOINTS if cfg.MODEL.TAG_PER_JOINT else 1
        f_ref, f_raw, self.final_channel = [], [], []
        for i in range(1, extra.NUM_DECONV_LAYERS):
            oup = (cfg.MODEL.NUM_JOINTS if cfg.LOSS.WITH_HEATMAPS_LOSS[i - 1] else 0) + \
                  (dim_tag if cfg.LOSS.WITH_AE_LOSS[i - 1] else 0)
            f_ref.append(SuperSepConv2d(extra.NUM_DECONV_FILTERS[i], oup, ker=5))
            f_raw.append(SuperSepConv2d(self.channel[-i - 3], oup, ker=5))
            self.final_channel.append(oup)
        self.final_refined, self.final_raw = nn.ModuleList(f_ref), nn.ModuleList(f_raw)
        self.num_deconv_layers = extra.NUM_DECONV_LAYERS
        self.loss_config = cfg.LOSS
        self._lp_cache = _EngineCache()
        self._lp_train_cache = _EngineCache()

    # -- engine ----------------------------------------------------------------
    def lp_engine(self, device=None, cfg_arch=None):
        """The engine of sub-architecture ``cfg_arch`` (default: ``arch_manager.search_arch``, which needs
        ``arch_manager.is_search``: otherwise every forward runs a new architecture and there is none to bind)."""
        from litepose_b200.engine import LitePoseEngine
        from litepose_b200.subnet import derive_supernet_subnet
        if cfg_arch is None:
            if not self.arch_manager.is_search:
                raise ValueError("SuperLitePose runs a new architecture (arch_manager.random_sample()) on every forward "
                                 "unless arch_manager.is_search is set with search_arch the architecture to evaluate; "
                                 "set them, or pass cfg_arch")
            cfg_arch = self.arch_manager.search_arch

        def build(state, dev):
            sub = derive_supernet_subnet(state, cfg_arch)
            return LitePoseEngine(sub.state_dict, sub.arch, dev, residual=sub.residual, strides=sub.strides)

        key = self._lp_device_key(device) + (_arch_key(cfg_arch),)
        return self._lp_cached(key, build, capacity=ENGINE_LRU)

    # -- forward ---------------------------------------------------------------
    def forward(self, x):
        cfg_arch = self.arch_manager.random_sample()
        if x.is_cuda and not self.training:
            # CUDA inference: hand-written sm_90a kernels only (raises if the library is missing)
            return self.lp_engine(x.device, cfg_arch).run(x, flip=False, out_fp32=x.dtype != torch.float16, clone=True)
        return self._forward_modules(x, cfg_arch)

    # -- BN recalibration -------------------------------------------------------
    def lp_recalibrate_bn(self, x):
        """What ``model.train(); model(x)`` does to this module, on the sm_90a kernels, without autograd: one
        ``arch_manager.random_sample()`` (as ``forward``), then the sub-network's train-mode forward.  Every BatchNorm
        it runs takes the batch statistics (biased variance) for the normalisation and updates its running statistics
        to (1 - momentum) * running + momentum * batch statistic (unbiased variance), the leading [:c] slice of a
        SuperBatchNorm2d only; num_batches_tracked grows by one on the plain BatchNorm2d of first.0 / first.1 (the
        SuperBatchNorm2d call F.batch_norm, which does not count).  The train / eval mode is left as it is.

        x: NCHW CUDA tensor, fp32 (fp16 under network_to_half).  Returns the outputs of the train-mode forward (fp32,
        fp16 for an fp16 x; they do not require grad).  The new statistics are staged on the device and copied into the
        buffers only once all of them are finite: otherwise ``LitePoseError`` names the layers and no buffer changes.
        Raises ValueError for a CPU tensor, a BatchNorm with momentum None, one value per channel (N*H*W == 1) and
        shapes the kernels do not take."""
        from litepose_b200 import bn_train
        from litepose_b200._lib import LitePoseError
        cfg_arch = self.arch_manager.random_sample()
        if not torch.is_tensor(x) or x.dim() != 4 or x.shape[1] != 3 or x.dtype not in (torch.float16, torch.float32):
            raise ValueError("lp_recalibrate_bn takes an NCHW 3-channel fp32 or fp16 image batch, got %s"
                             % ((tuple(x.shape), x.dtype) if torch.is_tensor(x) else type(x).__name__,))
        names = bn_train.bn_names(cfg_arch)
        mods = [self.get_submodule(n) for n in names]
        for n, m in zip(names, mods):
            if m.momentum is None:
                raise ValueError("%s: momentum None (a cumulative average) is not supported; the supernet's "
                                 "F.batch_norm call cannot take it either" % n)
            if not m.track_running_stats:
                raise ValueError("%s keeps no running statistics to recalibrate" % n)
        n_, _, h, w = x.shape
        if h % 16 or w % 16:
            raise ValueError("LitePose input height/width must be multiples of 16, got %dx%d" % (h, w))
        if n_ * (h // 16) * (w // 16) <= 1:
            raise ValueError("input %s leaves one value per channel at the backbone's last stage; train-mode BatchNorm "
                             "needs more than one (N*H*W > 1)" % (tuple(x.shape),))
        if not x.is_cuda:
            raise ValueError("lp_recalibrate_bn runs on the GPU kernels: it needs a CUDA tensor (the module tree runs "
                             "CPU tensors: model.train(); model(x))")
        plan = self._lp_train_plan(x, cfg_arch, names, mods)
        running = [(m.running_mean[:c], m.running_var[:c]) for m, c in zip(mods, plan.channels)]
        outs, staged = plan.run(x, running)
        flags = plan.flags.cpu()
        if bool(flags.any()):
            bad = [n for n, f in zip(names, flags.tolist()) if f]
            raise LitePoseError("BN recalibration: non-finite batch statistics in %s (no buffer was changed)"
                                % ", ".join(bad))
        dst, src = [], []
        for i, (m, c) in enumerate(zip(mods, plan.channels)):
            o = int(plan.offs[i])
            dst += [m.running_mean[:c], m.running_var[:c]]
            src += [staged[2, o:o + c], staged[3, o:o + c]]
        with torch.no_grad():
            torch._foreach_copy_(dst, src)      # in place: the version counters move, so the eval engine repacks
            for m in mods:
                if not isinstance(m, SuperBatchNorm2d) and m.num_batches_tracked is not None:
                    m.num_batches_tracked.add_(1)
        return outs

    def _lp_train_plan(self, x, cfg_arch, names, mods):
        """The cached train-mode plan of ``cfg_arch`` at x's shape, rebuilt when a parameter or a BatchNorm's
        momentum / eps changed (the running statistics are read at every run)"""
        from litepose_b200 import bn_train
        from litepose_b200.subnet import derive_supernet_subnet
        key = self._lp_device_key(x.device) + (_arch_key(cfg_arch), tuple(x.shape), x.dtype)
        sig = hash(tuple((id(t), t.data_ptr(), t._version) for t in self.parameters()) +
                   tuple((m.momentum, m.eps) for m in mods))
        cache = self._lp_train_cache
        with cache.lock:
            hit = cache.engines.pop(key, None)
            if hit is None or hit[1] != sig:
                sub = derive_supernet_subnet(self.state_dict(), cfg_arch)
                params = {n: (m.momentum, m.eps) for n, m in zip(names, mods)}
                n, _, h, w = x.shape
                hit = (bn_train.BNTrainPlan(sub, params, x.device, n, h, w, x.dtype), sig)
            cache.engines[key] = hit
            while len(cache.engines) > TRAIN_PLAN_LRU:
                del cache.engines[next(iter(cache.engines))]
            return hit[0]

    def _forward_modules(self, x, cfg_arch):
        x = self.first[1](self.first[0](x))
        x = self.first[3](self.first[2](x, cfg_arch["input_channel"]))
        feats = [x]
        for stage, st in zip(self.stage, cfg_arch["backbone_setting"]):
            y = feats[-1]
            for bi in range(st["num_blocks"]):
                t, k = st["block_setting"][bi]
                y = stage[bi](y, st["channel"], k, t)
            feats.append(y)
        outs = []
        refined, raw = feats[-1], feats[-2]
        filters = cfg_arch["deconv_setting"]
        for i in range(self.num_deconv_layers):
            refined = self.deconv_bnrelu[i](self.deconv_refined[i](refined, filters[i]) +
                                            self.deconv_raw[i](raw, filters[i]))
            raw = feats[-i - 3]
            if i > 0:
                outs.append(self.final_refined[i - 1](refined, self.final_channel[i - 1]) +
                            self.final_raw[i - 1](raw, self.final_channel[i - 1]))
        return outs

    # -- pretrained initialisation (reference pose_supermobilenet.py:173-209) --
    @staticmethod
    def _permute_bn(bn, idx):
        """weight and bias only: the reference moves the running statistics for modules whose type is exactly
        BatchNorm1d / BatchNorm2d, which no SuperBatchNorm2d is.  A module converted by
        litepose_b200.train_bn.convert_batchnorm counts as the class it was converted from (``lp_base``)."""
        bn.weight.data = torch.index_select(bn.weight.data, 0, idx)
        bn.bias.data = torch.index_select(bn.bias.data, 0, idx)
        if getattr(type(bn), "lp_base", type(bn)) in (nn.BatchNorm1d, nn.BatchNorm2d):
            bn.running_mean.data = torch.index_select(bn.running_mean.data, 0, idx)
            bn.running_var.data = torch.index_select(bn.running_var.data, 0, idx)

    def re_organize_weights(self):
        """Order the channels of the stem output and of every stage but the last by importance (sum of |w| of the
        1x1 that reads them first, descending), so that prefix slices keep the most important ones."""
        def order(conv):
            return torch.sort(torch.sum(torch.abs(conv.weight.data), dim=(0, 2, 3)), dim=0, descending=True)[1]

        nxt = self.stage[0][0].inv[0]
        idx = order(nxt)
        self.first[2].weight.data = torch.index_select(self.first[2].weight.data, 0, idx)
        self._permute_bn(self.first[3], idx)
        nxt.weight.data = torch.index_select(nxt.weight.data, 1, idx)
        for si in range(len(self.stage) - 1):
            nxt = self.stage[si + 1][0].inv[0]
            idx = order(nxt)
            nxt.weight.data = torch.index_select(nxt.weight.data, 1, idx)
            for bi, blk in enumerate(self.stage[si]):
                self._permute_bn(blk.point_conv[1], idx)
                blk.point_conv[0].weight.data = torch.index_select(blk.point_conv[0].weight.data, 0, idx)
                if bi > 0:      # blocks after the first read the stage's channels (and add them back)
                    blk.inv[0].weight.data = torch.index_select(blk.inv[0].weight.data, 1, idx)


def get_pose_net(cfg, is_train=False):
    model = SuperLitePose(cfg)
    if is_train and cfg.MODEL.INIT_WEIGHTS:
        print(cfg.MODEL.PRETRAINED)
        if os.path.isfile(cfg.MODEL.PRETRAINED):
            print("load pre-train model")
            state = torch.load(cfg.MODEL.PRETRAINED, map_location=torch.device('cpu'))
            keep = {}
            for k, v in state.items():
                if 'final' in k or 'deconv' in k:
                    continue
                keep[k[7:] if 'module' in k else k] = v
            model.load_state_dict(keep, strict=False)
            model.re_organize_weights()
            print("re-organize success!")
    return model
