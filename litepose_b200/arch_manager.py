"""The LitePose super-network's architecture sampler (reference arch_manager.py), restated in the package.

``SuperLitePose`` (litepose_b200/lib/models/pose_supermobilenet.py) owns one ``ArchManager`` as ``model.arch_manager``;
its forward asks it for the architecture to run.  The search side of the reference (calibrate_test.py, arch_search/)
sets ``is_search`` and ``search_arch`` to evaluate one candidate.  Attributes and draws are the reference's: every
``rand(c)`` is one ``random.randint(0, c - 1)`` call, in the same order, so a seeded ``random`` gives the same
architectures and leaves the same state behind."""
import random


def rand(c):
    return random.randint(0, c - 1)


def _make_divisible(v, divisor, min_value=None):
    floor = divisor if min_value is None else min_value
    out = max(floor, (int(v + divisor / 2) // divisor) * divisor)
    return out + divisor if out < 0.9 * v else out


class ArchManager(object):
    def __init__(self, cfg):
        self.cfg = cfg
        self.expansion = [6]
        self.kernel_size = [7]
        self.input_channel = 24
        self.width_mult = [1.0, 0.75, 0.5, 0.25]
        self.deconv_setting = cfg.MODEL.EXTRA.NUM_DECONV_FILTERS
        self.is_search = False
        self.search_arch = None
        # c, n, s of every stage: widest channel count, blocks drawn (fewer than the supernet holds), stride
        self.arch_setting = [[32, 4, 2], [64, 6, 2], [96, 8, 2], [160, 8, 1]]

    def rand_kernel_size(self):
        return self.kernel_size[rand(len(self.kernel_size))]

    def rand_expansion(self):
        return self.expansion[rand(len(self.expansion))]

    def rand_channel(self, c):
        return _make_divisible(c * self.width_mult[rand(len(self.width_mult))], 8)

    def _arch(self, img_size, channel, deconv):
        """cfg_arch dict of the mobile_configs JSON format; ``channel(c)`` gives a stage's width from its widest"""
        arch = {"img_size": img_size, "input_channel": channel(self.input_channel),
                "deconv_setting": [deconv(c) for c in self.deconv_setting], "backbone_setting": []}
        for c, n, s in self.arch_setting:
            arch["backbone_setting"].append({"num_blocks": n, "stride": s, "channel": channel(c),
                                             "block_setting": [[6, 7] for _ in range(n)]})
        return arch

    def random_sample(self):
        """``search_arch`` when searching, else a fresh draw: image size, stem width, the three deconv widths, then
        each stage's width (one ``randint`` each, in that order)"""
        if self.is_search:
            return self.search_arch
        return self._arch(256 + 64 * rand(5), self.rand_channel, self.rand_channel)

    def fixed_sample(self, reso=256, ratio=0.5):
        """every width scaled by ``ratio``; consumes no randomness"""
        def scaled(c):
            return _make_divisible(c * ratio, 8)
        return self._arch(reso, scaled, scaled)
