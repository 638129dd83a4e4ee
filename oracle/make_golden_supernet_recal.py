"""ORACLE (test infrastructure, not product code).

Generate tests/golden/supernet_recal_*.npz: the BN recalibration pass of the architecture search (calibrate_test.py:58-61,
``model.train(); model(images)``) run by the UNMODIFIED reference super-network (oracle/model_ref_supernet.build_reference,
its one torch-2 shim) on the CPU in fp32, for four architectures and three consecutive batches.

  supernet_recal_inputs.npz   the seeded weights' digest (the weights are rebuilt from the seed), the start state - every
                              BatchNorm's running_mean / running_var (perturbed, on a 2^-6 grid so the untouched suffixes
                              compress) and num_batches_tracked, concatenated in named_modules order - and the three
                              batches [3, 2, 3, 64, 96], fp16 values stored as fp16 (the fp32 and fp16 inputs are equal)
  supernet_recal_<arch>.npz   the architecture (JSON), the full-length concatenated buffers after each batch and the last
                              batch's two outputs; <arch> in search_XS, search_S, random_k53 (a seeded random_sample's
                              widths with 3 blocks of k = 5, 3, 5 per stage, seed stored), fixed_256_0.5

Run in the build container only:

    python -m oracle.make_golden_supernet_recal
"""
import json
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from litepose_b200 import synth  # noqa: E402
from litepose_b200.config import get_cfg  # noqa: E402
from oracle import refshim  # noqa: E402
from oracle.make_golden import OUT, sd_digest  # noqa: E402
from oracle.model_ref_supernet import build_reference, load_reference  # noqa: E402

HEIGHT, WIDTH, BATCH, STEPS = 64, 96, 2, 3


def bn_modules(model):
    return [(n, m) for n, m in model.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]


def perturb_(model, seed=5):
    """running statistics on a 2^-6 grid: mean in [-0.5, 0.5], var in [0.5, 1.5]; num_batches_tracked 5"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for _, m in bn_modules(model):
            c = m.num_features
            m.running_mean.copy_(torch.randint(-32, 33, (c,), generator=g).float() / 64)
            m.running_var.copy_(torch.randint(32, 97, (c,), generator=g).float() / 64)
            m.num_batches_tracked.fill_(5)


def state(model):
    mods = bn_modules(model)
    return (torch.cat([m.running_mean for _, m in mods]).numpy().copy(),
            torch.cat([m.running_var for _, m in mods]).numpy().copy(),
            np.array([int(m.num_batches_tracked) for _, m in mods], np.int64))


def random_k53(am, seed=1):
    """the widths of the draw random_sample makes after random.seed(seed), with 3 blocks per stage and kernels
    5, 3, 5 (the draws themselves are all k = 7, t = 6): both depthwise transforms of the supernet run"""
    random.seed(seed)
    arch = am.random_sample()
    for st in arch["backbone_setting"]:
        st["num_blocks"], st["block_setting"] = 3, [[6, 5], [6, 3], [6, 5]]
    return seed, arch


def golden_supernet_recal():
    refshim.load()
    _, arch_manager = load_reference()
    cfg = get_cfg(input_size=HEIGHT)
    am = arch_manager.ArchManager(cfg)

    def search(name):
        with open(os.path.join(refshim.REF_ROOT, "mobile_configs", "search-%s.json" % name)) as f:
            return json.load(f)

    seed, drawn = random_k53(am)
    cases = [("search_XS", search("XS"), -1), ("search_S", search("S"), -1), ("random_k53", drawn, seed),
             ("fixed_256_0.5", am.fixed_sample(256, 0.5), -1)]
    batches = torch.stack([synth.make_frames(BATCH, HEIGHT, seed=31 + i, width=WIDTH).half() for i in range(STEPS)])
    model = build_reference(cfg)
    digest = sd_digest(model.state_dict())
    perturb_(model)
    start = state(model)
    np.savez_compressed(os.path.join(OUT, "supernet_recal_inputs.npz"), digest=np.array(digest),
                        running_mean=start[0], running_var=start[1], num_batches_tracked=start[2],
                        batches=batches.numpy())
    for name, arch, seed in cases:
        model = build_reference(cfg)
        perturb_(model)
        model.arch_manager.is_search, model.arch_manager.search_arch = True, arch
        model.train()
        rm, rv, nbt = [], [], []
        with torch.no_grad():
            for i in range(STEPS):
                outs = model(batches[i].float())
                s = state(model)
                rm.append(s[0])
                rv.append(s[1])
                nbt.append(s[2])
        np.savez_compressed(os.path.join(OUT, "supernet_recal_%s.npz" % name), arch=np.array(json.dumps(arch)),
                            seed=np.array(seed), running_mean=np.stack(rm), running_var=np.stack(rv),
                            num_batches_tracked=np.stack(nbt), out0=outs[0].numpy(), out1=outs[1].numpy())


if __name__ == "__main__":
    torch.set_num_threads(8)
    golden_supernet_recal()
    for f in sorted(os.listdir(OUT)):
        if f.startswith("supernet_recal_"):
            print(f, os.path.getsize(os.path.join(OUT, f)))
