"""The BN recalibration goldens (tests/golden/supernet_recal_*.npz, oracle/make_golden_supernet_recal.py) as test inputs:
the seeded super-network with the goldens' start state, the batches, and per architecture the buffers after each batch
(test infrastructure)."""
import json
import os

import numpy as np
import torch

from litepose_b200 import synth
from litepose_b200.config import get_cfg
from litepose_b200.lib.models import pose_supermobilenet

ARCHS = ["search_XS", "search_S", "random_k53", "fixed_256_0.5"]
SIZE = 64      # the goldens' batches are 2 x 3 x 64 x 96 (the config's input size builds the same module)
# The kernel path keeps every raw pre-BN tensor in fp16, the module tree in fp32.  The statistics of the stem and of
# stages 0 and 1 stay within 0.3x the model tolerance 2e-3 max|ref| + 1e-4 of the reference's, but in training mode every
# layer renormalises with the batch's own statistics, and through the 30-60 BatchNorms of a random-weight super-network
# at 2 x 64 x 96 (48 values per channel in stage 3) those differences grow to a few percent of the batch variance.  The
# running variances of the last stage-3 expansions and the outputs then differ from the reference by up to ~11x the
# model tolerance (random_k53 out0 10.7x, search_S stage.3.9.inv.1 9.4x).
TOL_FACTOR = 12.0


def bn_modules(model):
    return [(n, m) for n, m in model.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]


def inputs(golden_dir):
    return np.load(os.path.join(golden_dir, "supernet_recal_inputs.npz"))


def golden(golden_dir, name):
    z = np.load(os.path.join(golden_dir, "supernet_recal_%s.npz" % name))
    return z, json.loads(str(z["arch"]))


def load_state_(model, rm, rv, nbt):
    """set every BatchNorm's buffers from the goldens' concatenated (named_modules order) arrays"""
    o = 0
    with torch.no_grad():
        for i, (_, m) in enumerate(bn_modules(model)):
            c = m.num_features
            m.running_mean.copy_(torch.from_numpy(rm[o:o + c]))
            m.running_var.copy_(torch.from_numpy(rv[o:o + c]))
            m.num_batches_tracked.fill_(int(nbt[i]))
            o += c
    return model


def state(model):
    mods = bn_modules(model)
    return (torch.cat([m.running_mean.detach().float().cpu() for _, m in mods]).numpy(),
            torch.cat([m.running_var.detach().float().cpu() for _, m in mods]).numpy(),
            np.array([int(m.num_batches_tracked) for _, m in mods], np.int64))


def supernet(golden_dir, arch):
    """the seeded SuperLitePose (the goldens' digest is checked by the caller) at the start state, searching ``arch``"""
    torch.manual_seed(0)
    m = synth.randomize_bn_(pose_supermobilenet.get_pose_net(get_cfg(input_size=SIZE)), 1)
    z = inputs(golden_dir)
    load_state_(m, z["running_mean"], z["running_var"], z["num_batches_tracked"])
    m.arch_manager.is_search, m.arch_manager.search_arch = True, arch
    return m


def used(model, arch):
    """{BatchNorm name: (offset into the concatenated buffers, channels the sub-network uses)}, plan order"""
    from litepose_b200.bn_train import bn_names
    from litepose_b200.subnet import derive_supernet_subnet
    sd = derive_supernet_subnet(model.state_dict(), arch).state_dict
    offs, o = {}, 0
    for n, m in bn_modules(model):
        offs[n] = o
        o += m.num_features
    return {n: (offs[n], int(sd[n + ".weight"].shape[0])) for n in bn_names(arch)}


def tol_used(got, ref):
    """fraction of the model tolerance 2e-3 max|ref| + 1e-4 that |got - ref| uses"""
    ref = np.asarray(ref, np.float64)
    lim = 2e-3 * np.abs(ref).max() + 1e-4
    return float(np.abs(np.asarray(got, np.float64) - ref).max() / lim)
