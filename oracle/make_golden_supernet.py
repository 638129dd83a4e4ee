"""ORACLE (test infrastructure, not product code).

Generate tests/golden/model_supernet_*.npz from the UNMODIFIED reference's lib/models/pose_supermobilenet.py (imported
in place through oracle/model_ref_supernet.load_reference, with its one torch-2 shim) at 128x128, batch 1.  Each file
holds the seeded state-dict digest (the weights themselves are rebuilt from the seed), the architecture as JSON, the
fp32 outputs and the outputs of the reference's network_to_half fp16 eager path, for:
  * search_XS, search_S        mobile_configs/search-{XS,S}.json
  * fixed_256_0.5              ArchManager.fixed_sample(256, 0.5)
  * random_seed{1,2}           the draw the forward itself makes after random.seed(s), plus the ``random`` state it
                               leaves (the Mersenne Twister words of random.getstate())
  * mixed                      a JSON architecture with [4,5] / [3,3] / [6,5] / [3,7] blocks, fewer blocks than the
                               supernet and equal stage-2 / stage-3 widths (stage 3 block 0 adds no identity there)
Run in the build container only:

    python -m oracle.make_golden_supernet
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

SIZE = 128
MIXED = {"img_size": 256, "input_channel": 16, "deconv_setting": [48, 24, 16], "backbone_setting": [
    {"num_blocks": 2, "stride": 2, "channel": 24, "block_setting": [[4, 5], [3, 3]]},
    {"num_blocks": 3, "stride": 2, "channel": 32, "block_setting": [[6, 5], [6, 7], [3, 7]]},
    {"num_blocks": 2, "stride": 2, "channel": 80, "block_setting": [[6, 7], [4, 5]]},
    {"num_blocks": 3, "stride": 1, "channel": 80, "block_setting": [[6, 7], [3, 3], [6, 5]]}]}


def cases(am):
    def search(name):
        with open(os.path.join(refshim.REF_ROOT, "mobile_configs", "search-%s.json" % name)) as f:
            return json.load(f)
    return [("search_XS", search("XS"), None), ("search_S", search("S"), None),
            ("fixed_256_0.5", am.fixed_sample(256, 0.5), None),
            ("random_seed1", None, 1), ("random_seed2", None, 2), ("mixed", MIXED, None)]


def run(model, x, arch, seed):
    """one forward of the reference: a fixed architecture through is_search, or the forward's own seeded draw"""
    am = model.arch_manager if hasattr(model, "arch_manager") else model[1].arch_manager
    am.is_search, am.search_arch = arch is not None, arch
    if seed is not None:
        random.seed(seed)
    with torch.no_grad():
        outs = model(x)
    return outs, random.getstate()


def golden_model_supernet():
    ns = refshim.load()
    _, arch_manager = load_reference()
    cfg = get_cfg(input_size=SIZE)
    model = build_reference(cfg)
    half = ns.fp16util.network_to_half(build_reference(cfg))
    x = synth.make_frames(1, SIZE, seed=11)
    for name, arch, seed in cases(arch_manager.ArchManager(cfg)):
        outs, state = run(model, x, arch, seed)
        outs_h, state_h = run(half, x, arch, seed)
        assert state == state_h
        if seed is not None:
            random.seed(seed)
            arch = arch_manager.ArchManager(cfg).random_sample()
            assert random.getstate() == state
        np.savez_compressed(
            os.path.join(OUT, "model_supernet_%s.npz" % name),
            digest=np.array(sd_digest(model.state_dict())), arch=np.array(json.dumps(arch)),
            seed=np.array(-1 if seed is None else seed), random_state=np.array(state[1], np.int64),
            out0=outs[0].numpy(), out1=outs[1].numpy(),
            out0_fp16eager=outs_h[0].numpy(), out1_fp16eager=outs_h[1].numpy())


if __name__ == "__main__":
    torch.set_num_threads(8)
    golden_model_supernet()
    for f in sorted(os.listdir(OUT)):
        if f.startswith("model_supernet_"):
            print(f, os.path.getsize(os.path.join(OUT, f)))
