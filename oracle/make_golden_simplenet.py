"""ORACLE (test infrastructure, not product code).

Generate tests/golden/model_simplenet_{XS,S}_128.npz from the UNMODIFIED reference's lib/models/pose_simplenet.py
(LitePose without the Fusion Deconv Head, imported in place through oracle/refshim.py): the seeded state-dict digest,
the fp32 outputs and the outputs of the reference's network_to_half fp16 eager path, as oracle/make_golden.py does for
pose_mobilenet.  Run in the build container only:

    python -m oracle.make_golden_simplenet
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from litepose_b200 import synth  # noqa: E402
from litepose_b200.config import get_arch, get_cfg  # noqa: E402
from oracle import refshim  # noqa: E402
from oracle.make_golden import OUT, sd_digest  # noqa: E402
from oracle.model_ref_simplenet import build_reference  # noqa: E402


def golden_model_simplenet():
    ns = refshim.load()
    for name, size in (("XS", 128), ("S", 128)):
        cfg = get_cfg(input_size=size)
        arch = get_arch(name)
        model = build_reference(cfg, arch)
        x = synth.make_frames(1, size, seed=11)
        with torch.no_grad():
            outs = model(x)
            half = ns.fp16util.network_to_half(build_reference(cfg, arch))
            outs_h = half(x)
        np.savez_compressed(
            os.path.join(OUT, "model_simplenet_%s_%d.npz" % (name, size)),
            digest=np.array(sd_digest(model.state_dict())),
            out0=outs[0].numpy(), out1=outs[1].numpy(),
            out0_fp16eager=outs_h[0].numpy(), out1_fp16eager=outs_h[1].numpy())


if __name__ == "__main__":
    torch.set_num_threads(8)
    golden_model_simplenet()
    for f in sorted(os.listdir(OUT)):
        if f.startswith("model_simplenet_"):
            print(f, os.path.getsize(os.path.join(OUT, f)))
