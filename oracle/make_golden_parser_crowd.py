"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates tests/golden/parser_crowd_*.npz: the UNMODIFIED reference's
HeatmapParser.top_k and HeatmapParser.parse (lib/core/group.py, imported in place through oracle/refshim.py) on planted
crowds past 64 persons, at MAX_NUM_PEOPLE = K above 64 (adjust and refine on).  The reference's Munkres is pure
Python, O(n^3) per joint, so the three cases take minutes.  Needs a reference checkout:

    python -m oracle.make_golden_parser_crowd
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from litepose_b200 import synth  # noqa: E402
from litepose_b200.config import get_cfg  # noqa: E402
from oracle import refshim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

CROWD_CASES = [
    # name, K = MAX_NUM_PEOPLE, map side, T, planted persons, seed
    ("p80_k96_t2", 96, 384, 2, 80, 11),
    ("p150_k128_t1", 128, 448, 1, 150, 12),
    ("p240_k256_t2", 256, 512, 2, 240, 13),
]


def crowd_cfg(k):
    cfg = get_cfg(input_size=256)
    cfg.DATASET.MAX_NUM_PEOPLE = k
    return cfg


def crowd_inputs(case):
    name, k, side, t, people, seed = case
    cfg = crowd_cfg(k)
    return cfg, synth.plant_crowd(cfg.DATASET.NUM_JOINTS, side, side, t, num_people=people, seed=seed)


def digest(det, tag):
    return hashlib.sha256(det.tobytes() + tag.tobytes()).hexdigest()


def main():
    ns = refshim.load()
    torch.set_num_threads(1)
    for case in CROWD_CASES:
        name, t = case[0], case[3]
        cfg, (det, tag) = crowd_inputs(case)
        nj = cfg.DATASET.NUM_JOINTS
        dt, tt = torch.from_numpy(det)[None], torch.from_numpy(tag)[None]
        rp = ns.group.HeatmapParser(cfg)
        top = rp.top_k(dt, tt)
        ans, scores = rp.parse(dt.clone(), tt.clone(), True, True)
        path = os.path.join(OUT, "parser_crowd_%s.npz" % name)
        np.savez_compressed(path, in_digest=np.array(digest(det, tag)), val_k=top["val_k"], loc_k=top["loc_k"],
                            tag_k=top["tag_k"], ans=np.array(ans[0], dtype=np.float32).reshape(-1, nj, 3 + t),
                            scores=np.array(scores, dtype=np.float32))
        print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
