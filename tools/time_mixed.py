"""Time the evaluation loop on a mixed list of image sizes, three ways in one run:

  1. per image   one infer_images call per image (batch 1: what valid.py does)
  2. per bucket  one infer_images call per source size (host bucketing on the equal-size path)
  3. mixed       ONE infer_images call on the whole list (size groups + ragged warp / parser)

    python tools/time_mixed.py [--arch S] [--size 512] [--images 32] [--iters 5] [--out time_mixed.json]

The list is seeded: COCO-like landscape and portrait sizes that fall into at least five network-size groups at
INPUT_SIZE 512.  Every image holds planted persons (a random-weight network detects nobody), so the parser does real
work.  Each arm: one warm-up pass (plans, graphs, buffers), then ``--iters`` timed passes, each a host clock around
blocking calls (every infer_images call ends in a device synchronise); the median is reported with frames/s, ms per
list and kernel launches per list (lp_launch_count), beside the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from litepose_b200 import _lib, synth  # noqa: E402
from litepose_b200.config import get_arch, get_cfg  # noqa: E402
from litepose_b200.lib.models.pose_mobilenet import get_pose_net  # noqa: E402
from litepose_b200.mixed import MixedPlan  # noqa: E402
from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd  # noqa: E402

# source sizes (H, W): landscape and portrait; at INPUT_SIZE 512 they map to 512x704, 704x512, 512x768, 768x512,
# 512x832 and 512x512 network inputs
POOL = [(480, 640), (640, 480), (427, 640), (640, 427), (333, 500), (612, 612), (375, 500), (500, 375)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # noqa: BLE001 - the number is reported as unknown, never guessed
        pl = "unknown (%s)" % e
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="S")
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_mixed.py needs a CUDA device")
    rng = np.random.RandomState(a.seed)
    shapes = [POOL[k] for k in rng.randint(0, len(POOL), a.images)]
    imgs = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    cfg = get_cfg(input_size=a.size)
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch(a.arch)), 1)).eval()
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True)
    J, T = pipe.params.num_joints, 2 if pipe.flip else 1
    mp = MixedPlan(shapes, pipe.scales, a.size, pipe.project, J, T)
    det_hw = [tuple(int(v) for v in mp.det_hw[mp.pos[i]]) for i in range(len(shapes))]
    plants = [PlantedCrowd(1, J, h, w, T, num_people=5, seed=100 + i) for i, (h, w) in enumerate(det_hw)]
    buckets = {}
    for i, s in enumerate(shapes):
        buckets.setdefault(s, []).append(i)
    b_in = {s: torch.from_numpy(np.stack([imgs[i] for i in idx])).pin_memory() for s, idx in buckets.items()}
    b_plant = {s: PlantedCrowd(len(idx), J, det_hw[idx[0]][0], det_hw[idx[0]][1], T, num_people=5, seed=7)
               for s, idx in buckets.items()}
    one = [torch.from_numpy(im)[None].pin_memory() for im in imgs]

    arms = {
        "per_image": lambda: [pipe.infer_images(one[i], plant=plants[i]) for i in range(len(imgs))],
        "per_bucket": lambda: [pipe.infer_images(b_in[s], plant=b_plant[s]) for s in buckets],
        "mixed": lambda: pipe.infer_images(imgs, plant=plants),
    }
    lib = _lib.load()
    res = {}
    for name, fn in arms.items():
        fn()                                          # warm-up: plans, graphs, grow-only buffers
        torch.cuda.synchronize()
        times, launches = [], []
        for _ in range(a.iters):
            l0 = lib.lp_launch_count()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            launches.append(int(lib.lp_launch_count() - l0))
        ms = float(np.median(times)) * 1e3
        res[name] = {"ms_per_list": round(ms, 2), "frames_per_s": round(len(imgs) / ms * 1e3, 1),
                     "launches_per_list": int(np.median(launches)), "ms_all": [round(t * 1e3, 2) for t in times]}
    name, pl = card()
    out = {"card": name, "power_limit": pl, "arch": a.arch, "input_size": a.size, "images": len(imgs),
           "size_groups": len(mp.groups), "source_buckets": len(buckets),
           "group_sizes": [[list(g.key[0]), g.n] for g in mp.groups], "arms": res}
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
