"""Time the pipeline's two grouping modes with the demo's settings (flip test, adjust and refine off), three arms on the
same frames and planted crowd:

  1. ae        LitePosePipeline(grouping="ae").step_device           (graph: network + glue + evaluation parser)
  2. fast      LitePosePipeline(grouping="fast").step_device         (graph: network + glue + peak finder + KM assign)
  3. stitched  the ae step, then fast_utils.group.HeatmapParser.parse_batch on the step's det / tag (by hand, outside the
               graph: what a user had to write before the fast mode existed)

    python tools/time_fast.py [--arch S] [--size 512] [--batch 32] [--people 5] [--iters 20] [--rounds 5] [--out f.json]

Each arm is warmed up (plans, graph capture), then timed with CUDA events around ``--iters`` back-to-back steps; the
arms alternate for ``--rounds`` rounds and the median per-step time of each arm is reported (with the spread), next to
the card's name and power limit.  Before timing, the fast step's payload is checked against parse_batch on the same
maps (element for element), so the numbers belong to a correct result."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from litepose_b200 import _lib, synth  # noqa: E402
from litepose_b200.config import get_arch, get_cfg  # noqa: E402
from litepose_b200.fast_utils.group import HeatmapParser as FastParser  # noqa: E402
from litepose_b200.lib.models.pose_mobilenet import get_pose_net  # noqa: E402
from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd  # noqa: E402


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
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--people", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_fast.py needs a CUDA device")
    cfg = get_cfg(input_size=a.size, flip_test=False, adjust=False, refine=False)
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch(a.arch)), 1)).eval().cuda()
    ae = LitePosePipeline(model, cfg, use_graphs=True, grouping="ae")
    fast = LitePosePipeline(model, cfg, use_graphs=True, grouping="fast")
    parser = FastParser(cfg)
    x = synth.make_frames(a.batch, a.size, seed=1234).half().cuda()
    plant = PlantedCrowd(a.batch, 14, a.size, a.size, 1, num_people=a.people, seed=77, device="cuda")

    def stitched():
        ae.step_device(x, plant)
        st = ae._get_state(a.batch, a.size, a.size, x.dtype, plant)
        return parser.parse_batch(st["det"], st["tag"])

    arms = {"ae": lambda: ae.step_device(x, plant), "fast": lambda: fast.step_device(x, plant), "stitched": stitched}
    for fn in arms.values():                      # warm-up: plans, graph capture, buffers
        fn()
    torch.cuda.synchronize()

    # the fast step's payload == parse_batch on the maps of the same step
    packed = fast.step_device(x, plant).cpu().numpy()
    st = fast._get_state(a.batch, a.size, a.size, x.dtype, plant)
    num, ans = [t.cpu().numpy() for t in parser.parse_batch(st["det"], st["tag"])]
    M, J = fast.fast["M"], fast.params.num_joints
    ok = bool(np.array_equal(packed[:, :-2].reshape(a.batch, M, J, 4), ans) and np.array_equal(packed[:, -2], num)
              and (packed[:, -1] == 0).all())
    if not ok:
        raise SystemExit("fast step payload differs from parse_batch on the same maps")

    lib = _lib.load()
    launches = {}
    for name, fn in arms.items():
        l0 = lib.lp_launch_count()
        fn()
        launches[name] = int(lib.lp_launch_count() - l0)     # host-side launches (0 inside a replayed graph)
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.iters)
    res = {}
    for name, t in times.items():
        ms = float(np.median(t))
        res[name] = {"ms_per_step": round(ms, 3), "frames_per_s": round(a.batch / ms * 1e3, 1),
                     "ms_min": round(min(t), 3), "ms_max": round(max(t), 3), "host_launches_per_step": launches[name]}
    name, pl = card()
    out = {"card": name, "power_limit": pl, "arch": a.arch, "input_size": a.size, "batch": a.batch,
           "people": a.people, "settings": "flip test, adjust, refine off", "persons_found": num[:8].tolist(),
           "iters": a.iters, "rounds": a.rounds, "fast_payload_equals_parse_batch": ok, "arms": res}
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
