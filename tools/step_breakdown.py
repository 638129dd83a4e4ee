"""Per-kernel breakdown of one benchmark-configuration step (LitePose-S 512x512, batch 32, flip + glue + parser) under
torch.profiler with CUDA activities: total device time, launches and share of the step per kernel name.

The step runs without CUDA graphs so that every launch is its own trace record; kernel times are those of the graphed
step, the gaps between kernels are not.  As in the benchmark, the plain and the mirrored pass are two batch-N launch
sequences on two streams.  Numbers printed under the profiler are a breakdown, not bench values.  ``--demo`` takes the
demo's settings (flip test, adjust and refine off), ``--grouping fast`` the pipeline's fast grouping mode."""
import argparse
import collections
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from litepose_b200 import synth  # noqa: E402
from litepose_b200.config import get_arch, get_cfg  # noqa: E402
from litepose_b200.lib.models.pose_mobilenet import get_pose_net  # noqa: E402
from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd  # noqa: E402


def gpu_info(index=0):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, limit = [v.strip() for v in r.stdout.strip().split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(index), "unknown"


def short(name, width=96):
    return name if len(name) <= width else name[:width - 3] + "..."


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="S")
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--people", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5, help="profiled steps; totals are per step")
    ap.add_argument("--out", default=None, help="also write the table to this file")
    ap.add_argument("--demo", action="store_true", help="the demo's settings: flip test, adjust and refine off")
    ap.add_argument("--grouping", default="ae", choices=["ae", "fast"], help="the pipeline's grouping mode")
    a = ap.parse_args()

    dev = torch.device("cuda", 0)
    if a.demo:
        cfg = get_cfg(input_size=a.size, flip_test=False, adjust=False, refine=False)
    else:
        cfg = get_cfg(input_size=a.size)
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch(a.arch)), 1)).eval().to(dev)
    pipe = LitePosePipeline(model, cfg, use_graphs=False, grouping=a.grouping)
    x = synth.make_frames(a.batch, a.size, seed=1234).half().to(dev)
    plant = PlantedCrowd(a.batch, 14, a.size, a.size, 2 if pipe.flip else 1, num_people=a.people, seed=77, device=dev)
    for _ in range(3):
        pipe.step_device(x, plant)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e0.record()
        for _ in range(a.steps):
            pipe.step_device(x, plant)
        e1.record()
        torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / a.steps

    tot = collections.defaultdict(float)
    cnt = collections.Counter()
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        tot[ev.name] += us
        cnt[ev.name] += 1
    kern_us = sum(tot.values()) / a.steps
    name, limit = gpu_info()
    lines = ["# %s, power limit %s" % (name, limit),
             "# LitePose-%s %dx%d batch %d, one step = %s + glue + %s parser, no CUDA graphs, %d steps profiled"
             % (a.arch, a.size, a.size, a.batch, "2 backbone passes (flip)" if pipe.flip else "1 backbone pass",
                a.grouping, a.steps),
             "# step wall time under the profiler %.3f ms; summed device time of all kernels/copies %.3f ms per step"
             % (step_ms, kern_us / 1e3),
             "# the plain and the mirrored pass run concurrently on two streams, so summed device time exceeds wall time"
             if pipe.flip else "# summed device time exceeds wall time where kernels overlap",
             "# share = kernel time / summed device time",
             "%10s %8s %7s  %s" % ("us/step", "launches", "share", "kernel")]
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        lines.append("%10.1f %8d %6.1f%%  %s" % (v / a.steps, cnt[k] // a.steps, 100.0 * v / a.steps / kern_us, short(k)))
    text = "\n".join(lines)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
