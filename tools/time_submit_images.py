"""Time the asynchronous list API against the blocking list call on the same seeded mixed lists:

  1. sequential   one blocking infer_images(list) per list
  2. async        submit_images / collect_images with two lists in flight
  3. sharded      (under torchrun, R ranks) every list split by litepose_b200.dist.plan_shards, one NCCL gather per
                  list on rank 0, two lists in flight

    python tools/time_submit_images.py [--arch S] [--size 512] [--images 32] [--lists 8] [--rounds 5] [--out F]
    torchrun --nproc_per_node R tools/time_submit_images.py ...

The lists are seeded as in tools/time_mixed.py (COCO-like landscape and portrait sizes, at least five network-size
groups at INPUT_SIZE 512, planted persons in every image); each list has its own composition.  LitePose-S, flip test,
adjust + refine.  Arms 1 and 2 alternate for ``--rounds`` rounds after one warm-up pass each; every round is a host
clock around all lists that ends once every result is on the host.  The results of every arm are checked against arm
1, image for image.  Reported: medians of lists/s and frames/s, the host time spent inside submit_images per list, and
the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from litepose_b200 import synth  # noqa: E402
from litepose_b200.config import get_arch, get_cfg  # noqa: E402
from litepose_b200.lib.models.pose_mobilenet import get_pose_net  # noqa: E402
from litepose_b200.mixed import MixedPlan  # noqa: E402
from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd  # noqa: E402
from time_mixed import POOL, card  # noqa: E402


def same(a, b):
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if x[-1] != y[-1] or not np.array_equal(x[0], y[0]):
            return False
        if len(x) == 3 and not np.array_equal(np.asarray(x[1], np.float32), np.asarray(y[1], np.float32)):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="S")
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--lists", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_submit_images.py needs a CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    group = None
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl")
        group = dist.group.WORLD
    cfg = get_cfg(input_size=a.size)
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch(a.arch)), 1)).eval()
    pipe = LitePosePipeline(model.cuda(), cfg, use_graphs=True)
    J, T = pipe.params.num_joints, pipe.T
    rng = np.random.RandomState(a.seed)
    lists, groups = [], []
    for k in range(a.lists):
        shapes = [POOL[j] for j in rng.randint(0, len(POOL), a.images)]
        imgs = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
        mp = MixedPlan(shapes, pipe.scales, a.size, pipe.project, J, T)
        plants = [PlantedCrowd(1, J, int(mp.det_hw[mp.pos[i]][0]), int(mp.det_hw[mp.pos[i]][1]), T, num_people=5,
                               seed=1000 * k + i) for i in range(len(shapes))]
        lists.append((shapes, imgs, plants))
        groups.append(len(mp.groups))
    frames = sum(len(s) for s, _, _ in lists)
    submit_s = []

    def sequential():
        return [pipe.infer_images(imgs, plant=pl) for _, imgs, pl in lists]

    def in_flight(submit, collect):
        out, pend = [], []
        for lst in lists:
            t0 = time.perf_counter()
            tk = submit(lst)
            submit_s.append(time.perf_counter() - t0)
            pend.append(tk)
            if len(pend) == 2:
                out.append(collect(pend.pop(0)))
        out.extend(collect(tk) for tk in pend)
        return out

    def async_():
        return in_flight(lambda lst: pipe.submit_images(lst[1], plant=lst[2]), pipe.collect_images)

    def sharded():
        from litepose_b200.dist import merge_shards, plan_shards

        def submit(lst):
            shapes, imgs, pl = lst
            plan = plan_shards(shapes, cfg, world)
            mine = plan.indices[rank]
            return plan, pipe.submit_images([imgs[i] for i in mine], plant=[pl[i] for i in mine], group=group, dst=0,
                                            plan=plan)

        def collect(t):
            res = pipe.collect_images(t[1])
            return None if res is None else merge_shards(res, t[0])
        return in_flight(submit, collect)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    res = {}
    ref = None
    if rank == 0:
        arms = {"sequential": sequential, "async": async_}
        times = {k: [] for k in arms}
        outs = {k: fn() for k, fn in arms.items()}          # warm-up: plans, arenas, grow-only buffers of both slots
        ref = outs["sequential"]
        identical = all(same(x, y) for x, y in zip(outs["async"], ref))
        del submit_s[:]
        for _ in range(a.rounds):
            for k, fn in arms.items():
                dt, out = timed(fn)
                times[k].append(dt)
                identical = identical and all(same(x, y) for x, y in zip(out, ref))
        for k, ts in times.items():
            med = float(np.median(ts))
            res[k] = {"lists_per_s": round(a.lists / med, 2), "frames_per_s": round(frames / med, 1),
                      "ms_per_list": round(med / a.lists * 1e3, 2), "ms_rounds": [round(t * 1e3, 1) for t in ts]}
        res["async"]["submit_host_ms_per_list"] = {"median": round(float(np.median(submit_s)) * 1e3, 3),
                                                   "max": round(float(np.max(submit_s)) * 1e3, 3)}
        res["identical"] = bool(identical)
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        sharded()                                               # warm-up
        ts, ok = [], True
        for _ in range(a.rounds):
            dist.barrier()
            dt, out = timed(sharded)
            ts.append(dt)
            if rank == 0:
                ok = ok and all(same(x, y) for x, y in zip(out, ref))
        if rank == 0:
            med = float(np.median(ts))
            res["sharded"] = {"ranks": world, "lists_per_s": round(a.lists / med, 2),
                              "frames_per_s": round(frames / med, 1), "ms_rounds": [round(t * 1e3, 1) for t in ts],
                              "identical": bool(ok)}
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        name, pl = card()
        out = {"card": name, "power_limit": pl, "arch": a.arch, "input_size": a.size, "images_per_list": a.images,
               "lists": a.lists, "size_groups": groups, "rounds": a.rounds, "arms": res}
        line = json.dumps(out)
        print(line)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
