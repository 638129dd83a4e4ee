"""Time one BN recalibration batch of the super-network: the module tree in training mode (fp32, cudnn.benchmark, grad
enabled, as calibrate_test.py runs it) against SuperLitePose.lp_recalibrate_bn on the kernels.

    python tools/time_recal.py [--rounds 7] [--iters 5] [--out time_recal.json]

Per case: CUDA-event time per batch, median over alternating rounds (tree, kernels, tree, ...), the library launches per
batch, and the host cost of building a train plan for a new candidate (derive_supernet_subnet + packing + planning,
the cache emptied).  Prints the card name and power limit with the numbers."""
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
from litepose_b200.config import get_cfg  # noqa: E402
from litepose_b200.lib.models import pose_supermobilenet  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
CASES = [("search_XS", 256), ("search_S", 448)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_recal.py measures on the GPU; no CUDA device found")
    torch.backends.cudnn.benchmark = True
    name, limits = card()
    print("card: %s, power limit / max SM clock: %s" % (name, limits))
    lib = _lib.load()
    results = []
    for arch_name, size in CASES:
        # the reference's mobile_configs/search-{XS,S}.json, as the recalibration goldens carry them
        arch = json.loads(str(np.load(os.path.join(GOLDEN, "supernet_recal_%s.npz" % arch_name))["arch"]))
        torch.manual_seed(0)
        model = synth.randomize_bn_(pose_supermobilenet.get_pose_net(get_cfg(input_size=size)), 1).cuda()
        model.arch_manager.is_search, model.arch_manager.search_arch = True, arch
        x = synth.make_frames(args.batch, size, seed=3).cuda()

        def tree():
            model.train()
            model(x)

        def kernels():
            model.lp_recalibrate_bn(x)

        model.eval()
        t0 = time.perf_counter()
        model.lp_recalibrate_bn(x)
        torch.cuda.synchronize()
        first = time.perf_counter() - t0
        builds = []
        for _ in range(3):
            model._lp_train_cache.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model._lp_train_plan(x, arch, *_mods(model, arch))
            torch.cuda.synchronize()
            builds.append(time.perf_counter() - t0)
        for _ in range(2):
            tree()
            kernels()
        lib.lp_reset_launch_count()
        kernels()
        torch.cuda.synchronize()
        launches = int(lib.lp_launch_count())
        t_tree, t_kern = [], []
        for _ in range(args.rounds):
            t_tree.append(timed(tree, args.iters))
            t_kern.append(timed(kernels, args.iters))
        r = {"arch": arch_name, "size": size, "batch": args.batch, "card": name, "power_limit_max_sm_clock": limits,
             "tree_ms": float(np.median(t_tree)), "kernels_ms": float(np.median(t_kern)),
             "tree_ms_rounds": t_tree, "kernels_ms_rounds": t_kern, "launches_per_batch": launches,
             "plan_build_s": float(np.median(builds)), "first_call_s": first}
        r["speedup"] = r["tree_ms"] / r["kernels_ms"]
        print(json.dumps(r))
        results.append(r)
        del model
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


def _mods(model, arch):
    from litepose_b200.bn_train import bn_names
    names = bn_names(arch)
    return names, [model.get_submodule(n) for n in names]


if __name__ == "__main__":
    main()
