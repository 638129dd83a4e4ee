"""Times sub-networks of the LitePose super-network (pose_supermobilenet) on the sm_90a engine against the same
module tree in stock PyTorch fp16 (cuDNN, benchmark mode; the supernet's own forward, slicing its weights per call):
the plain and the mirrored pass of the flip test per batch, for search-XS, search-S and fixed_sample(512, 1.0), each
at its own img_size.  It also times what an architecture search pays per candidate on the host: deriving the
sub-network from the supernet's state dict (on the device, as the module holds it) and packing its engine.

One forward sample is the time of --iters back-to-back (plain + mirrored) forwards bracketed by CUDA events, divided by
--iters; the variants are alternated for --rounds rounds.  The derive-and-pack time is a host clock around
derive_supernet_subnet + LitePoseEngine, ending in a device synchronise, --rounds times per architecture.  Median, min
and max are reported with the card's name and power limit, as one JSON line.

    python tools/time_supernet.py [--batch 32] [--rounds 7] [--iters 10] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from litepose_b200 import synth  # noqa: E402
from litepose_b200.arch_manager import ArchManager  # noqa: E402
from litepose_b200.config import get_arch, get_cfg  # noqa: E402
from litepose_b200.engine import LitePoseEngine  # noqa: E402
from litepose_b200.lib.models import pose_supermobilenet  # noqa: E402
from litepose_b200.subnet import derive_supernet_subnet  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def stats(v):
    return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_supernet.py needs a CUDA device")
    torch.backends.cudnn.benchmark = True
    cfg = get_cfg()
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_supermobilenet.get_pose_net(cfg), 1).eval().cuda()
    half = synth.randomize_bn_(pose_supermobilenet.get_pose_net(cfg), 1).eval().cuda().half()
    archs = {"search-XS": get_arch("XS"), "search-S": get_arch("S"),
             "fixed_sample(512, 1.0)": ArchManager(cfg).fixed_sample(512, 1.0)}
    fns, inputs = {}, {}
    for name, arch in archs.items():
        size = int(arch["img_size"])
        x = synth.make_frames(args.batch, size, seed=3).cuda().half()
        xf = torch.flip(x, [3]).contiguous()
        inputs[name] = (x, xf)
        eng = model.lp_engine(cfg_arch=arch)

        def run_engine(eng=eng, x=x):
            eng.run(x, flip=False, out_fp32=False, clone=False)
            eng.run(x, flip=True, out_fp32=False, clone=False)

        def run_cudnn(arch=arch, x=x, xf=xf):
            with torch.no_grad():
                half._forward_modules(x, arch)       # the module tree, not the engine
                half._forward_modules(xf, arch)

        fns["%s %d sm_90a engine" % (name, size)] = run_engine
        fns["%s %d cuDNN fp16" % (name, size)] = run_cudnn
    for fn in fns.values():                       # warm-up: plans, cuDNN algorithm choice, module loads
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    samples = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                fn()
            b.record()
            b.synchronize()
            samples[k].append(a.elapsed_time(b) / args.iters)
    sd = model.state_dict()
    derive = {}
    for name, arch in archs.items():
        v = []
        for _ in range(args.rounds):
            torch.cuda.synchronize()
            t = time.perf_counter()
            sub = derive_supernet_subnet(sd, arch)
            LitePoseEngine(sub.state_dict, sub.arch, "cuda", residual=sub.residual, strides=sub.strides)
            torch.cuda.synchronize()
            v.append((time.perf_counter() - t) * 1e3)
        derive[name] = stats(v)
    res = {"gpu": gpu_info(), "batch": args.batch, "what": "plain + mirrored forward, ms per batch",
           "rounds": args.rounds, "iters": args.iters, "ms": {k: stats(v) for k, v in samples.items()},
           "derive_and_pack_ms": derive}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
