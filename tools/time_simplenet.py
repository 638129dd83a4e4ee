"""Times the forward of LitePose with the Fusion Deconv Head (pose_mobilenet) against the paper's ablation without it
(pose_simplenet): the plain and the mirrored pass of the flip test, as the evaluation runs them, on the sm_90a engine
and, for comparison, on the same nn.Module graph in stock PyTorch fp16 (cuDNN, benchmark mode).

Both models are built from the same seed (LitePose-S by default, 512x512, batch 32, fp16 input).  One sample is the
time of --iters back-to-back (plain + mirrored) forwards bracketed by CUDA events, divided by --iters; the variants
are alternated for --rounds rounds so that drift on a shared card hits all of them alike; median, min and max per
variant are reported with the card's name and power limit, as one JSON line.

    python tools/time_simplenet.py [--arch S] [--size 512] [--batch 32] [--rounds 7] [--iters 10] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from litepose_b200 import synth  # noqa: E402
from litepose_b200.config import get_arch, get_cfg  # noqa: E402
from litepose_b200.lib.models import pose_mobilenet, pose_simplenet  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def build(mod, arch, size):
    torch.manual_seed(0)
    return synth.randomize_bn_(mod.get_pose_net(get_cfg(input_size=size), False, get_arch(arch)), 1).eval().cuda()


def variants(arch, size, x):
    out = {}
    xf = torch.flip(x, [3]).contiguous()
    for name, mod in (("pose_mobilenet", pose_mobilenet), ("pose_simplenet", pose_simplenet)):
        eng = build(mod, arch, size).lp_engine()

        def run_engine(eng=eng):
            eng.run(x, flip=False, out_fp32=False, clone=False)
            eng.run(x, flip=True, out_fp32=False, clone=False)

        half = build(mod, arch, size).half()

        def run_cudnn(m=half):
            with torch.no_grad():
                m._forward_modules(x)            # the module tree, not the engine
                m._forward_modules(xf)

        out[name + " sm_90a engine"] = run_engine
        out[name + " cuDNN fp16"] = run_cudnn
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="S")
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_simplenet.py needs a CUDA device")
    torch.backends.cudnn.benchmark = True
    x = synth.make_frames(args.batch, args.size, seed=3).cuda().half()
    fns = variants(args.arch, args.size, x)
    for fn in fns.values():                       # warm-up: plans, graphs of cuDNN algorithms, module loads
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
    res = {"gpu": gpu_info(), "arch": args.arch, "size": args.size, "batch": args.batch,
           "what": "plain + mirrored forward, ms per batch", "rounds": args.rounds, "iters": args.iters,
           "ms": {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
                  for k, v in samples.items()}}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
