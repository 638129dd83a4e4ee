"""Times the evaluation parser on crowds: LitePose-S at 512 and 640, batch 32 (flip test, adjust + refine), planted crowds
of 30 / 100 / 200 persons at MAX_NUM_PEOPLE = K = 30 / 128 / 256.  Per setting: CUDA-event times of the whole step
(frames on the device -> packed result) and of each parser stage on that step's maps (NMS + top-K, tag matching,
adjust + refine), plus the persons found.  Prints the GPU name and power limit first, then one JSON line per setting.

    python tools/time_crowd.py [--steps 10] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from litepose_b200 import _lib, synth  # noqa: E402
from litepose_b200.config import get_arch, get_cfg  # noqa: E402
from litepose_b200.lib.models.pose_mobilenet import get_pose_net  # noqa: E402
from litepose_b200.pipeline import LitePosePipeline, PlantedCrowd  # noqa: E402

SETTINGS = [(30, 30), (100, 128), (200, 256)]      # (planted persons, K)
SIZES = [512, 640]
BATCH = 32


def gpu_line():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def event_ms(fn, steps):
    """mean CUDA-event time of fn() over `steps` calls (after two warm-up calls)"""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def stage_ms(pipe, det, tag, steps):
    """the parser chain of DeviceParser.run on (det, tag), one event pair per stage, averaged over `steps` runs"""
    p, lib = pipe.parser, pipe.lib
    n, j, h, w = det.shape
    t = tag.shape[4]
    b, _ = p._buffers(det.device, n, h, w, t)
    s = torch.cuda.current_stream().cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    acc = [0.0, 0.0, 0.0]
    for it in range(steps + 2):
        ev[0].record()
        p.top_k_device(det, tag, p.det_thr)
        ev[1].record()
        p.match_device(det.device, n, h, w, t)
        ev[2].record()
        _lib.check(lib.lp_adjust_refine_f32(det.data_ptr(), tag.data_ptr(), n, j, h, w, t, p.pcap, b["ans"].data_ptr(),
                                            b["num"].data_ptr(), b["scores"].data_ptr(), 1, 1, b["ws_ref"].data_ptr(),
                                            b["ws_ref"].numel(), s), "lp_adjust_refine_f32")
        ev[3].record()
        torch.cuda.synchronize()
        if it >= 2:
            for k in range(3):
                acc[k] += ev[k].elapsed_time(ev[k + 1])
    return [a / steps for a in acc], b["num"].cpu().tolist()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_crowd.py measures on a CUDA device; none is available")
    gpu = gpu_line()
    print("# GPU: %s" % gpu, flush=True)
    results = []
    for size in SIZES:
        for people, k in SETTINGS:
            cfg = get_cfg(input_size=size)
            cfg.DATASET.MAX_NUM_PEOPLE = k
            torch.manual_seed(0)
            model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch("S")), 1)).eval().cuda()
            pipe = LitePosePipeline(model, cfg, use_graphs=True, keep=k)
            plant = PlantedCrowd(BATCH, 14, size, size, 2, num_people=people, seed=5, device="cuda")
            x = synth.make_frames(BATCH, size, seed=1).half().cuda()
            step = event_ms(lambda: pipe.step_device(x, plant), args.steps)
            st = pipe._get_state(BATCH, size, size, torch.float16, plant)
            (topk, match, refine), num = stage_ms(pipe, st["det"], st["tag"], args.steps)
            r = {"size": size, "batch": BATCH, "planted": people, "K": k, "step_ms": round(step, 3),
                 "topk_ms": round(topk, 3), "match_ms": round(match, 3), "adjust_refine_ms": round(refine, 3),
                 "persons_min": min(num), "persons_max": max(num), "gpu": gpu}
            print(json.dumps(r), flush=True)
            results.append(r)
            del pipe, model
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
