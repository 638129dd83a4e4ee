"""valid.py's command line on synthetic images:  the reference's evaluation loop (valid.py:95-233) with the dataset
replaced by seeded uint8 images (this image has neither the datasets nor yacs / pycocotools; SURVEY.md 8b last row).

    python tools/valid_synthetic.py --cfg experiments/crowd_pose/mobilenet/mobile.yaml \
        --superconfig mobile_configs/search-S.json [--images 8 --height 480 --width 640] [KEY VALUE ...]

Same flow as valid.py: update_config (defaults <- file <- opts), INPUT_SIZE from the architecture, get_pose_net,
network_to_half when FP16.ENABLED, HeatmapParser, then per batch LitePosePipeline.infer_images = the loop body
(:198-233).  Deviations: synthetic images instead of the dataloader, random-init weights unless TEST.MODEL_FILE exists,
no dataset.evaluate.  --dry-run stops before the first CUDA call and prints the resolved configuration."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="valid.py on synthetic images")
    ap.add_argument("--cfg", required=True)
    ap.add_argument("--superconfig", default=None)
    ap.add_argument("--images", type=int, default=8, help="batch of equally sized synthetic images")
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--sizes", default=None, metavar="HxW,HxW,...",
                    help="a mixed list of image sizes (one image each) instead of --images x --height x --width")
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--dry-run", action="store_true")
    ap.add_argument("opts", nargs=argparse.REMAINDER, help="KEY VALUE pairs, as valid.py takes them")
    return ap.parse_args(argv)


def main(argv=None):
    args = parse_args(argv)
    from litepose_b200.config import load_experiment
    from litepose_b200.pipeline import LitePosePipeline
    cfg, arch = load_experiment(args.cfg, args.superconfig, args.opts)
    if arch is None:
        raise SystemExit("--superconfig is required for pose_mobilenet (valid.py:106-111)")
    LitePosePipeline._validate_cfg(cfg)
    sizes = None
    if args.sizes:
        try:
            sizes = [tuple(int(v) for v in s.lower().split("x")) for s in args.sizes.split(",")]
        except ValueError:
            raise SystemExit("--sizes: HxW,HxW,... expected, got %r" % args.sizes)
        if any(len(s) != 2 or min(s) <= 0 for s in sizes):
            raise SystemExit("--sizes: HxW,HxW,... expected, got %r" % args.sizes)
    summary = {"model": cfg.MODEL.NAME, "input_size": cfg.DATASET.INPUT_SIZE, "joints": cfg.DATASET.NUM_JOINTS,
               "scale_factor": list(cfg.TEST.SCALE_FACTOR), "flip_test": cfg.TEST.FLIP_TEST,
               "project2image": cfg.TEST.PROJECT2IMAGE, "fp16": cfg.FP16.ENABLED, "adjust": cfg.TEST.ADJUST,
               "refine": cfg.TEST.REFINE,
               "images": [args.images, args.height, args.width, 3] if sizes is None else [[h, w, 3] for h, w in sizes]}
    if args.dry_run:
        print(json.dumps(summary))
        return summary
    import numpy as np
    import torch
    from litepose_b200.lib.models.pose_mobilenet import get_pose_net
    if not torch.cuda.is_available():
        raise SystemExit("a CUDA device is required (there is no CPU path)")
    torch.manual_seed(0)
    model = get_pose_net(cfg, is_train=True, cfg_arch=arch)          # valid.py:130-132 passes is_train=True as well
    if cfg.TEST.MODEL_FILE and os.path.isfile(cfg.TEST.MODEL_FILE):
        model.load_state_dict(torch.load(cfg.TEST.MODEL_FILE, map_location="cpu"), strict=True)
    model = model.cuda().eval()       # FP16.ENABLED: the frames are fed as fp16 (what tofp16 does, fp16util.py:40-47); the
    pipe = LitePosePipeline(model, cfg)   # engine computes in fp16 with BN folded in fp32 either way (DESIGN.md 3)
    rng = np.random.RandomState(0)
    if sizes is None:
        imgs = torch.from_numpy(rng.randint(0, 256, (args.images, args.height, args.width, 3)).astype(np.uint8)).pin_memory()
    else:                             # a mixed list: one infer_images call on images of different sizes
        imgs = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    res = pipe.infer_images(imgs, half=bool(cfg.FP16.ENABLED))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.repeat):
        res = pipe.infer_images(imgs, half=bool(cfg.FP16.ENABLED))
    dt = (time.perf_counter() - t0) / args.repeat
    summary.update({"persons": [r[2] for r in res], "frames_per_s": len(imgs) / dt, "ms_per_batch": dt * 1e3})
    print(json.dumps(summary))
    return summary


if __name__ == "__main__":
    main()
