"""Measure the BatchNorm layers of LitePose training: the NCHW train-mode BatchNorm kernels (lp_bn_nchw_*) against
PyTorch's per op, whole steps with and without them, and where the fully converted step spends its device time.

    python tools/time_train_bn.py [--out DIR (default time_train_bn_out)] [--rounds 7] [--iters 5] [--skip-profile]

1. per op: every distinct BatchNorm shape of LitePose-S at 448^2 batch 16, fp32 and fp16, without an activation and
   with ReLU6: lp_bn_nchw_fwd against F.batch_norm (train mode) + F.relu6(inplace=True), and lp_bn_nchw_bwd (dx,
   dgamma, dbeta) against torch.autograd.grad through the same two ops.  Each launch follows an L2 flush (a 256 MB
   memset outside the timed events); medians over alternating rounds; GB/s = the bytes of the passes a fused kernel
   needs (forward 3: x read twice, y written; backward 5: x and dy read twice, dx written) over the median time.
2. per step: three builds, alternating rounds, medians of CUDA-event step times (forward, loss, backward, Adam; fp32):
   unconverted, convert_depthwise, and convert_depthwise + convert_batchnorm, for LitePose-S at 448^2 and the
   super-network at 512^2 (one drawn architecture), batch 16.  The per-round times are kept to show the spread.
3. profile: torch.profiler over one step of the fully converted build (LitePose-S at 448^2 and the super-network at
   352^2, batch 16); the kernels are classed by name (cuDNN / ATen batch-norm kernels, the clamp / hardtanh /
   threshold kernels of the activations, this project's bnt_* kernels) and the full table goes to DIR/profile_*.txt.
Prints the card name and power limit with the numbers; DIR/time_train_bn.json holds them all."""
import argparse
import copy
import json
import os
import random
import subprocess
import sys

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from litepose_b200 import _lib, synth  # noqa: E402
from litepose_b200.config import get_arch, get_cfg  # noqa: E402
from litepose_b200.lib.models import pose_mobilenet, pose_supermobilenet  # noqa: E402
from litepose_b200.train_bn import convert_batchnorm  # noqa: E402
from litepose_b200.train_dw import convert_depthwise  # noqa: E402

BATCH = 16
ACT_NAMES = {_lib.ACT_NONE: "none", _lib.ACT_RELU6: "relu6"}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def bn_class(kernel):
    """which part of a BatchNorm + activation layer a kernel name belongs to, or None"""
    k = kernel.lower()
    if "bnt_" in k:
        return "ours"
    if "bn_fw" in k or "bn_bw" in k or "batch_norm" in k or "batchnorm" in k:
        return "bn"
    if "clamp" in k or "hardtanh" in k or "threshold" in k:
        return "act"
    return None


def litepose_s():
    torch.manual_seed(0)
    return synth.randomize_bn_(pose_mobilenet.get_pose_net(get_cfg(input_size=448), False, get_arch("S")), 1)


def supernet(size):
    torch.manual_seed(0)
    return synth.randomize_bn_(pose_supermobilenet.get_pose_net(get_cfg(input_size=size)), 1)


def make_step(model, x, seed):
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)

    def step():
        random.seed(seed)            # the super-network draws its architecture per forward: the same one every step
        opt.zero_grad(set_to_none=True)
        outs = model(x)
        loss = sum(o.float().square().mean() for o in outs)
        loss.backward()
        opt.step()
    return step


def profile_step(tag, model, x, seed, out_dir):
    from torch.profiler import ProfilerActivity, profile
    step = make_step(model.cuda().train(), x, seed)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    total, share = 0.0, {"ours": 0.0, "bn": 0.0, "act": 0.0}
    rows = []
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if t <= 0 or e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        total += t
        c = bn_class(e.key)
        if c:
            share[c] += t
        rows.append((t, e.count, c or "", e.key))
    rows.sort(reverse=True)
    with open(os.path.join(out_dir, "profile_%s.txt" % tag), "w") as f:
        f.write("device time of one training step, %s; us, calls, class (ours: bnt_*, bn: other batch-norm kernels, "
                "act: clamp / hardtanh / threshold), kernel\n" % tag)
        for t, n, c, k in rows:
            f.write("%10.1f %5d %-4s %s\n" % (t, n, c, k[:160]))
    r = {"case": tag, "device_us": total}
    for c, t in share.items():
        r["%s_us" % c] = t
        r["%s_share" % c] = t / total
    print(json.dumps(r))
    return r


def bn_shapes(model, size):
    """distinct (C, H, W) of the BatchNorm inputs of a LitePose forward at size^2"""
    shapes = []

    def hook(m, inp, out):
        key = tuple(inp[0].shape[1:])
        if key not in shapes:
            shapes.append(key)
    hs = [m.register_forward_hook(hook) for m in model.modules() if isinstance(m, nn.BatchNorm2d)]
    with torch.no_grad():
        model.train()(torch.zeros(1, 3, size, size))
    for h in hs:
        h.remove()
    return shapes


def _time(fns, rounds, iters, flush):
    """medians over alternating rounds of per-launch CUDA-event times, each launch after an L2 flush"""
    for fn in fns.values():             # warm-up (cuDNN picks its algorithm here)
        for _ in range(2):
            fn()
    t = {k: [] for k in fns}
    for _ in range(rounds):
        for key, fn in fns.items():
            vals = []
            for _ in range(iters):
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                b.synchronize()
                vals.append(a.elapsed_time(b))
            t[key].append(float(np.median(vals)))
    return {k: float(np.median(v)) for k, v in t.items()}


def per_op(rounds, iters):
    lib = _lib.load()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    results = []
    for (c, h, w) in bn_shapes(litepose_s(), 448):
        for dt in (torch.float32, torch.float16):
            code = _lib.LP_DT_F32 if dt == torch.float32 else _lib.LP_DT_F16
            x = (torch.randn(BATCH, c, h, w, device="cuda") * 2 + 0.5).to(dt)
            dy = torch.randn_like(x)
            g, b = torch.rand(c, device="cuda") + 0.5, torch.randn(c, device="cuda") * 0.1
            rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
            y, dx = torch.empty_like(x), torch.empty_like(x)
            saved, dg, db = torch.empty(4, c, device="cuda"), torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
            nb = lib.lp_bn_nchw_workspace_bytes(BATCH, c, h, w)
            ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
            st = torch.cuda.current_stream().cuda_stream
            es = x.element_size()
            for act in (_lib.ACT_NONE, _lib.ACT_RELU6):
                xr, gr, br = x.clone().requires_grad_(True), g.clone().requires_grad_(True), b.clone().requires_grad_(True)

                def torch_fwd(xr=xr, gr=gr, br=br, act=act):
                    out = F.batch_norm(xr, rm, rv, gr, br, True, 0.1, 1e-5)
                    return F.relu6(out, inplace=True) if act == _lib.ACT_RELU6 else out
                yt = torch_fwd()
                ops = {
                    "fwd": ({"ours": lambda act=act: lib.lp_bn_nchw_fwd(
                                x.data_ptr(), g.data_ptr(), b.data_ptr(), rm.data_ptr(), rv.data_ptr(), 0.1, 1e-5,
                                y.data_ptr(), saved.data_ptr(), BATCH, c, h, w, act, code, ws.data_ptr(), nb, st),
                             "torch": lambda: torch_fwd()}, 3 * x.numel() * es),
                    "bwd": ({"ours": lambda act=act: lib.lp_bn_nchw_bwd(
                                x.data_ptr(), dy.data_ptr(), g.data_ptr(), saved.data_ptr(), dx.data_ptr(),
                                dg.data_ptr(), db.data_ptr(), BATCH, c, h, w, act, code, ws.data_ptr(), nb, st),
                             "torch": lambda yt=yt, xr=xr, gr=gr, br=br: torch.autograd.grad(
                                 yt, (xr, gr, br), dy, retain_graph=True)}, 5 * x.numel() * es),
                }
                for name, (fns, nbytes) in ops.items():
                    t = _time(fns, rounds, iters, flush)
                    mo, mt = t["ours"], t["torch"]
                    r = {"op": name, "act": ACT_NAMES[act], "dtype": str(dt)[6:], "N": BATCH, "C": c, "H": h, "W": w,
                         "ours_ms": mo, "torch_ms": mt, "speedup": mt / mo, "ours_GBps": nbytes / mo / 1e6,
                         "torch_GBps": nbytes / mt / 1e6, "bytes": nbytes}
                    print(json.dumps(r))
                    results.append(r)
                del xr, gr, br, yt
            del x, dy, y, dx, ws
            torch.cuda.empty_cache()
    return results


def per_step(rounds, iters):
    results = []
    for tag, make, size, seed in (("LitePose-S", litepose_s, 448, 0), ("supernet", lambda: supernet(512), 512, 11)):
        base = make()
        x = synth.make_frames(BATCH, size, seed=1).cuda()
        builds = {"unconverted": copy.deepcopy(base),
                  "depthwise": convert_depthwise(copy.deepcopy(base)),
                  "depthwise+bn": convert_batchnorm(convert_depthwise(copy.deepcopy(base)))}
        steps = {k: make_step(m.cuda().train(), x, seed) for k, m in builds.items()}
        for fn in steps.values():
            for _ in range(3):
                fn()
        t = {k: [] for k in steps}
        for _ in range(rounds):
            for k, fn in steps.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(iters):
                    fn()
                b.record()
                b.synchronize()
                t[k].append(a.elapsed_time(b) / iters)
        r = {"case": tag, "size": size, "batch": BATCH, "rounds": t}
        for k, v in t.items():
            r["%s_ms" % k] = float(np.median(v))
            r["%s_spread_ms" % k] = float(np.max(v) - np.min(v))
        r["bn_speedup_over_depthwise"] = r["depthwise_ms"] / r["depthwise+bn_ms"]
        print(json.dumps(r))
        results.append(r)
        del base, builds, steps
        torch.cuda.empty_cache()
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="time_train_bn_out")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--skip-profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_train_bn.py measures on the GPU; no CUDA device found")
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    os.makedirs(args.out, exist_ok=True)
    name, limits = card()
    print("card: %s, power limit / max SM clock: %s" % (name, limits))
    res = {"card": name, "power_limit_max_sm_clock": limits}
    res["per_op"] = per_op(args.rounds, args.iters)
    res["per_step"] = per_step(args.rounds, args.iters)
    if not args.skip_profile:
        res["profile"] = []
        for tag, make, size, seed in (("litepose_s_448_b16", litepose_s, 448, 0),
                                      ("supernet_352_b16", lambda: supernet(352), 352, 11)):
            model = convert_batchnorm(convert_depthwise(make()))
            res["profile"].append(profile_step(tag + "_converted", model,
                                               synth.make_frames(BATCH, size, seed=1).cuda(), seed, args.out))
    with open(os.path.join(args.out, "time_train_bn.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
