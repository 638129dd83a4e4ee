"""Measure the depthwise convolutions of LitePose training: where a module-tree training step spends its device time,
the NCHW depthwise kernels (lp_dw_nchw_*) against PyTorch's per op, and whole steps converted against unconverted.

    python tools/time_train_dw.py [--out DIR (default time_train_dw_out)] [--rounds 7] [--iters 5] [--skip-profile]

1. profile: torch.profiler over one fp32 training step (forward, loss, backward, Adam; cudnn.benchmark, TF32 off) of
   the unconverted module tree: LitePose-S at 448^2 batch 16, and the super-network at a drawn size (batch 16).  The
   kernels are classed by name (PyTorch's conv_depthwise2d forward / backward / grad_weight kernels, cuDNN kernels
   whose name says depthwise, and this project's dw_* kernels) and the depthwise share of device time is printed;
   the full kernel table goes to DIR/profile_*.txt.
2. per op: every distinct depthwise shape of LitePose-S at 448^2 batch 16, fp32 and fp16: lp_dw_nchw_fwd / _dgrad /
   _wgrad against F.conv2d and aten.convolution_backward with only the input / only the weight gradient requested.
   Each launch follows an L2 flush (a 256 MB memset outside the timed events); medians over alternating rounds;
   GB/s = the bytes the op must move (fwd x + w + y, dgrad dy + w + dx, wgrad x + dy + dw) over the median time.
3. per step: converted against unconverted (alternating rounds, medians of CUDA-event step times): LitePose-S at 448^2
   batch 16, the super-network at 256^2 and 512^2 (one drawn architecture each, batch 16).
Prints the card name and power limit with the numbers; DIR/time_train_dw.json holds them all."""
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
from litepose_b200.train_dw import convert_depthwise  # noqa: E402

BATCH = 16


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def dw_class(kernel):
    """which depthwise pass a kernel name belongs to, or None"""
    k = kernel.lower()
    if "dw_wgrad" in k or "grad_weight" in k and "depthwise" in k:
        return "wgrad"
    if "dw_dgrad" in k or "depthwise" in k and "backward" in k:
        return "dgrad"
    if "dw_fwd" in k or "depthwise" in k:
        return "fwd"
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
    total, share = 0.0, {"fwd": 0.0, "dgrad": 0.0, "wgrad": 0.0}
    rows = []
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if t <= 0 or e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        total += t
        c = dw_class(e.key)
        if c:
            share[c] += t
        rows.append((t, e.count, c or "", e.key))
    rows.sort(reverse=True)
    with open(os.path.join(out_dir, "profile_%s.txt" % tag), "w") as f:
        f.write("device time of one training step, %s; us, calls, depthwise class, kernel\n" % tag)
        for t, n, c, k in rows:
            f.write("%10.1f %5d %-6s %s\n" % (t, n, c, k[:160]))
    r = {"case": tag, "device_us": total}
    for c, t in share.items():
        r["dw_%s_us" % c] = t
        r["dw_%s_share" % c] = t / total
    r["dw_share"] = sum(share.values()) / total
    print(json.dumps(r))
    return r


def dw_shapes(model, size):
    """distinct (C, H, W, k, stride) of the depthwise convs of a LitePose forward at size^2"""
    shapes = []

    def hook(m, inp, out):
        key = (inp[0].shape[1], inp[0].shape[2], inp[0].shape[3], m.kernel_size[0], m.stride[0])
        if key not in shapes:
            shapes.append(key)
    hs = [m.register_forward_hook(hook) for m in model.modules()
          if isinstance(m, nn.Conv2d) and m.groups > 1 and m.groups == m.in_channels]
    with torch.no_grad():
        model.train()(torch.zeros(1, 3, size, size))
    for h in hs:
        h.remove()
    return shapes


def per_op(rounds, iters):
    lib = _lib.load()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    results = []
    for (c, h, w, k, s) in dw_shapes(litepose_s(), 448):
        for dt in (torch.float32, torch.float16):
            code = _lib.LP_DT_F32 if dt == torch.float32 else _lib.LP_DT_F16
            x = torch.randn(BATCH, c, h, w, device="cuda").to(dt)
            wt = (torch.randn(c, 1, k, k, device="cuda") / k).to(dt)
            y = F.conv2d(x, wt, None, s, k // 2, 1, c)
            dy = torch.randn_like(y)
            dx, dw = torch.empty_like(x), torch.empty_like(wt)
            nb = lib.lp_dw_nchw_wgrad_workspace_bytes(BATCH, c, h, w, k, s)
            ws = torch.empty(max(nb, 4), dtype=torch.uint8, device="cuda")
            yk = torch.empty_like(y)
            st = torch.cuda.current_stream().cuda_stream
            es = x.element_size()
            ops = {
                "fwd": (lambda: lib.lp_dw_nchw_fwd(x.data_ptr(), wt.data_ptr(), yk.data_ptr(), BATCH, c, h, w, k, s,
                                                   code, st),
                        lambda: F.conv2d(x, wt, None, s, k // 2, 1, c), (x.numel() + y.numel() + wt.numel()) * es),
                "dgrad": (lambda: lib.lp_dw_nchw_dgrad(dy.data_ptr(), wt.data_ptr(), dx.data_ptr(), BATCH, c, h, w, k,
                                                       s, code, st),
                          lambda: torch.ops.aten.convolution_backward(dy, x, wt, None, [s, s], [k // 2] * 2, [1, 1],
                                                                      False, [0, 0], c, [True, False, False]),
                          (x.numel() + y.numel() + wt.numel()) * es),
                "wgrad": (lambda: lib.lp_dw_nchw_wgrad(x.data_ptr(), dy.data_ptr(), dw.data_ptr(), BATCH, c, h, w, k,
                                                       s, code, ws.data_ptr(), nb, st),
                          lambda: torch.ops.aten.convolution_backward(dy, x, wt, None, [s, s], [k // 2] * 2, [1, 1],
                                                                      False, [0, 0], c, [False, True, False]),
                          (x.numel() + y.numel() + wt.numel()) * es),
            }
            for name, (ours, theirs, nbytes) in ops.items():
                t = {"ours": [], "torch": []}
                for fn in (ours, theirs):       # warm-up (cuDNN benchmark picks its algorithm here)
                    for _ in range(2):
                        fn()
                for _ in range(rounds):
                    for key, fn in (("ours", ours), ("torch", theirs)):
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
                mo, mt = float(np.median(t["ours"])), float(np.median(t["torch"]))
                r = {"op": name, "dtype": str(dt)[6:], "N": BATCH, "C": c, "H": h, "W": w, "k": k, "stride": s,
                     "ours_ms": mo, "torch_ms": mt, "ours_GBps": nbytes / mo / 1e6, "torch_GBps": nbytes / mt / 1e6,
                     "bytes": nbytes}
                print(json.dumps(r))
                results.append(r)
            del x, wt, y, dy, dx, dw, ws, yk
            torch.cuda.empty_cache()
    return results


def per_step(rounds, iters):
    results = []
    cases = [("LitePose-S", litepose_s, 448, 0)]
    for size in (256, 512):
        cases.append(("supernet", lambda size=size: supernet(size), size, 11))
    for tag, make, size, seed in cases:
        base = make()
        x = synth.make_frames(BATCH, size, seed=1).cuda()
        ref = copy.deepcopy(base).cuda().train()
        conv = convert_depthwise(copy.deepcopy(base)).cuda().train()
        steps = {"unconverted": make_step(ref, x, seed), "converted": make_step(conv, x, seed)}
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
        r = {"case": tag, "size": size, "batch": BATCH, "unconverted_ms": float(np.median(t["unconverted"])),
             "converted_ms": float(np.median(t["converted"])), "rounds": t}
        r["speedup"] = r["unconverted_ms"] / r["converted_ms"]
        print(json.dumps(r))
        results.append(r)
        del base, ref, conv, steps
        torch.cuda.empty_cache()
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="time_train_dw_out")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--skip-profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_train_dw.py measures on the GPU; no CUDA device found")
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    os.makedirs(args.out, exist_ok=True)
    name, limits = card()
    print("card: %s, power limit / max SM clock: %s" % (name, limits))
    res = {"card": name, "power_limit_max_sm_clock": limits}
    if not args.skip_profile:
        random.seed(3)
        size = random.choice(range(256, 513, 32))
        res["profile"] = [profile_step("litepose_s_448_b16", litepose_s(), synth.make_frames(BATCH, 448, seed=1).cuda(),
                                       0, args.out),
                          profile_step("supernet_%d_b16" % size, supernet(size),
                                       synth.make_frames(BATCH, size, seed=1).cuda(), 11, args.out)]
    res["per_op"] = per_op(args.rounds, args.iters)
    res["per_step"] = per_step(args.rounds, args.iters)
    with open(os.path.join(args.out, "time_train_dw.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
