"""Times lp_pw1x1_f16 alone at the eight 1x1-conv shapes one LitePose-S 512x512 pass runs outside the fused block
kernels (stride-2 expansions and projections, stage-3 expansions), by default at batch 32.

CUDA events bracket each launch; L2 is flushed between launches, so every launch reads its input from HBM.  Each shape
is warmed up, then launched until at least --window-ms of kernel time has been timed; the median launch is reported.
MB moved is computed from the shape: fp16 A read plus fp16 output written (none of these launches has a residual;
the weights, at most 0.2 MB, are left out).  TB/s = MB moved / median time.

    python tools/time_pw.py [--batches 32,64] [--lib path/to/liblitepose_b200.so]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from litepose_b200 import _lib  # noqa: E402

# (what, rows at batch 32, K, N, act)
SHAPES = [
    ("stage-0 s2 expansion 256^2", 2097152, 16, 96, 2),
    ("stage-0 s2 projection 128^2", 524288, 96, 16, 0),
    ("stage-1 s2 expansion 128^2", 524288, 16, 96, 2),
    ("stage-1 s2 projection 64^2", 131072, 96, 32, 0),
    ("stage-2 s2 expansion 64^2", 131072, 32, 192, 2),
    ("stage-2 s2 projection 32^2", 32768, 192, 48, 0),
    ("stage-3 first expansion 32^2", 32768, 48, 288, 2),
    ("stage-3 expansion 32^2", 32768, 120, 720, 2),
]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32", help="comma-separated batch sizes")
    ap.add_argument("--window-ms", type=float, default=150.0, help="timed kernel time per shape")
    ap.add_argument("--lib", default=None, help="time this build of the library instead of the in-tree one")
    a = ap.parse_args()
    if a.lib:
        _lib.LIB_PATH = os.path.abspath(a.lib)
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    flush = torch.empty(128 << 20, dtype=torch.uint8, device=dev)    # 2.5x the 50 MB L2
    s = torch.cuda.current_stream().cuda_stream
    results = []
    for batch in [int(b) for b in a.batches.split(",")]:
        for what, m32, k, n, act in SHAPES:
            m = m32 * batch // 32
            rs = np.random.RandomState(k * 1000 + n)
            w16 = np.ascontiguousarray((rs.randn(n, k) / k ** 0.5).astype(np.float16)).view(np.uint16)
            bias = (rs.randn(n) * 0.1).astype(np.float32)
            wp = np.zeros(lib.lp_pw1x1_packed_elems(k, n), np.uint16)
            bp = np.zeros(lib.lp_pw1x1_packed_bias_elems(n), np.float32)
            _lib.check(lib.lp_pw1x1_pack(w16.ctypes.data, bias.ctypes.data, k, n, wp.ctypes.data, bp.ctypes.data))
            wd = torch.from_numpy(wp).view(torch.float16).to(dev)
            bd = torch.from_numpy(bp).to(dev)
            x = torch.randn((m, k), device=dev).half()
            y = torch.empty((m, n), dtype=torch.float16, device=dev)

            def launch():
                _lib.check(lib.lp_pw1x1_f16(x.data_ptr(), wd.data_ptr(), bd.data_ptr(), None, y.data_ptr(), m, k, n, act, s))

            def timed(iters):
                evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
                for e0, e1 in evs:
                    flush.zero_()
                    e0.record()
                    launch()
                    e1.record()
                torch.cuda.synchronize()
                return [e0.elapsed_time(e1) * 1e3 for e0, e1 in evs]

            warm = timed(20)
            iters = max(50, int(a.window_ms * 1e3 / float(np.median(warm))) + 1)
            ts = timed(iters)
            us = float(np.median(ts))
            mb = m * (k + n) * 2 / 1e6
            results.append({"batch": batch, "shape": what, "M": m, "K": k, "N": n, "us": round(us, 2),
                            "mean_us": round(float(np.mean(ts)), 2), "iters": iters, "MB": round(mb, 1),
                            "TBps": round(mb / us, 3)})     # MB per us = TB/s
            del x, y
    gpu = gpu_info()
    print("# %s" % gpu)
    print("# lp_pw1x1_f16 alone, L2 flushed between launches, median of >= %.0f ms of launches" % a.window_ms)
    print("%5s  %-30s %8s %4s %4s %9s %8s %6s" % ("batch", "shape", "M", "K", "N", "us", "MB", "TB/s"))
    for r in results:
        print("%5d  %-30s %8d %4d %4d %9.1f %8.1f %6.2f" % (r["batch"], r["shape"], r["M"], r["K"], r["N"], r["us"],
                                                         r["MB"], r["TBps"]))
    for b in sorted({r["batch"] for r in results}):
        rb = [r for r in results if r["batch"] == b]
        tot_us, tot_mb = sum(r["us"] for r in rb), sum(r["MB"] for r in rb)
        print("# batch %d: one pass %.1f us for %.0f MB (%.2f TB/s)" % (b, tot_us, tot_mb, tot_mb / tot_us))
    print(json.dumps({"gpu": gpu, "lib": _lib.LIB_PATH, "results": results}))


if __name__ == "__main__":
    main()
