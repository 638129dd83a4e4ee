"""Helpers for the -m gpu parity tests: call the C ABI on torch CUDA tensors and build
fp32 CPU references (oracle side) on the same seeded inputs."""
import numpy as np
import torch
import torch.nn.functional as F

from litepose_b200 import _lib
from mma_emul import lift16


def stream():
    return torch.cuda.current_stream().cuda_stream


def nhwc16(x_nchw):
    """fp32 NCHW CPU -> fp16 NHWC CUDA"""
    return x_nchw.permute(0, 2, 3, 1).contiguous().half().cuda()


def from_nhwc(y):
    return y.float().cpu().permute(0, 3, 1, 2).contiguous()


def q16(t):
    return t.half().float()


def tol_check(got, ref, rel=2e-3, abs_=1e-4, what=""):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = (got - ref).abs().max().item()
    lim = rel * ref.abs().max().item() + abs_
    _record(what, err, lim)
    assert err <= lim, "%s: max err %.3e > %.3e (max|ref| %.3e)" % (what, err, lim, ref.abs().max().item())
    return err


def _record(what, err, lim):
    """Append measured error / limit to gpurun_out/errors.jsonl (headroom bookkeeping, best effort)."""
    import json
    import os
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    try:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "errors.jsonl"), "a") as f:
            f.write(json.dumps({"what": what, "err": err, "lim": lim, "ratio": err / lim if lim else None}) + "\n")
    except OSError:
        pass


def check_bound(got, ref, mag, k, what):
    """got against the fp64 value ref of a K-term reduction, element by element: |got - ref| <= 2^-11 |ref| +
    K 2^-22 mag + 2^-24, mag = the same reduction over magnitudes with fp16 subnormal operands raised to 2^-14
    (mma_emul.lift16).  The K 2^-22 mag term covers the tensor-core accumulation measured on the H100
    (mma_emul.MODEL): per K = 16 step at most 17 terms cut below 2^(E - 25) and one fp32 rounding toward zero, with
    2^E at most the largest lifted product or the incoming sum, (17 * 2^-25 + 2^-23) mag per step, about a fifth of
    the term.  A subnormal operand's exponent enters E as -14, which is why its magnitude is lifted.  The worst
    err / bound is recorded with _record."""
    got = np.asarray(got, np.float64).reshape(ref.shape)
    assert np.isfinite(got).all(), what
    bound = 2.0 ** -11 * np.abs(ref) + k * 2.0 ** -22 * mag + 2.0 ** -24
    ratio = np.abs(got - ref) / bound
    worst = float(ratio.max())
    _record("fp64 " + what, worst, 1.0)
    assert worst <= 1.0, "%s: err/bound %.3f at %s" % (what, worst, np.unravel_index(ratio.argmax(), ratio.shape))


def check_reduction(got, a, wt, bias, res, k, what, act=_lib.ACT_NONE):
    """got [M, N] against act(a @ wt^T + bias) + res in fp64, element by element (check_bound)"""
    a64, w64 = a.reshape(-1, k).astype(np.float64), wt.astype(np.float64)
    ref = a64 @ w64.T
    mag = lift16(a64) @ lift16(w64).T
    if bias is not None:
        ref += bias.astype(np.float64)
        mag += np.abs(bias.astype(np.float64))
    if act == _lib.ACT_RELU:
        ref = np.maximum(ref, 0)
    elif act == _lib.ACT_RELU6:
        ref = np.clip(ref, 0, 6)
    if res is not None:
        r64 = res.reshape(ref.shape).astype(np.float64)
        ref += r64
        mag += np.abs(r64)
    check_bound(got, ref, mag, k, what)


def pack_pw(w, bias):
    lib = _lib.load()
    n, k = w.shape
    w16 = np.ascontiguousarray(w.half().numpy()).view(np.uint16)
    wp = np.zeros(lib.lp_pw1x1_packed_elems(k, n), np.uint16)
    bp = np.zeros(lib.lp_pw1x1_packed_bias_elems(n), np.float32)
    b = None if bias is None else np.ascontiguousarray(bias.float().numpy())
    _lib.check(lib.lp_pw1x1_pack(w16.ctypes.data, None if b is None else b.ctypes.data, k, n, wp.ctypes.data,
                                 bp.ctypes.data))
    return torch.from_numpy(wp).view(torch.float16).cuda(), torch.from_numpy(bp).cuda()
