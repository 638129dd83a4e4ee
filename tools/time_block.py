"""Times the block-level kernels at the stage shapes of LitePose-S @512 (CUDA events, L2 flushed), by default at
batch 64 (a batch-32 step runs the plain and the mirrored pass concurrently on two streams, about the work of one
batch-64 launch): fused block kernel vs expansion GEMM + fused depthwise/projection kernel.  The stage-3 shapes
(Co = 120) do not fit the fused block kernel; they time the expansion and lp_dw7_project_f16 only.  dw_tmacs is the
depthwise work (N*H*W*Ce*49 MAC) over the time of the fused block kernel, or of lp_dw7_project_f16 where there is none.
The stride-2 blocks with Cin <= 16 time lp_block_s2_f16 against the expansion GEMM + stride-2 depthwise + projection
GEMM it replaces; hbm_gbs is the fused kernel's compulsory traffic (input read once, output written once) over its time."""
import os, sys, json, argparse, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from litepose_b200 import _lib
lib = _lib.load()
dev = torch.device("cuda", 0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=64)
args = ap.parse_args()

def timeit(fn, iters=12, skip=3):
    ts = []
    for i in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        if i >= skip: ts.append(e0.elapsed_time(e1) * 1e3)
    return sum(ts) / len(ts)

def pack_pw(w, K, N):
    w16 = np.ascontiguousarray(w.astype(np.float16)).view(np.uint16)
    wp = np.zeros(lib.lp_pw1x1_packed_elems(K, N), np.uint16); bp = np.zeros(lib.lp_pw1x1_packed_bias_elems(N), np.float32)
    _lib.check(lib.lp_pw1x1_pack(w16.ctypes.data, None, K, N, wp.ctypes.data, bp.ctypes.data))
    return torch.from_numpy(wp).view(torch.float16).to(dev), torch.from_numpy(bp).to(dev)

out = {}
s = torch.cuda.current_stream().cuda_stream
for (hw, cin, ce, co) in ((128, 16, 96, 16), (64, 32, 192, 32), (32, 48, 288, 48), (32, 48, 288, 120), (32, 120, 720, 120)):
    n = args.batch
    rs = np.random.RandomState(0)
    x = torch.randn((n, hw, hw, cin), device=dev).half()
    we = (rs.randn(ce, cin) / cin ** 0.5).astype(np.float32)
    fused = lib.lp_block_s1_supported(cin, ce, co)
    if fused:
        wek = np.zeros(lib.lp_block_s1_wexp_elems(cin, ce), np.uint16)
        w16 = np.ascontiguousarray(we.astype(np.float16)).view(np.uint16)
        _lib.check(lib.lp_block_s1_pack_wexp(w16.ctypes.data, cin, ce, wek.ctypes.data))
        wed = torch.from_numpy(wek).view(torch.float16).to(dev)
    be = torch.zeros(ce, device=dev); bd = torch.zeros(ce, device=dev)
    wd = (torch.randn((49, ce), device=dev) * 0.1).half()
    wpd, bpd = pack_pw(rs.randn(co, ce) / ce ** 0.5, ce, co)
    wexp, bexp = pack_pw(we, cin, ce)
    e = torch.empty((n, hw, hw, ce), dtype=torch.float16, device=dev)
    o = torch.empty((n, hw, hw, co), dtype=torch.float16, device=dev)
    res = x if cin == co else None
    t_blk = None
    if fused:
        t_blk = timeit(lambda: _lib.check(lib.lp_block_s1_f16(x.data_ptr(), wed.data_ptr(), be.data_ptr(), wd.data_ptr(), bd.data_ptr(),
                                                               wpd.data_ptr(), bpd.data_ptr(), 1, o.data_ptr(), n, hw, hw, cin, ce, co, s)))
    t_exp = timeit(lambda: _lib.check(lib.lp_pw1x1_f16(x.data_ptr(), wexp.data_ptr(), bexp.data_ptr(), None, e.data_ptr(), n * hw * hw, cin, ce, 2, s)))
    t_dwp = timeit(lambda: _lib.check(lib.lp_dw7_project_f16(e.data_ptr(), wd.data_ptr(), bd.data_ptr(), wpd.data_ptr(), bpd.data_ptr(),
                                                              res.data_ptr() if res is not None else None, o.data_ptr(),
                                                              n, hw, hw, ce, co, s)))
    out["%dx%dx%dx%d->%d->%d" % (n, hw, hw, cin, ce, co)] = {"block_us": t_blk, "expand_us": t_exp, "dw_project_us": t_dwp,
                                                              "dw_tmacs": n * hw * hw * ce * 49 / (t_blk or t_dwp) / 1e6}
# stride-2 blocks with Cin <= 16 (stage 0 / 1, block 0): lp_block_s2_f16 against the three-launch chain
for (hw, cin, ce, co) in ((256, 16, 96, 16), (128, 16, 96, 32)):
    n = args.batch
    rs = np.random.RandomState(0)
    x = torch.randn((n, hw, hw, cin), device=dev).half()
    we = (rs.randn(ce, cin) / cin ** 0.5).astype(np.float32)
    wek = np.zeros(lib.lp_block_s1_wexp_elems(cin, ce), np.uint16)
    w16 = np.ascontiguousarray(we.astype(np.float16)).view(np.uint16)
    _lib.check(lib.lp_block_s1_pack_wexp(w16.ctypes.data, cin, ce, wek.ctypes.data))
    wed = torch.from_numpy(wek).view(torch.float16).to(dev)
    be = torch.zeros(ce, device=dev); bd = torch.zeros(ce, device=dev)
    wd = (torch.randn((49, ce), device=dev) * 0.1).half()
    wpd, bpd = pack_pw(rs.randn(co, ce) / ce ** 0.5, ce, co)
    wexp, bexp = pack_pw(we, cin, ce)
    ho = hw // 2
    e = torch.empty((n, hw, hw, ce), dtype=torch.float16, device=dev)
    d = torch.empty((n, ho, ho, ce), dtype=torch.float16, device=dev)
    o = torch.empty((n, ho, ho, co), dtype=torch.float16, device=dev)
    t_blk = timeit(lambda: _lib.check(lib.lp_block_s2_f16(x.data_ptr(), wed.data_ptr(), be.data_ptr(), wd.data_ptr(), bd.data_ptr(),
                                                           wpd.data_ptr(), bpd.data_ptr(), o.data_ptr(), n, hw, hw, cin, ce, co, s)))
    t_exp = timeit(lambda: _lib.check(lib.lp_pw1x1_f16(x.data_ptr(), wexp.data_ptr(), bexp.data_ptr(), None, e.data_ptr(), n * hw * hw, cin, ce, 2, s)))
    t_dw = timeit(lambda: _lib.check(lib.lp_dwconv_f16(e.data_ptr(), wd.data_ptr(), bd.data_ptr(), d.data_ptr(), n, ce, hw, hw, 7, 2, 2, s)))
    t_pj = timeit(lambda: _lib.check(lib.lp_pw1x1_f16(d.data_ptr(), wpd.data_ptr(), bpd.data_ptr(), None, o.data_ptr(), n * ho * ho, ce, co, 0, s)))
    chain = t_exp + t_dw + t_pj
    out["s2 %dx%dx%dx%d->%d->%d" % (n, hw, hw, cin, ce, co)] = {
        "block_s2_us": t_blk, "expand_us": t_exp, "dwconv_s2_us": t_dw, "project_us": t_pj, "chain_us": chain,
        "speedup": chain / t_blk, "dw_tmacs": n * ho * ho * ce * 49 / t_blk / 1e6,
        "hbm_gbs": n * (hw * hw * cin + ho * ho * co) * 2 / t_blk / 1e3}
try:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    gpu = r.stdout.strip().splitlines()[0]
except Exception:
    gpu = torch.cuda.get_device_name(0)
print(json.dumps({"gpu": gpu, "shapes": out}))
