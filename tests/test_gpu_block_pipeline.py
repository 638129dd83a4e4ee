"""-m gpu: the fused stride-1 block kernel (lp_block_s1_f16) against the unfused pair that computes the same block in two
launches, lp_pw1x1_f16 (expansion + ReLU6, fp16 intermediate in HBM) + lp_dw7_project_f16 (depthwise + projection
+ identity).

Both paths expand each K=16 slice in fp32 and round to fp16 after bias + ReLU6, run the same packed-fp16 depthwise chain
and accumulate the projection in fp32 K block by K block, so the fused kernel's output is bit-identical to the pair's.
The pair is also checked against the fp32 oracle with fp16 storage of the two intermediates."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from litepose_b200 import _lib
from gpu_util import from_nhwc, nhwc16, pack_pw, q16, stream, tol_check

pytestmark = pytest.mark.gpu

# (n, h, w, cin, ce, co, identity)
MODEL_SHAPES = [
    (2, 128, 128, 16, 96, 16, True),       # XS/S stage 0
    (2, 64, 64, 32, 192, 32, True),        # XS/S stage 1
    (2, 32, 32, 48, 288, 48, True),        # XS/S stage 2 (streaming layout)
    (2, 128, 128, 24, 144, 24, True),      # M/L stage 0
    (2, 64, 64, 48, 288, 48, True),        # M stage 1
    (2, 64, 64, 64, 384, 64, True),        # L stage 1
    (3, 40, 52, 16, 96, 16, True),         # ragged tiles on both axes
    (2, 20, 28, 48, 288, 48, True),
]
SCHEDULE_SHAPES = [
    (16, 128, 128, 16, 96, 16, True),      # ~8 tiles per persistent CTA: buffer parities wrap many times
    (8, 64, 64, 32, 192, 32, True),
    (20, 32, 32, 48, 288, 48, True),       # streaming layout, several tiles per CTA
    (4, 64, 64, 32, 160, 32, False),       # odd slab count (5), no identity
    (5, 48, 48, 16, 96, 16, False),        # odd slab count (3), no identity, odd tile count per CTA
    (1, 32, 48, 32, 192, 32, True),        # 6 tiles: grid far below the SM count
    (1, 16, 16, 16, 32, 16, False),        # one slab, one K block, one tile
    (2, 32, 32, 32, 64, 48, False),        # two slabs, Co padded 48 -> three projection chunks
    (1, 16, 16, 64, 160, 64, True),        # widest input / output
    (3, 48, 48, 40, 320, 56, False),       # streaming layout, ragged Co chunking
]


def _block(n, h, w, cin, ce, co, res):
    g = torch.Generator().manual_seed(cin * 5 + ce * 3 + co + h + n)
    x = q16(torch.randn(n, cin, h, w, generator=g))
    we = q16(torch.randn(ce, cin, generator=g) / (cin ** 0.5))
    be = torch.randn(ce, generator=g) * 0.2
    wd = q16(torch.randn(ce, 1, 7, 7, generator=g) * 0.1)
    bd = torch.randn(ce, generator=g) * 0.1
    wp = q16(torch.randn(co, ce, generator=g) / (ce ** 0.5))
    bp = torch.randn(co, generator=g) * 0.1
    return x, we, be, wd, bd, wp, bp


@pytest.mark.parametrize("n,h,w,cin,ce,co,res", MODEL_SHAPES + SCHEDULE_SHAPES)
def test_block_s1_matches_unfused_pair(n, h, w, cin, ce, co, res):
    lib = _lib.load()
    assert lib.lp_block_s1_supported(cin, ce, co) == 1
    x, we, be, wd, bd, wp, bp = _block(n, h, w, cin, ce, co, res)
    xd = nhwc16(x)
    wdd = wd.reshape(ce, 49).t().contiguous().half().cuda()
    bed, bdd = be.cuda(), bd.cuda()
    wpk, bpk = pack_pw(wp, bp)
    # fused: expansion weights in the block kernel's packing
    we16 = np.ascontiguousarray(we.half().numpy()).view(np.uint16)
    wek = np.zeros(lib.lp_block_s1_wexp_elems(cin, ce), np.uint16)
    _lib.check(lib.lp_block_s1_pack_wexp(we16.ctypes.data, cin, ce, wek.ctypes.data))
    wed = torch.from_numpy(wek).view(torch.float16).cuda()
    fused = torch.full((n, h, w, co), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_block_s1_f16(xd.data_ptr(), wed.data_ptr(), bed.data_ptr(), wdd.data_ptr(), bdd.data_ptr(),
                                   wpk.data_ptr(), bpk.data_ptr(), 1 if res else 0, fused.data_ptr(),
                                   n, h, w, cin, ce, co, stream()), "block_s1")
    # unfused pair
    wek2, bek2 = pack_pw(we, be)
    e = torch.full((n, h, w, ce), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_pw1x1_f16(xd.data_ptr(), wek2.data_ptr(), bek2.data_ptr(), None, e.data_ptr(), n * h * w, cin, ce,
                                2, stream()), "pw1x1")
    pair = torch.full((n, h, w, co), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_dw7_project_f16(e.data_ptr(), wdd.data_ptr(), bdd.data_ptr(), wpk.data_ptr(), bpk.data_ptr(),
                                      xd.data_ptr() if res else None, pair.data_ptr(), n, h, w, ce, co, stream()),
               "dw7_project")
    torch.cuda.synchronize()
    what = "block_s1 n%d %dx%d cin%d ce%d co%d" % (n, h, w, cin, ce, co)
    assert not torch.isnan(fused).any(), what
    ndiff = (fused.view(torch.int16) != pair.view(torch.int16)).sum().item()
    assert ndiff == 0, "%s: %d of %d outputs differ from the unfused pair (max |diff| %.3e)" % (
        what, ndiff, fused.numel(), (fused.float() - pair.float()).abs().max().item())
    # the pair itself against the fp32 oracle (fp16 storage of both intermediates)
    if n * h * w <= 2 * 128 * 128:
        mid = q16(F.relu6(F.conv2d(q16(F.relu6(F.conv2d(x, we.view(ce, cin, 1, 1), be))), wd, bd, 1, 3, 1, ce)))
        ref = F.conv2d(mid, wp.view(co, ce, 1, 1), bp)
        if res:
            ref = ref + x
        tol_check(from_nhwc(fused), ref, what=what)


def test_block_s1_repeated_launches_identical():
    """persistent CTAs keep no state between launches: the same input gives the same bits every launch"""
    lib = _lib.load()
    n, h, w, cin, ce, co = 12, 64, 64, 32, 192, 32
    x, we, be, wd, bd, wp, bp = _block(n, h, w, cin, ce, co, True)
    xd = nhwc16(x)
    wdd = wd.reshape(ce, 49).t().contiguous().half().cuda()
    bed, bdd = be.cuda(), bd.cuda()
    wpk, bpk = pack_pw(wp, bp)
    we16 = np.ascontiguousarray(we.half().numpy()).view(np.uint16)
    wek = np.zeros(lib.lp_block_s1_wexp_elems(cin, ce), np.uint16)
    _lib.check(lib.lp_block_s1_pack_wexp(we16.ctypes.data, cin, ce, wek.ctypes.data))
    wed = torch.from_numpy(wek).view(torch.float16).cuda()
    outs = []
    for _ in range(3):
        o = torch.full((n, h, w, co), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(lib.lp_block_s1_f16(xd.data_ptr(), wed.data_ptr(), bed.data_ptr(), wdd.data_ptr(), bdd.data_ptr(),
                                       wpk.data_ptr(), bpk.data_ptr(), 1, o.data_ptr(), n, h, w, cin, ce, co, stream()),
                   "block_s1")
        outs.append(o)
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(o.view(torch.int16), outs[0].view(torch.int16))
