"""-m gpu: lp_dw7_project_f16 at projection widths above 64 (the warp-specialised wide kernel) against the same call
split into ceil(Co/64) launches of at most 64 output channels each (the narrow kernel), then concatenated.

Both run the same packed-fp16 depthwise chain, and each output column accumulates its fp32 projection over the same
K=16 slices in channel order, adding bias and residual in the same order, so the outputs must be bit-identical."""
import pytest
import torch

from litepose_b200 import _lib
from gpu_util import nhwc16, pack_pw, q16, stream

pytestmark = pytest.mark.gpu

# (n, h, w, ce, co, res)
SHAPES = [
    (2, 32, 32, 720, 120, True),       # LitePose-S stage 3
    (2, 32, 32, 288, 120, False),      # its first block (Ce = 288: 9 slabs, odd)
    (1, 32, 32, 288, 72, True),        # Co = 72: five 16-column chunks
    (2, 32, 32, 480, 80, True),        # XS stage 3 width
    (1, 32, 32, 576, 96, False),
    (1, 32, 32, 960, 160, True),       # widest projection, 30 slabs
    (1, 16, 16, 960, 136, False),      # nine chunks
    (2, 16, 16, 720, 128, True),
    (1, 20, 40, 432, 72, False),       # ragged map, 27 slabs
    (2, 48, 48, 720, 120, True),       # ragged vertically (48 = 6 tiles of 8), many tiles
    (24, 48, 48, 720, 120, True),      # many tiles per persistent CTA
    (1, 8, 16, 288, 120, True),        # one tile: grid far below the SM count
    (3, 20, 40, 96, 160, False),       # 3 slabs, ragged map
    (1, 16, 16, 8, 72, True),          # one slab with 8 channels: the odd-slab group has nothing to do
]


@pytest.mark.parametrize("n,h,w,ce,co,res", SHAPES)
def test_dw7_project_wide_matches_narrow_launches(n, h, w, ce, co, res):
    lib = _lib.load()
    g = torch.Generator().manual_seed(ce * 3 + co + h + n)
    x = q16(torch.rand(n, ce, h, w, generator=g) * 3.0)
    wd = q16(torch.randn(ce, 1, 7, 7, generator=g) * 0.15)
    bd = torch.randn(ce, generator=g) * 0.1
    wp = q16(torch.randn(co, ce, generator=g) / (ce ** 0.5))
    bp = torch.randn(co, generator=g) * 0.1
    r = q16(torch.randn(n, co, h, w, generator=g)) if res else None
    xd = nhwc16(x)
    wdd = wd.reshape(ce, 49).t().contiguous().half().cuda()
    bdd = bd.cuda()
    rd = nhwc16(r) if res else None

    wpk, bpk = pack_pw(wp, bp)
    wide = torch.full((n, h, w, co), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_dw7_project_f16(xd.data_ptr(), wdd.data_ptr(), bdd.data_ptr(), wpk.data_ptr(), bpk.data_ptr(),
                                      rd.data_ptr() if res else None, wide.data_ptr(), n, h, w, ce, co, stream()),
               "dw7_project wide")
    parts = []
    for c0 in range(0, co, 64):
        c1 = min(co, c0 + 64)
        wpk_s, bpk_s = pack_pw(wp[c0:c1].contiguous(), bp[c0:c1].contiguous())
        rd_s = rd[..., c0:c1].contiguous() if res else None
        o = torch.full((n, h, w, c1 - c0), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(lib.lp_dw7_project_f16(xd.data_ptr(), wdd.data_ptr(), bdd.data_ptr(), wpk_s.data_ptr(),
                                          bpk_s.data_ptr(), rd_s.data_ptr() if res else None, o.data_ptr(), n, h, w,
                                          ce, c1 - c0, stream()), "dw7_project narrow")
        parts.append(o)
        torch.cuda.synchronize()      # rd_s / the packed slices must outlive their launch
    narrow = torch.cat(parts, dim=-1)
    what = "dw7_project n%d %dx%d ce%d co%d res%d" % (n, h, w, ce, co, res)
    assert not torch.isnan(wide).any(), what
    ndiff = (wide.view(torch.int16) != narrow.view(torch.int16)).sum().item()
    assert ndiff == 0, "%s: %d of %d outputs differ from the narrow launches (max |diff| %.3e)" % (
        what, ndiff, wide.numel(), (wide.float() - narrow.float()).abs().max().item())


def test_dw7_project_wide_repeated_launches_identical():
    """persistent CTAs keep no state between launches: the same input gives the same bits every launch"""
    lib = _lib.load()
    n, h, w, ce, co = 8, 32, 32, 720, 120
    g = torch.Generator().manual_seed(5)
    xd = nhwc16(q16(torch.rand(n, ce, h, w, generator=g) * 3.0))
    wdd = q16(torch.randn(49, ce, generator=g) * 0.15).half().cuda()
    bdd = (torch.randn(ce, generator=g) * 0.1).cuda()
    wpk, bpk = pack_pw(q16(torch.randn(co, ce, generator=g) / (ce ** 0.5)), torch.randn(co, generator=g) * 0.1)
    outs = []
    for _ in range(3):
        o = torch.full((n, h, w, co), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(lib.lp_dw7_project_f16(xd.data_ptr(), wdd.data_ptr(), bdd.data_ptr(), wpk.data_ptr(), bpk.data_ptr(),
                                          None, o.data_ptr(), n, h, w, ce, co, stream()), "dw7_project wide")
        outs.append(o)
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(o.view(torch.int16), outs[0].view(torch.int16))
