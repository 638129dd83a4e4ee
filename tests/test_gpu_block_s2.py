"""-m gpu: the fused stride-2 block kernel (lp_block_s2_f16) equals the three-kernel chain it replaces,
lp_pw1x1_f16 (ReLU6) -> lp_dwconv_f16 (k7, stride 2, ReLU6, packed fp16) -> lp_pw1x1_f16, value for value.

Both expand with one wgmma per K=16 slice and round (acc + bias) to fp16 before the ReLU6, both run the depthwise chain
of dw_inner.cuh (stride 2 has no mirrored lanes), and both project over the same K=16 slices in channel order (four per
64-channel K block, the slices past Ce adding exact zeros) with one rounding of acc + bias."""
import numpy as np
import pytest
import torch

import dw_emul as de
from litepose_b200 import _lib
from gpu_util import pack_pw, stream

pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _inputs(n, h, w, cin, ce, co, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, h, w, cin)).astype(np.float16)
    we = (rng.standard_normal((ce, cin)) / cin ** 0.5).astype(np.float16)
    be = (rng.standard_normal(ce) * 0.2).astype(np.float32)
    _, wd, bd = de.make_inputs(1, ce, 1, 1, 7, "relu6", seed + 1)
    wp = (rng.standard_normal((co, ce)) / ce ** 0.5).astype(np.float16)
    bp = (rng.standard_normal(co) * 0.1).astype(np.float32)
    return x, we, be, wd, bd, wp, bp


def _pw(a, wpk, bpk, m, k, n, act):
    lib = _lib.load()
    out = torch.full((m, n), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_pw1x1_f16(a.data_ptr(), wpk.data_ptr(), bpk.data_ptr(), None, out.data_ptr(), m, k, n, act,
                                stream()), "pw1x1")
    return out


class _Block(object):
    """device weights of one block in both layouts (fused kernel and chain)"""

    def __init__(self, n, h, w, cin, ce, co, seed):
        lib = _lib.load()
        self.shape = (n, h, w, cin, ce, co)
        x, we, be, wd, bd, wp, bp = _inputs(n, h, w, cin, ce, co, seed)
        self.xd, self.wdd, self.bdd, self.bed = _dev(x), _dev(wd), _dev(bd), _dev(be)
        self.wpk, self.bpk = pack_pw(torch.from_numpy(wp), torch.from_numpy(bp))
        wek = np.zeros(lib.lp_block_s1_wexp_elems(cin, ce), np.uint16)
        _lib.check(lib.lp_block_s1_pack_wexp(we.view(np.uint16).ctypes.data, cin, ce, wek.ctypes.data))
        self.wed = torch.from_numpy(wek).view(torch.float16).cuda()
        self.wek2, self.bek2 = pack_pw(torch.from_numpy(we), torch.from_numpy(be))

    def fused(self):
        lib = _lib.load()
        n, h, w, cin, ce, co = self.shape
        out = torch.full((n, h // 2, w // 2, co), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(lib.lp_block_s2_f16(self.xd.data_ptr(), self.wed.data_ptr(), self.bed.data_ptr(), self.wdd.data_ptr(),
                                       self.bdd.data_ptr(), self.wpk.data_ptr(), self.bpk.data_ptr(), out.data_ptr(), n,
                                       h, w, cin, ce, co, stream()), "block_s2")
        torch.cuda.synchronize()
        return out.cpu().numpy()

    def chain(self):
        lib = _lib.load()
        n, h, w, cin, ce, co = self.shape
        e = _pw(self.xd, self.wek2, self.bek2, n * h * w, cin, ce, de.ACT_RELU6)
        mid = torch.full((n, h // 2, w // 2, ce), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(lib.lp_dwconv_f16(e.data_ptr(), self.wdd.data_ptr(), self.bdd.data_ptr(), mid.data_ptr(), n, ce, h, w,
                                     7, 2, de.ACT_RELU6, stream()), "dwconv")
        out = _pw(mid, self.wpk, self.bpk, n * (h // 2) * (w // 2), ce, co, de.ACT_NONE)
        torch.cuda.synchronize()
        return out.cpu().numpy().reshape(n, h // 2, w // 2, co)


def assert_equal_values(got, want, what):
    got = np.asarray(got)
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    neq = got != want            # float compare: -0 == +0
    assert not neq.any(), "%s: %d of %d elements differ (first at %s: %r vs %r)" % (
        what, neq.sum(), neq.size, np.argwhere(neq)[0], got[neq][0], want[neq][0])


SHAPES = [
    (2, 256, 256, 16, 96, 16),      # LitePose-XS / S stage 0, block 0
    (2, 128, 128, 16, 96, 32),      # LitePose-XS / S stage 1, block 0
    (2, 256, 256, 16, 96, 24),      # LitePose-M stage 0, block 0
    (3, 40, 52, 16, 96, 16),        # ragged: 20 x 26 output, partial tiles in x and y
    (2, 4, 6, 16, 96, 16),          # 2 x 3 output: one tile, mostly outside the map
    (2, 64, 64, 16, 32, 16),        # one slab: the second warpgroup has none
    (2, 64, 64, 16, 160, 16),       # five slabs, three K blocks
    (2, 64, 64, 16, 96, 8),         # half a projection chunk
    (2, 64, 64, 16, 96, 40),        # three projection chunks, the last one partial
    (2, 64, 64, 8, 48, 16),         # Cin = 8 (zero-filled K half), a partial slab
    (16, 256, 256, 16, 96, 16),     # about 16 tiles per CTA
    (1, 32, 32, 16, 96, 16),        # two tiles: a grid below the SM count
]


@pytest.mark.parametrize("n,h,w,cin,ce,co", SHAPES)
def test_block_s2_equals_pw1x1_dwconv_pw1x1(n, h, w, cin, ce, co):
    lib = _lib.load()
    assert lib.lp_block_s2_supported(cin, ce, co) == 1
    lib.lp_set_dw_precision(-1)
    blk = _Block(n, h, w, cin, ce, co, cin * 5 + ce * 3 + co + h + w + n)
    assert_equal_values(blk.fused(), blk.chain(), "block_s2 n%d %dx%d cin%d ce%d co%d" % (n, h, w, cin, ce, co))


def test_block_s2_repeated_launches_identical():
    blk = _Block(4, 128, 128, 16, 96, 32, 7)
    first = blk.fused()
    for _ in range(3):
        again = blk.fused()
        assert np.array_equal(first.view(np.uint16), again.view(np.uint16))


def test_block_s2_rejects_odd_maps_on_device():
    lib = _lib.load()
    x = torch.zeros(1 << 16, dtype=torch.float16, device="cuda")
    for h, w in ((31, 32), (32, 33)):
        rc = lib.lp_block_s2_f16(x.data_ptr(), x.data_ptr(), None, x.data_ptr(), None, x.data_ptr(), None, x.data_ptr(),
                                 1, h, w, 16, 96, 16, stream())
        assert rc == 1 and b"lp_block_s2_f16" in lib.lp_last_error()


def test_litepose_s_512_plan_fuses_blocks_a_and_b():
    """an S-512 plan runs stage 0 / 1 block 0 (16 -> 96 -> 16 / 32) as block_s2 and keeps the k7 s2 dw7 of stage 2"""
    from litepose_b200 import synth
    from litepose_b200.config import get_arch, get_cfg
    from litepose_b200.engine import LitePoseEngine
    from litepose_b200.lib.models.pose_mobilenet import get_pose_net

    arch = get_arch("S")
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(get_cfg(input_size=512), False, arch), 1).eval()
    eng = LitePoseEngine(model.state_dict(), arch, "cuda")
    plan = eng.plan_for(2, 512, 512, torch.float16, True)
    s2 = [tuple(op.args[8:14]) for op in plan["ops"] if op.name == "block_s2"]
    assert s2 == [(2, 256, 256, 16, 96, 16), (2, 128, 128, 16, 96, 32)]
    dw7_s2 = [op for op in plan["ops"] if op.name == "dw7" and tuple(op.args[8:10]) == (7, 2)]
    assert len(dw7_s2) == 1 and dw7_s2[0].args[4:8] == [2, dw7_s2[0].args[5], 64, 64]
