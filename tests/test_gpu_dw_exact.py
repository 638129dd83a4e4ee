"""-m gpu: the depthwise kernels against the bit-exact emulator (dw_emul.py), and the fused kernels reduced to it.

(a) lp_dwconv_f16 equals dw_emul.dwconv element for element, for every (k, stride, precision, activation), and at the
    stride-2 7x7 launches of a LitePose-S 512x512 pass.
(b) lp_set_dw_precision selects the arithmetic it names; -1 restores the per-kernel-size default.
(c) The fused kernels equal the unfused kernels they replace, as values:
      lp_dw7_project_f16(x) == lp_pw1x1_f16(lp_dwconv_f16(x, k7 s1 ReLU6, prec 2), proj, bias, residual)
    (same packed-fp16 depthwise; both projections accumulate the same K=16 slices in order, zero slices add exact zeros,
    and both epilogues round (acc + bias) + residual to fp16 once), lp_block_s1_f16 == pw1x1 . dwconv . pw1x1, and
    lp_head_fused_f16 == lp_head_pw_dual_f16 on two lp_dwconv_f16(k5, prec 0, ReLU) outputs.
(d) The tensor-core reductions element by element against fp64 on exactly the fp16 operands they multiply (the emulated
    depthwise output for the fused kernels): |got - ref| <= 2^-11 |ref| + K 2^-22 S + 2^-24, S = sum |a| |w| + |bias| +
    |residual| (fp16 subnormal operands lifted to 2^-14).  The K 2^-22 S term covers the tensor-core accumulation
    measured on the H100 (mma_emul.MODEL: 16 products and the addend cut to 25 bits below the block's leading exponent,
    rounded toward zero into fp32; gpu_util.check_bound derives the bound); the worst err / bound of each case is
    recorded with gpu_util._record."""
import numpy as np
import pytest
import torch

import dw_emul as de
from litepose_b200 import _lib
from gpu_util import check_reduction, pack_pw, stream

pytestmark = pytest.mark.gpu

CHANNELS = [8, 24, 40, 96, 144, 720]     # 8, 24, 40: a partial 32-channel slab
KINDS = ["relu6", "signed", "tiny"]
COMBOS = [(p, a) for p in (0, 1, 2) for a in (0, 1, 2)]


def dw_cases(k, s, prec, act):
    """(n, c, h, w, kind, seed) per (k, s, prec, act): a map ragged against the 32 (s1) / 16 (s2 output) tiles with one of
    CHANNELS (rotating through the (prec, act) combinations, so every k, s sees every channel count), a map with
    W < 8 and W % 4 != 0 (partial mirrored stores), and a tiny map (2x2 for stride 2)."""
    i = COMBOS.index((prec, act))
    c = CHANNELS[(i + k + s) % len(CHANNELS)]
    n = 3 if c <= 144 else 1
    seed = 1000 * k + 100 * s + 10 * prec + act
    if s == 1:
        maps = [(n, c, 37, 45), (3, 40, 9, 6), (3, 24, 5, 5)]
    else:
        maps = [(n, c, 38, 42), (3, 40, 6, 10), (3, 24, 2, 2)]
    return [m + (KINDS[(i + j) % 3], seed + j) for j, m in enumerate(maps)]


def prec_switch_case(k):
    return (2, 40, 37, 45, "relu6", 77 + k)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_dwconv(x, wt, b, k, s, act):
    """lp_dwconv_f16 at the current precision setting; numpy in, numpy out"""
    lib = _lib.load()
    n, h, w, c = x.shape
    xd, wd, bd = _dev(x), _dev(wt), _dev(b)
    y = torch.full((n, h // s, w // s, c), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_dwconv_f16(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), y.data_ptr(), n, c, h, w, k, s, act,
                                 stream()), "dwconv")
    torch.cuda.synchronize()
    return y.cpu().numpy()


def assert_equal_values(got, want, what):
    got = np.asarray(got)
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    neq = got != want            # float compare: -0 == +0 (hmax may leave a -0)
    assert not neq.any(), "%s: %d of %d elements differ (first at %s: %r vs %r)" % (
        what, neq.sum(), neq.size, np.argwhere(neq)[0], got[neq][0], want[neq][0])


@pytest.fixture
def dw_precision():
    """sets lp_set_dw_precision for the test and always restores the per-kernel-size default"""
    lib = _lib.load()
    try:
        yield lib.lp_set_dw_precision
    finally:
        lib.lp_set_dw_precision(-1)


# ---------------------------------------------------------------- (a) lp_dwconv_f16 == emulator
@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("s", [1, 2])
@pytest.mark.parametrize("prec,act", COMBOS)
def test_dwconv_bit_exact(k, s, prec, act, dw_precision):
    dw_precision(prec)
    for n, c, h, w, kind, seed in dw_cases(k, s, prec, act):
        x, wt, b = de.make_inputs(n, c, h, w, k, kind, seed)
        got = run_dwconv(x, wt, b, k, s, act)
        assert_equal_values(got, de.dwconv(x, wt, b, k, s, act, prec),
                            "dwconv k%d s%d prec%d act%d n%d c%d %dx%d %s" % (k, s, prec, act, n, c, h, w, kind))


def test_dwconv_bit_exact_litepose_s_512_stride2_launches(dw_precision):
    """the stride-2 7x7 depthwise launches of a LitePose-S 512x512 batch-2 pass, shapes from the engine's own plan"""
    from litepose_b200 import synth
    from litepose_b200.config import get_arch, get_cfg
    from litepose_b200.engine import LitePoseEngine
    from litepose_b200.lib.models.pose_mobilenet import get_pose_net

    dw_precision(-1)
    arch = get_arch("S")
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(get_cfg(input_size=512), False, arch), 1).eval()
    eng = LitePoseEngine(model.state_dict(), arch, "cuda")
    plan = eng.plan_for(2, 512, 512, torch.float16, True)
    shapes = sorted({tuple(op.args[4:11]) for op in plan["ops"] if op.name == "dw7" and tuple(op.args[8:10]) == (7, 2)})
    assert shapes, "no stride-2 7x7 depthwise launch in the plan"
    for i, (n, c, h, w, k, s, act) in enumerate(shapes):
        x, wt, b = de.make_inputs(n, c, h, w, k, "relu6", 500 + i)
        got = run_dwconv(x, wt, b, k, s, act)
        assert_equal_values(got, de.dwconv(x, wt, b, k, s, act, de.default_prec(k)),
                            "LitePose-S 512 dw7 n%d c%d %dx%d" % (n, c, h, w))


# ---------------------------------------------------------------- (b) the precision switch
@pytest.mark.parametrize("k", [3, 5, 7])
def test_dw_precision_switch(k, dw_precision):
    n, c, h, w, kind, seed = prec_switch_case(k)
    x, wt, b = de.make_inputs(n, c, h, w, k, kind, seed)
    want = {p: de.dwconv(x, wt, b, k, 1, de.ACT_RELU6, p) for p in (0, 1, 2)}
    for p, q in ((0, 1), (0, 2), (1, 2)):
        assert (want[p] != want[q]).any(), "the input does not tell prec %d from %d" % (p, q)
    for p in (0, 1, 2, -1):
        dw_precision(p)
        got = run_dwconv(x, wt, b, k, 1, de.ACT_RELU6)
        assert_equal_values(got, want[p if p >= 0 else de.default_prec(k)], "k%d lp_set_dw_precision(%d)" % (k, p))


# ---------------------------------------------------------------- (c) fused kernels == the unfused kernels
# (n, h, w, ce, co, res): Co <= 64 run dw_project_kernel, wider dw_project_wide_kernel
DW7_PROJECT_SHAPES = [
    (2, 32, 32, 96, 16, True), (1, 16, 16, 96, 16, False), (2, 48, 32, 192, 32, True), (1, 32, 32, 288, 48, True),
    (2, 16, 16, 144, 24, True), (3, 64, 64, 96, 16, True), (5, 96, 112, 160, 32, True), (36, 32, 32, 288, 48, True),
    (20, 48, 48, 48, 8, False), (6, 80, 80, 32, 16, True), (1, 20, 36, 224, 64, False), (2, 37, 45, 40, 64, True),
    (2, 32, 32, 720, 120, True), (2, 32, 32, 288, 120, False), (1, 32, 32, 288, 72, True), (1, 32, 32, 960, 160, True),
    (1, 20, 40, 432, 72, False), (24, 48, 48, 720, 120, True), (1, 8, 16, 288, 120, True), (3, 20, 40, 96, 160, False),
    (1, 16, 16, 8, 72, True),
]


def _proj_inputs(n, h, w, ce, co, res, seed):
    rng = np.random.default_rng(seed)
    x, wd, bd = de.make_inputs(n, ce, h, w, 7, "relu6", seed)
    wp = (rng.standard_normal((co, ce)) / ce ** 0.5).astype(np.float16)
    bp = (rng.standard_normal(co) * 0.1).astype(np.float32)
    r = rng.standard_normal((n, h, w, co)).astype(np.float16) if res else None
    return x, wd, bd, wp, bp, r


def _pw(a, wpk, bpk, r, m, k, n, act):
    lib = _lib.load()
    out = torch.full((m, n), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_pw1x1_f16(a.data_ptr(), wpk.data_ptr(), bpk.data_ptr(), None if r is None else r.data_ptr(),
                                out.data_ptr(), m, k, n, act, stream()), "pw1x1")
    return out


def _dw7_project(xd, wdd, bdd, wpk, bpk, rd, n, h, w, ce, co):
    lib = _lib.load()
    out = torch.full((n, h, w, co), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_dw7_project_f16(xd.data_ptr(), wdd.data_ptr(), bdd.data_ptr(), wpk.data_ptr(), bpk.data_ptr(),
                                      None if rd is None else rd.data_ptr(), out.data_ptr(), n, h, w, ce, co, stream()),
               "dw7_project")
    return out


@pytest.mark.parametrize("n,h,w,ce,co,res", DW7_PROJECT_SHAPES)
def test_dw7_project_equals_dwconv_then_pw1x1(n, h, w, ce, co, res, dw_precision):
    lib = _lib.load()
    dw_precision(2)
    x, wd, bd, wp, bp, r = _proj_inputs(n, h, w, ce, co, res, ce * 3 + co + h + n)
    xd, wdd, bdd = _dev(x), _dev(wd), _dev(bd)
    rd = _dev(r) if res else None
    wpk, bpk = pack_pw(torch.from_numpy(wp), torch.from_numpy(bp))
    fused = _dw7_project(xd, wdd, bdd, wpk, bpk, rd, n, h, w, ce, co)
    mid = torch.full((n, h, w, ce), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_dwconv_f16(xd.data_ptr(), wdd.data_ptr(), bdd.data_ptr(), mid.data_ptr(), n, ce, h, w, 7, 1,
                                 de.ACT_RELU6, stream()), "dwconv")
    pair = _pw(mid, wpk, bpk, rd, n * h * w, ce, co, de.ACT_NONE)
    torch.cuda.synchronize()
    assert_equal_values(fused.cpu().numpy().reshape(-1, co), pair.cpu().numpy(),
                        "dw7_project n%d %dx%d ce%d co%d res%d" % (n, h, w, ce, co, res))


@pytest.mark.parametrize("n,h,w,cin,ce,co,res", [
    (2, 128, 128, 16, 96, 16, True), (2, 64, 64, 32, 192, 32, True), (2, 32, 32, 48, 288, 48, True),
    (2, 128, 128, 24, 144, 24, True), (2, 64, 64, 48, 288, 48, True), (2, 64, 64, 64, 384, 64, True),
    (3, 40, 52, 16, 96, 16, True), (2, 20, 28, 48, 288, 48, True),
])
def test_block_s1_equals_pw1x1_dwconv_pw1x1(n, h, w, cin, ce, co, res, dw_precision):
    """one case per LitePose block shape of test_gpu_block_pipeline.MODEL_SHAPES"""
    lib = _lib.load()
    dw_precision(2)
    rng = np.random.default_rng(cin * 5 + ce * 3 + co + h + n)
    x = rng.standard_normal((n, h, w, cin)).astype(np.float16)
    we = (rng.standard_normal((ce, cin)) / cin ** 0.5).astype(np.float16)
    be = (rng.standard_normal(ce) * 0.2).astype(np.float32)
    _, wd, bd = de.make_inputs(1, ce, 1, 1, 7, "relu6", ce + h)
    wp = (rng.standard_normal((co, ce)) / ce ** 0.5).astype(np.float16)
    bp = (rng.standard_normal(co) * 0.1).astype(np.float32)
    xd, wdd, bdd, bed = _dev(x), _dev(wd), _dev(bd), _dev(be)
    wpk, bpk = pack_pw(torch.from_numpy(wp), torch.from_numpy(bp))
    wek = np.zeros(lib.lp_block_s1_wexp_elems(cin, ce), np.uint16)
    _lib.check(lib.lp_block_s1_pack_wexp(we.view(np.uint16).ctypes.data, cin, ce, wek.ctypes.data))
    wed = torch.from_numpy(wek).view(torch.float16).cuda()
    fused = torch.full((n, h, w, co), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_block_s1_f16(xd.data_ptr(), wed.data_ptr(), bed.data_ptr(), wdd.data_ptr(), bdd.data_ptr(),
                                   wpk.data_ptr(), bpk.data_ptr(), 1 if res else 0, fused.data_ptr(), n, h, w, cin, ce,
                                   co, stream()), "block_s1")
    wek2, bek2 = pack_pw(torch.from_numpy(we), torch.from_numpy(be))
    e = _pw(xd, wek2, bek2, None, n * h * w, cin, ce, de.ACT_RELU6)
    mid = torch.full((n, h, w, ce), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_dwconv_f16(e.data_ptr(), wdd.data_ptr(), bdd.data_ptr(), mid.data_ptr(), n, ce, h, w, 7, 1,
                                 de.ACT_RELU6, stream()), "dwconv")
    chain = _pw(mid, wpk, bpk, xd if res else None, n * h * w, ce, co, de.ACT_NONE)
    torch.cuda.synchronize()
    assert_equal_values(fused.cpu().numpy().reshape(-1, co), chain.cpu().numpy(),
                        "block_s1 n%d %dx%d cin%d ce%d co%d" % (n, h, w, cin, ce, co))


HEAD_SHAPES = [
    (2, 32, 32, 24, 16, 28, True), (1, 64, 64, 32, 16, 14, True), (1, 48, 16, 40, 24, 28, False),
    (2, 16, 16, 64, 24, 34, True), (1, 20, 36, 24, 16, 28, True), (6, 96, 96, 24, 16, 28, True),
    (5, 80, 96, 40, 24, 28, False), (1, 37, 45, 72, 40, 128, True),
]


def _head_inputs(n, h, w, c1, c2, co, seed):
    rng = np.random.default_rng(seed)
    x1, d1, b1 = de.make_inputs(n, c1, h, w, 5, "signed", seed + 1)
    x2, d2, b2 = de.make_inputs(n, c2, h, w, 5, "signed", seed + 2)
    w1 = (rng.standard_normal((co, c1)) / c1 ** 0.5).astype(np.float16)
    w2 = (rng.standard_normal((co, c2)) / c2 ** 0.5).astype(np.float16)
    return x1, d1, b1, x2, d2, b2, w1, w2


def _head_fused(x1, d1, b1, x2, d2, b2, w1, w2, n, h, w, c1, c2, co, fp32):
    lib = _lib.load()
    dwc = np.zeros(lib.lp_head_fused_dw_elems(c1, c2), np.uint16)
    bdc = np.zeros(dwc.size // 25, np.float32)
    pwc = np.zeros(lib.lp_head_fused_pw_elems(c1, c2, co), np.uint16)
    _lib.check(lib.lp_head_fused_pack(d1.view(np.uint16).ctypes.data, b1.ctypes.data, d2.view(np.uint16).ctypes.data,
                                      b2.ctypes.data, w1.view(np.uint16).ctypes.data, w2.view(np.uint16).ctypes.data,
                                      c1, c2, co, dwc.ctypes.data, bdc.ctypes.data, pwc.ctypes.data))
    dwd, bdd, pwd = _dev(dwc.view(np.float16)), _dev(bdc), _dev(pwc.view(np.float16))
    s1, s2 = _dev(x1), _dev(x2)
    out = torch.full((n, co, h, w), float("nan"), dtype=torch.float32 if fp32 else torch.float16, device="cuda")
    _lib.check(lib.lp_head_fused_f16(s1.data_ptr(), s2.data_ptr(), dwd.data_ptr(), bdd.data_ptr(), pwd.data_ptr(),
                                     out.data_ptr(), 1 if fp32 else 0, n, h, w, c1, c2, co, stream()), "head_fused")
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("n,h,w,c1,c2,co,fp32", HEAD_SHAPES)
def test_head_fused_equals_dwconv_then_head_pw_dual(n, h, w, c1, c2, co, fp32, dw_precision):
    """Both kernels run one wgmma per K=16 slice into fp32 accumulators that start at zero and store them unrounded
    (fp32) or rounded once (fp16).  lp_head_pw_dual_f16 walks the K blocks of the first source, then those of the
    second; the fused head walks the slab-padded concatenation [C1 | C2] in 64-channel blocks.  Both orders visit the
    16-channel slices of C1 then of C2 in channel order; the fused order only adds slices of zero channels (dwconv
    output 0 against zero-packed weights), which leave the accumulators unchanged, so the results are equal values."""
    lib = _lib.load()
    dw_precision(0)
    x1, d1, b1, x2, d2, b2, w1, w2 = _head_inputs(n, h, w, c1, c2, co, c1 * 7 + c2 + co)
    fused = _head_fused(x1, d1, b1, x2, d2, b2, w1, w2, n, h, w, c1, c2, co, fp32)
    t1 = _dev(run_dwconv(x1, d1, b1, 5, 1, de.ACT_RELU))
    t2 = _dev(run_dwconv(x2, d2, b2, 5, 1, de.ACT_RELU))
    wp = np.zeros(lib.lp_head_packed_elems(c1, c2, co), np.uint16)
    _lib.check(lib.lp_head_pack(w1.view(np.uint16).ctypes.data, w2.view(np.uint16).ctypes.data, c1, c2, co,
                                wp.ctypes.data))
    wd = _dev(wp.view(np.float16))
    out = torch.full((n, co, h, w), float("nan"), dtype=torch.float32 if fp32 else torch.float16, device="cuda")
    _lib.check(lib.lp_head_pw_dual_f16(t1.data_ptr(), t2.data_ptr(), wd.data_ptr(), out.data_ptr(), 1 if fp32 else 0,
                                       n, h, w, c1, c2, co, stream()), "head_pw_dual")
    torch.cuda.synchronize()
    assert_equal_values(fused, out.cpu().numpy(), "head_fused n%d %dx%d c1 %d c2 %d co %d" % (n, h, w, c1, c2, co))


# ---------------------------------------------------------------- (d) tensor-core reductions against fp64
DW7_PROJECT_FP64_SHAPES = [
    (2, 32, 32, 96, 16, True), (2, 16, 16, 144, 24, True), (2, 48, 32, 192, 32, True), (1, 20, 36, 224, 64, False),
    (2, 37, 45, 40, 64, True), (1, 32, 32, 720, 120, True), (1, 20, 40, 432, 72, False), (1, 16, 16, 960, 160, True),
    (3, 20, 40, 96, 160, False), (1, 16, 16, 8, 72, True),
]


@pytest.mark.parametrize("n,h,w,ce,co,res", DW7_PROJECT_FP64_SHAPES)
def test_dw7_project_projection_fp64(n, h, w, ce, co, res):
    x, wd, bd, wp, bp, r = _proj_inputs(n, h, w, ce, co, res, ce * 3 + co + h + n)
    wpk, bpk = pack_pw(torch.from_numpy(wp), torch.from_numpy(bp))
    got = _dw7_project(_dev(x), _dev(wd), _dev(bd), wpk, bpk, _dev(r) if res else None, n, h, w, ce, co)
    torch.cuda.synchronize()
    a = de.dwconv(x, wd, bd, 7, 1, de.ACT_RELU6, 2)
    check_reduction(got.cpu().numpy().reshape(-1, co), a, wp, bp, r, ce,
                    "dw7_project n%d %dx%d ce%d co%d res%d" % (n, h, w, ce, co, res))


@pytest.mark.parametrize("n,h,w,c1,c2,co,fp32", [HEAD_SHAPES[i] for i in (0, 2, 3, 4, 7)])
def test_head_fused_projection_fp64(n, h, w, c1, c2, co, fp32):
    x1, d1, b1, x2, d2, b2, w1, w2 = _head_inputs(n, h, w, c1, c2, co, c1 * 7 + c2 + co)
    got = _head_fused(x1, d1, b1, x2, d2, b2, w1, w2, n, h, w, c1, c2, co, fp32)
    a = np.concatenate([de.dwconv(x1, d1, b1, 5, 1, de.ACT_RELU, 0), de.dwconv(x2, d2, b2, 5, 1, de.ACT_RELU, 0)], -1)
    check_reduction(got.transpose(0, 2, 3, 1).reshape(-1, co), a, np.concatenate([w1, w2], 1), None, None, c1 + c2,
                    "head_fused n%d %dx%d c1 %d c2 %d co %d fp32 %d" % (n, h, w, c1, c2, co, fp32))


# (m, k, n, act, res)
PW_EDGE_SHAPES = [
    (1, 8, 8, 0, False),          # K = 8: a 64-wide TMA box over an 8-wide tensor; a single row
    (63, 8, 24, 2, True),         # residual with N % 64 != 0
    (65, 72, 24, 1, True),        # K = 72: a second K block with 8 valid channels
    (64, 72, 168, 2, False),      # N = 168: two 128-column chunks, the second with 40 columns
    (65, 72, 168, 0, True),       # ... with a residual over the partial chunk
    (1, 96, 1024, 0, True),       # N = 1024 = PW_MAX_BIAS: eight chunks
    (300, 32, 1024, 2, False),
    (63, 448, 256, 0, True),      # streaming weights (7 K blocks of two 128-row chunks), small M
    (1, 960, 160, 0, False),      # streaming weights, one chunk of 160 columns, one row
    (65, 960, 160, 2, True),
    (4096, 24, 8, 1, True),       # N = 8
]


@pytest.mark.parametrize("m,k,n,act,res", PW_EDGE_SHAPES)
def test_pw1x1_fp64(m, k, n, act, res):
    rng = np.random.default_rng(m * 7 + k * 3 + n)
    a = rng.standard_normal((m, k)).astype(np.float16)
    wt = (rng.standard_normal((n, k)) / k ** 0.5).astype(np.float16)
    b = (rng.standard_normal(n) * 0.1).astype(np.float32)
    r = rng.standard_normal((m, n)).astype(np.float16) if res else None
    wpk, bpk = pack_pw(torch.from_numpy(wt), torch.from_numpy(b))
    got = _pw(_dev(a), wpk, bpk, _dev(r) if res else None, m, k, n, act)
    torch.cuda.synchronize()
    check_reduction(got.cpu().numpy(), a, wt, b, r, k, "pw1x1 m%d k%d n%d act%d res%d" % (m, k, n, act, res), act)
