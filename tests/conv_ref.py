"""CPU references for the stem and fusion-deconv kernels (test infrastructure, numpy / torch CPU only).

  fma32        fmaf(x, w, c) for fp32 x, fp16 w and fp32 c, bit-exact: the product has at most 24 + 11 = 35 significant
               bits and is exact in float64; p + c is formed in float64 with its TwoSum error e (p + c = s + e exactly);
               s lies between two fp32 neighbours whose midpoint m is exact in float64, and the sign of (s - m) + e
               (s - m is exact, and a rounded sum keeps the sign of the exact one) picks the neighbour; zero is a tie
               and goes to the even one.  Rounding float64(p + c) straight to fp32 would double-round where s lands
               on a midpoint that p + c is not on.
  stem_conv    lp_stem_conv3x3_s2 (stem.cu) bit for bit: acc = fp32 bias, acc = fmaf(x, w, acc) over the taps in the
               order c, ky, kx with the weights widened from fp16, clamp to [0, 6] in fp32, one RNE rounding to fp16.
  stem_im2col  the A operand of the fused stem's first GEMM (stem_fused.cu P1): [M, 32], k = c*9 + ky*3 + kx for the
               27 taps of the fp16 image, then 5 zero columns.
  deconv_f64   ReLU(ConvT4x4s2p1(refined) + ConvT4x4s2p1(raw) + bias) in float64, with the same sum over magnitudes
               (fp16 subnormals lifted to 2^-14: the magnitude of the bound of gpu_util.check_bound).
  kernel selection of lp_fusion_deconv_f16 (gemm_tc.cu, deconv_rows.cu), restated from the sources."""
import numpy as np
import torch
import torch.nn.functional as F

from mma_emul import lift16

_F64, _F32, _F16 = np.float64, np.float32, np.float16


# ---------------------------------------------------------------- fp32 fused multiply-add
def fma32(x, w, c):
    """fmaf(x, w, c) with x fp32, w fp16 (or any value with <= 11 significant bits), c fp32 -> fp32, correctly rounded"""
    p = np.asarray(x, _F32).astype(_F64) * np.asarray(w, _F64)     # exact: <= 35 significant bits
    c = np.asarray(c, _F32).astype(_F64)
    s = p + c
    bb = s - p                                                     # TwoSum: p + c == s + e exactly
    e = (p - (s - bb)) + (c - bb)
    f = s.astype(_F32)
    exact = f.astype(_F64) == s                                    # s is an fp32 value: |e| is far below half its ulp
    up = f.astype(_F64) < s
    lo = np.where(up, f, np.nextafter(f, _F32(-np.inf)))
    hi = np.where(up, np.nextafter(f, _F32(np.inf)), f)
    m = (lo.astype(_F64) + hi.astype(_F64)) * 0.5                  # exact: 25 significant bits
    d = (s - m) + e
    even_hi = (hi.view(np.int32) & 1) == 0
    out = np.where(d > 0, hi, np.where(d < 0, lo, np.where(even_hi, hi, lo)))
    return np.where(exact, f, out).astype(_F32)


# ---------------------------------------------------------------- stem
def _image_nhwc_padded(x, flip):
    """[N,3,H,W] -> [N,H+2,W+2,3] with the one-pixel zero border, mirrored along W for the flip pass"""
    x = np.asarray(x)
    if flip:
        x = x[..., ::-1]
    n, c, h, w = x.shape
    xp = np.zeros((n, h + 2, w + 2, c), x.dtype)
    xp[:, 1:h + 1, 1:w + 1] = x.transpose(0, 2, 3, 1)
    return xp


def _taps(x, flip):
    """the 27 (c, ky, kx) input planes of the stride-2 3x3 stem, in that order, each [N, Ho, Wo]"""
    xp = _image_nhwc_padded(x, flip)
    ho, wo = (xp.shape[1] - 2) // 2, (xp.shape[2] - 2) // 2
    return [xp[:, ky:ky + 2 * ho:2, kx:kx + 2 * wo:2, c] for c in range(3) for ky in range(3) for kx in range(3)]


def stem_conv(x, w, bias, flip):
    """lp_stem_conv3x3_s2 bit for bit.  x [N,3,H,W] fp32 or fp16, w [32, 27] fp16, bias [32] fp32 -> [N,Ho,Wo,32] fp16"""
    fp32 = np.asarray(x).dtype == _F32
    taps = _taps(x, flip)
    w = np.asarray(w, _F16)
    n, ho, wo = taps[0].shape
    acc = np.broadcast_to(np.asarray(bias, _F32), (n, ho, wo, 32)).copy()
    for t, xs in enumerate(taps):
        xs = xs[..., None]
        if fp32:
            acc = fma32(xs, w[:, t], acc)
        else:       # an fp16 x fp16 product is exact in fp32: the fp32 add is fmaf's only rounding
            acc = xs.astype(_F32) * w[:, t].astype(_F32) + acc
    return np.minimum(np.maximum(acc, _F32(0)), _F32(6)).astype(_F16)


def stem_im2col(x16, flip):
    """[N,3,H,W] fp16 -> [N*Ho*Wo, 32] fp16: row = output pixel, k = c*9 + ky*3 + kx, columns 27..31 zero"""
    taps = _taps(np.asarray(x16, _F16), flip)
    a = np.zeros(taps[0].shape + (32,), _F16)
    for t, xs in enumerate(taps):
        a[..., t] = xs
    return a.reshape(-1, 32)


# ---------------------------------------------------------------- fusion deconv
def deconv_f64(xr, xw, wr, ww, bias):
    """xr [N,H,W,Cr], xw [N,H,W,Cw] NHWC; wr [Cr,Co,4,4], ww [Cw,Co,4,4]; bias [Co] -> (ref, mag), [N,2H,2W,Co] float64:
    ref = ReLU(ConvT(xr, wr) + ConvT(xw, ww) + bias), mag = ConvT(L(xr), L(wr)) + ConvT(L(xw), L(ww)) + |bias|,
    L = mma_emul.lift16"""
    def t(a):
        return torch.from_numpy(np.ascontiguousarray(np.asarray(a, _F64)))

    def nchw(a):
        return t(a).permute(0, 3, 1, 2)

    b = t(bias).view(1, -1, 1, 1)
    ref = F.conv_transpose2d(nchw(xr), t(wr), None, 2, 1) + F.conv_transpose2d(nchw(xw), t(ww), None, 2, 1) + b
    mag = (F.conv_transpose2d(t(lift16(xr)).permute(0, 3, 1, 2), t(lift16(wr)), None, 2, 1) +
           F.conv_transpose2d(t(lift16(xw)).permute(0, 3, 1, 2), t(lift16(ww)), None, 2, 1) + b.abs())
    return ref.clamp_min(0).permute(0, 2, 3, 1).numpy(), mag.permute(0, 2, 3, 1).numpy()


def deconv_subpixel(x, w):
    """ConvT4x4s2p1 without torch, in the kernels' sub-pixel form: output pixel (2y+a, 2x+b) sums input pixel
    (y+dy, x+dx) times kernel element (ki, kj) over dy in {0, a ? +1 : -1}, dx in {0, b ? +1 : -1},
    ki = 1 + a if dy == 0 else (0 if a else 3), kj likewise.  x [N,H,W,C], w [C,Co,4,4] -> [N,2H,2W,Co] float64"""
    x = np.asarray(x, _F64)
    w = np.asarray(w, _F64)
    n, h, wd, _ = x.shape
    xp = np.zeros((n, h + 2, wd + 2, x.shape[3]))
    xp[:, 1:h + 1, 1:wd + 1] = x
    out = np.zeros((n, 2 * h, 2 * wd, w.shape[1]))
    for a in (0, 1):
        for b in (0, 1):
            for dy in (0, 1 if a else -1):
                for dx in (0, 1 if b else -1):
                    ki = 1 + a if dy == 0 else (0 if a else 3)
                    kj = 1 + b if dx == 0 else (0 if b else 3)
                    src = xp[:, 1 + dy:1 + dy + h, 1 + dx:1 + dx + wd]
                    out[:, a::2, b::2] += src @ w[:, :, ki, kj]
    return out


def round16(v):
    return (v + 15) // 16 * 16


def rows_channels_ok(cr, cw, co):
    """deconv_rows_channels_ok: the row kernel holds all 16 weight sub-tiles and K = Cr + Cw <= 64 in one slot pixel;
    its shared memory (deconv_rows.cu dr_smem_bytes) fits the 227 KB limit up to Co = 32"""
    return cr % 8 == 0 and cw % 8 == 0 and co % 8 == 0 and cr + cw <= 64 and co <= 32


def uses_rows_kernel(cr, cw, co, w):
    """lp_fusion_deconv_f16 runs deconv_rows_kernel for these shapes, gemm_tc_kernel<MODE_DECONV> for all others"""
    return rows_channels_ok(cr, cw, co) and w >= 64


def tiled_packed_elems(cr, cw, co):
    """weights of the tiled kernel: per 64-channel K block of either branch, 9 taps x 16 (tap, phase) sub-tiles in all
    ((1 + 2 + 1)^2: a tap with dy = 0 serves two row phases, dy = +-1 one), each round16(Co) x 64"""
    kblocks = (cr + 63) // 64 + (cw + 63) // 64
    return 16 * kblocks * round16(co) * 64


def deconv_inputs(n, h, w, cr, cw, co, seed):
    """refined / raw NHWC fp16, weights [C, Co, 4, 4] fp16 (fan-in scaled), bias [Co] fp32.  Odd output channels get a
    bias ~8x the typical accumulator, so that their outputs are a large bias cancelled by the products: there an error
    in how the bias is added is not hidden by the magnitude term of the bound."""
    rng = np.random.default_rng(seed)
    xr = rng.standard_normal((n, h, w, cr)).astype(_F16)
    xw = rng.standard_normal((n, h, w, cw)).astype(_F16)
    wr = (rng.standard_normal((cr, co, 4, 4)) / cr ** 0.5).astype(_F16)
    ww = (rng.standard_normal((cw, co, 4, 4)) / cw ** 0.5).astype(_F16)
    bias = (rng.standard_normal(co) * np.where(np.arange(co) % 2 == 1, 8.0, 0.2)).astype(_F32)
    return xr, xw, wr, ww, bias


# (n, h, w, cr, cw, co): lp_fusion_deconv_f16 runs the row kernel on these ...
DECONV_ROWS_CASES = [
    (1, 3, 64, 16, 16, 16),       # W = 64 exactly: one 64-pixel strip; 3 rows, fewer items than SMs
    (1, 2, 200, 24, 16, 8),       # a partial last strip (128 + 72 pixels); Cr + Cw = 40: an odd chunk count (5)
    (2, 4, 96, 40, 24, 32),       # Cr + Cw = 64: k16 = 4; Co = 32, the widest the row kernel takes
    (1, 1, 128, 16, 8, 24),       # H = 1; Cr + Cw = 24 (3 chunks)
    (3, 5, 130, 32, 24, 16),      # Cr + Cw = 56 (7 chunks); a 2-pixel second strip
    (6, 40, 300, 8, 16, 8),       # 720 rows in 3 strips: each CTA's run crosses images and strips
    (8, 128, 128, 24, 16, 32),    # 1024 rows: long runs that cross images
]
# ... and the tiled gemm_tc kernel on these
DECONV_TILED_CASES = [
    (2, 12, 63, 16, 16, 16),      # W = 63: row-kernel channels one pixel below the switch; 32 x 4 tiles
    (1, 4, 32, 64, 32, 56),       # 32 x 4 tiles; Co = 56
    (2, 8, 16, 40, 24, 40),       # 16 x 8 tiles; Cr = 40: a K block with a half-filled last slice (k16 = 3); Co = 40
    (2, 16, 8, 24, 56, 48),       # 8 x 16 tiles; Cw = 56 (k16 = 4, 8 channels in the last slice); Co = 48
    (1, 20, 24, 72, 40, 64),      # Co = 64: all 16 accumulator chunks; Cr = 72: a second K block of 8 channels
    (2, 10, 12, 160, 96, 64),     # 5 K blocks (45 of the 48 steps): LitePose-L level 0, 160 + 96 -> 64
    (1, 16, 80, 80, 48, 16),      # W >= 64 but Cr + Cw > 64
    (1, 6, 100, 24, 16, 40),      # W >= 64 but Co > 32
]
PLAN_SIZES = [("XS", 448), ("S", 512), ("M", 512), ("L", 640)]


_plans = {}


def plan_ops(arch_name, size, n=1):
    """the launches of the engine's plan for one fp16 batch of n size x size images (built on the host, no device)"""
    key = (arch_name, size, n)
    if key not in _plans:
        from litepose_b200 import engine, synth
        from litepose_b200.config import get_arch, get_cfg
        from litepose_b200.lib.models.pose_mobilenet import get_pose_net
        arch = get_arch(arch_name)
        torch.manual_seed(0)
        model = synth.randomize_bn_(get_pose_net(get_cfg(input_size=size), False, arch), 1).eval()
        eng = engine.LitePoseEngine(model.state_dict(), arch, "cpu")
        _plans[key] = eng._build_plan(n, size, size, torch.float16, True, alloc=engine._Bump())["ops"]
    return _plans[key]


def plan_stem_shape(arch_name, size):
    """(n, h, w, C0) of the plan's fused stem launch"""
    ops = [op for op in plan_ops(arch_name, size) if op.name == "stem_fused"]
    assert len(ops) == 1, "%s@%d does not run the fused stem" % (arch_name, size)
    return tuple(ops[0].args[10:14])


def plan_deconv_shapes(arch_name, size):
    """(n, h, w, Cr, Cw, Co) of the plan's three fusion-deconv launches"""
    shapes = [tuple(op.args[5:11]) for op in plan_ops(arch_name, size) if op.name == "deconv"]
    assert len(shapes) == 3
    return shapes


def pick_spatial_tile(h, w):
    """gemm_tc.cu pick_spatial_tile: the 128-pixel tile (TW, TH) in {(32, 4), (16, 8), (8, 16)} that covers the map
    with the fewest padded pixels, the first (widest) on ties"""
    best = None
    for tw in (32, 16, 8):
        th = 128 // tw
        cover = ((w + tw - 1) // tw * tw) * ((h + th - 1) // th * th)
        if best is None or cover < best[0]:
            best = (cover, tw)
    return best[1]
