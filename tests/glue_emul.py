"""CPU restatement of the fused test-time glue, csrc/glue.cu, bit for bit (test infrastructure, numpy only).

glue(...) returns what lp_glue_f32 / lp_glue_scale_f32 write into det [N,J,Hd,Wd] and tag [N,Jt,Hd,Wd,T]; glue_path
restates glue_launch's choice among the four code paths, glue_f64 is the same operation in float64 (same fp32 source
coordinates and lambdas) and glue_bound the per-path distance between the two.

The arithmetic is the one the compiled kernels perform, read off the sm_90a build (nvcc 12.9, -O3, default
-fmad=true, no -ftz; `nvcc -ptx` for the contraction nvcc chose, `cuobjdump -sass` for what ptxas did to it):
  - Every two-term sum p*a + q*b becomes one rounded product and one FFMA: fma(p, a, fl(q*b)) ("first fused", F1)
    or fma(q, b, fl(p*a)) ("second fused", F2).  ptxas adds no contraction of its own: per kernel the SASS has as many
    FFMA (outside the division sequences) and FMUL as the PTX has fma.rn and mul, and as many FADD as add + sub.
  - glue_x4_kernel: up4 and proj4 are F1 everywhere (`FMUL R, b, 0.25 ; FFMA R, a, 0.75, R` etc.).  The block is
    built as in the source: the 3x3 quarter-resolution neighbourhood is up-sampled along x then y with the SOURCE
    index clamped (the mid rows / columns 2a-1 and 2a+2 of an edge block are extrapolated values, not copies of the
    edge), the half-resolution map is added and halved, and the projection runs along y (GL_PROJ's column pass) then
    along x.  `(x + y) / 2.f` is `FADD` + `FMUL 0.5`, except for the mid row 2a+2 of both heat maps, whose only use
    is `0.25f * m[3]` in proj4: ptxas folds the two multiplies into one `FMUL.D4 R, s, 0.5` (8 per thread).  The
    averaged det is `FADD` + `FMUL 0.5`.
  - glue_kernel, quad x2 branch (GL_Q): F1 everywhere, along x then y, on the shared mid-level tile.
  - glue_kernel, mid-level tile and unprojected branch (bilerp on global memory): the heat maps use F2 for both row
    lerps and F1 for the column lerp; the tags F1, F1, F1; except that the tile's plain-pass tag (s_t0) has F2 on its
    first row lerp.  The plain heat is `FADD` of o1 and the bilerp, then `FMUL 0.5`.
  - glue_kernel, generic projected branch (GL_P on the tile): ha F2, F2, F1; t0, hf and t1 F1, F1, F1.
  - lerp_coord: src = fma(scale, fl(dst + 0.5), -0.5) (`FFMA`), clamped at 0, truncated; l1 = src - i0 and
    l0 = 1 - l1 are `FADD`s; scale = H2 / Hd and h / H2 are IEEE divisions (div.rn.f32).
  - Epilogue of glue_kernel: (ha + hf) * 0.5, then `FADD` of the accumulated det, then an IEEE division by divide_by.
In the normal range the FMUL.D4 equals two multiplies; on fp32-subnormal results it rounds once where two multiplies
round twice, which D4_ROUNDS_ONCE states (measured, see tests/test_gpu_glue_exact.py).

Paths other than x4 differ from each other at the edges: the x4 and quad branches weight a clamped neighbour with the
constant 0.25 / 0.75 (0.25 s + 0.75 s), the bilerp weights it with the lambdas (1, 0), and all of them differ from
ATen's CUDA upsample_bilinear2d, whose 1 * s + 0 * s' is not 0.25 s + 0.75 s bit for bit (and differs for non-finite
neighbours).  That equality is not a goal here."""
from fractions import Fraction

import numpy as np

_F64, _F32 = np.float64, np.float32
U32 = 2.0 ** -24                       # unit roundoff of fp32
SUB_ULP = 2.0 ** -149                  # spacing of the fp32 subnormals

GL_TO, GL_TM = 64, 40                  # glue.cu: output tile side and mid-level tile limit
D4_ROUNDS_ONCE = True
"""FMUL.D4 R, s, 0.5 computes s * 0.5 / 4 with one rounding (measured on an H100 80GB HBM3: the subnormal input kind
of tests/test_gpu_glue_exact.py decides it; two roundings fail there)."""


# ---------------------------------------------------------------- exact fp32 FMA
def fma32(a, b, c):
    """fp32 fma(a, b, c) with one rounding.  a*b is exact in float64 (48 significant bits, exponent >= -298); the sum
    s = fl64(a*b + c) and its error e (TwoSum) give the exact value s + e; rounding s to odd when e != 0 keeps the
    sticky information, and float64 (53 bits) -> fp32 (24 bits) from a round-to-odd value is the correctly rounded
    result (Boldo and Melquiond, 2008), subnormal results included."""
    a, b, c = np.broadcast_arrays(*(np.asarray(x, _F32).astype(_F64) for x in (a, b, c)))
    p = a * b
    s = p + c
    bp = s - c
    e = (p - bp) + (c - (s - bp))
    odd = (np.atleast_1d(s).view(np.int64) & 1).reshape(s.shape) == 1
    fix = (e != 0) & ~odd
    if np.any(fix):
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(_F32)


def fma32_exact(a, b, c):
    """one fp32 fma through fractions.Fraction: the exact value, rounded to nearest even into fp32 (the self-test's
    reference; shares no code with fma32)"""
    a, b, c = (_F32(x) for x in (a, b, c))
    v = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if v == 0:
        z = float(a) * float(b) + float(c)      # sign of an exact zero as IEEE gives it
        return _F32(z)
    return round_fraction32(v)


def round_fraction32(v):
    """exact rational -> fp32, round to nearest even (finite results only)"""
    neg = v < 0
    m = -v if neg else v
    e = m.numerator.bit_length() - m.denominator.bit_length()
    if Fraction(2) ** e > m:
        e -= 1
    q = max(e, -126) - 23                            # exponent of one ulp at m (subnormal spacing below 2^-126)
    t = m / Fraction(2) ** q
    n = t.numerator // t.denominator
    r = t - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    out = _F32(float(Fraction(n) * Fraction(2) ** q))
    return -out if neg else out


def mul32(a, b):
    return (np.asarray(a, _F32) * np.asarray(b, _F32)).astype(_F32)


def add32(a, b):
    return (np.asarray(a, _F32) + np.asarray(b, _F32)).astype(_F32)


def d4(s):
    """FMUL.D4 R, s, 0.5: s * 0.5 / 4"""
    s = np.asarray(s, _F32)
    if D4_ROUNDS_ONCE:
        return (s.astype(_F64) * 0.125).astype(_F32)     # exact in float64, one rounding
    return mul32(mul32(s, 0.5), 0.25)


def lin2(p, a, q, b, fuse):
    """p*a + q*b as compiled: fuse 1 = fma(p, a, fl(q*b)), fuse 2 = fma(q, b, fl(p*a))"""
    if fuse == 1:
        return fma32(p, a, mul32(q, b))
    return fma32(q, b, mul32(p, a))


# ---------------------------------------------------------------- which kernel path (glue_launch)
def glue_tile_side(h, w, Hd, Wd):
    to = GL_TO
    while to >= 8:
        if (2 * h) / Hd * to + 3 <= GL_TM and (2 * w) / Wd * to + 3 <= GL_TM:
            return to
        to >>= 1
    return 0


def glue_path(N, J, h, w, Hd, Wd, flip=True, Jm=None, tag_shared=False, accumulate=False, divide_by=1.0,
              has_tag=True, entry="scale", j=0):
    """The branch joint ``j`` of one glue call runs: "x4" (glue_x4_kernel), "quad" (glue_kernel's constant-weight x2
    branch), "generic" (glue_kernel, any other projection) or "unprojected" (Hd, Wd == 2h, 2w).  ``entry`` "f32" is
    lp_glue_f32 (x4 always allowed), "scale" lp_glue_scale_f32 (x4 only for a plain call).  Raises ValueError where
    glue_launch refuses the projection.  With a shared tag map only the j == 0 blocks write tags, so only they are
    "plain": the other joints take the generic branch for the same call."""
    Jm = J if Jm is None else Jm
    allow_x4 = True if entry == "f32" else (not accumulate and divide_by == 1.0 and has_tag)
    allow_x4 = allow_x4 and Jm == J and not tag_shared
    project = not (Hd == 2 * h and Wd == 2 * w)
    if project and glue_tile_side(h, w, Hd, Wd) == 0:
        raise ValueError("projection %dx%d -> %dx%d shrinks by more than 4.6x" % (2 * h, 2 * w, Hd, Wd))
    if allow_x4 and flip and Hd == 4 * h and Wd == 4 * w and N * J <= 65535 and h <= 65535:
        return "x4"
    if not project:
        return "unprojected"
    tag_here = has_tag and not (tag_shared and j != 0)
    plain = not accumulate and divide_by == 1.0 and tag_here
    if Hd == 4 * h and Wd == 4 * w and flip and plain:
        return "quad"
    return "generic"


# ---------------------------------------------------------------- lerp_coord, bilerp
def lerp_coord(n_out, scale, n_in):
    """i0, i1, l0, l1 for dst = 0 .. n_out-1 (fp32 lambdas, as the kernel computes them)"""
    dst = np.arange(n_out).astype(_F32)
    src = fma32(_F32(scale), add32(dst, 0.5), _F32(-0.5))
    src = np.where(src < 0, _F32(0), src).astype(_F32)
    i0 = np.minimum(src.astype(np.int64), n_in - 1)
    i1 = i0 + (i0 < n_in - 1)
    l1 = (src - i0.astype(_F32)).astype(_F32)
    l0 = (_F32(1) - l1).astype(_F32)
    return i0, i1, l0, l1


def _scale(a, b):
    return _F32(_F32(a) / _F32(b))


def bilerp(p, ly, lx, fuse):
    """bilerp over the last two axes of p at the rows ly and columns lx (lerp_coord tuples): the row lerps with
    fuse[0] / fuse[1], the column lerp with fuse[2]"""
    y0, y1, yl0, yl1 = ly
    x0, x1, xl0, xl1 = lx
    g = lambda yy, xx: p[..., yy[:, None], xx[None, :]]
    r0 = lin2(xl0[None, :], g(y0, x0), xl1[None, :], g(y0, x1), fuse[0])
    r1 = lin2(xl0[None, :], g(y1, x0), xl1[None, :], g(y1, x1), fuse[1])
    return lin2(yl0[:, None], r0, yl1[:, None], r1, fuse[2])


HEAT, TAG, TILE_T0 = (2, 2, 1), (1, 1, 1), (2, 1, 1)


def _split(o0, o1, f0, f1, fidx, J, Jm, tag_shared):
    """the per-joint planes of one call: heat / tag of the plain and mirrored pass, o1 / f1 planes"""
    t_idx = [Jm] * J if tag_shared else [Jm + j for j in range(J)]
    a = (o0[:, :J], o0[:, t_idx], o1[:, :J])
    b = None
    if f0 is not None:
        fj = list(fidx)
        tf = [Jm] * J if tag_shared else [Jm + k for k in fj]
        b = (f0[:, fj], f0[:, tf], f1[:, fj])
    return a, b


def _mid_maps(a, b, h, w, tile):
    """glue_kernel's mid-level maps [N,J,2h,2w]: ha, t0, hf, t1 (hf / t1 mirrored), as the tile fill (tile=True) or the
    unprojected branch computes them"""
    H2, W2 = 2 * h, 2 * w
    ly, lx = lerp_coord(H2, _scale(h, H2), h), lerp_coord(W2, _scale(w, W2), w)
    ha = mul32(add32(a[2], bilerp(a[0], ly, lx, HEAT)), 0.5)
    t0 = bilerp(a[1], ly, lx, TILE_T0 if tile else TAG)
    hf = t1 = None
    if b is not None:
        hf = mul32(add32(b[2], bilerp(b[0], ly, lx, HEAT)), 0.5)[..., ::-1]
        t1 = bilerp(b[1], ly, lx, TAG)[..., ::-1]
    return ha, t0, hf, t1


def _up2_first(x, axis):
    """x2 up-sample along ``axis`` with constant weights and clamped neighbours, F1: out[2m] = .25 x[m-1] + .75 x[m],
    out[2m+1] = .75 x[m] + .25 x[m+1]"""
    axis %= x.ndim
    n = x.shape[axis]
    idx = np.arange(n)
    t = lambda i: np.take(x, np.clip(i, 0, n - 1), axis=axis)
    ev = lin2(0.25, t(idx - 1), 0.75, t(idx), 1)
    od = lin2(0.75, t(idx), 0.25, t(idx + 1), 1)
    out = np.stack([ev, od], axis=axis + 1)
    shp = list(x.shape)
    shp[axis] = 2 * n
    return out.reshape(shp)


def _up2_ext(q, axis):
    """glue_x4_kernel's up4: the mid samples -1 .. 2n of a x2 up-sample along ``axis`` with the quarter-resolution
    index clamped (2n + 2 samples, F1)"""
    n = q.shape[axis]
    t = lambda i: np.take(q, np.clip(i, 0, n - 1), axis=axis)
    m = np.arange(-1, 2 * n + 1)
    i = m // 2                                          # m = 2i: .25 q[i-1] + .75 q[i];  m = 2i+1: .75 q[i] + .25 q[i+1]
    ev = lin2(0.25, t(i - 1), 0.75, t(i), 1)
    od = lin2(0.75, t(i), 0.25, t(i + 1), 1)
    sel = (m % 2 == 0).reshape([-1 if k == axis % q.ndim else 1 for k in range(q.ndim)])
    return np.where(sel, ev, od).astype(_F32)


def _proj4(m, axis, heat):
    """proj4 along ``axis`` of an extended mid array (samples -1 .. 2n): outputs 0 .. 4n-1.  ``heat``: m holds the
    sums s = up + o1 and the halving is applied here, with the FMUL.D4 on the 0.25 * m[3] term of every block"""
    axis %= m.ndim
    n2 = m.shape[axis] - 2
    mm = mul32(m, 0.5) if heat else m
    t = lambda k: np.take(mm, k + 1, axis=axis)          # mid sample k (k >= -1)
    k = np.arange(n2)                                     # out[2k] from k-1, k; out[2k+1] from k, k+1
    ev = lin2(0.25, t(k - 1), 0.75, t(k), 1)
    nxt = np.take(m, k + 2, axis=axis)
    q = mul32(t(k + 1), 0.25)
    if heat:
        blk3 = (k % 2 == 1).reshape([-1 if a == axis % m.ndim else 1 for a in range(m.ndim)])
        q = np.where(blk3, d4(nxt), q).astype(_F32)      # out[4i+3] = .75 m[2i+1] + .25 m[2i+2]
    od = fma32(0.75, t(k), q)
    out = np.stack([ev, od], axis=axis + 1)
    shp = list(m.shape)
    shp[axis] = 2 * n2
    return out.reshape(shp)


def _x4(a, b, h, w):
    """glue_x4_kernel: det [N,J,4h,4w], t0, t1"""
    H2, W2 = 2 * h, 2 * w
    ry, rx = np.clip(np.arange(-1, H2 + 1), 0, H2 - 1), np.clip(np.arange(-1, W2 + 1), 0, W2 - 1)

    def mids(p):
        return _up2_ext(_up2_ext(p, -1), -2)              # along x (each row), then along y

    o1a = a[2][..., ry[:, None], rx[None, :]]
    sa = add32(mids(a[0]), o1a)                           # (up + o1), halved inside _proj4
    o1b = b[2][..., ry[:, None], rx[None, :]]
    sb = add32(mids(b[0]), o1b)[..., ::-1]                # mirrored block, columns reversed
    ta, tb = mids(a[1]), mids(b[1])[..., ::-1]
    proj = lambda m, heat: _proj4(_proj4(m, -2, heat), -1, False)    # rows (GL_PROJ's column pass), then columns
    pa, pf = proj(sa, True), proj(sb, True)
    return mul32(add32(pa, pf), 0.5), proj(ta, False), proj(tb, False)


def _quad(ha, t0, hf, t1):
    up = lambda s: _up2_first(_up2_first(s, -1), -2)      # GL_Q: along x, then y
    return mul32(add32(up(ha), up(hf)), 0.5), up(t0), up(t1)


def _generic(ha, t0, hf, t1, h, w, Hd, Wd):
    H2, W2 = 2 * h, 2 * w
    ly, lx = lerp_coord(Hd, _scale(H2, Hd), H2), lerp_coord(Wd, _scale(W2, Wd), W2)
    pa, p0 = bilerp(ha, ly, lx, HEAT), bilerp(t0, ly, lx, TAG)
    if hf is None:
        return pa, p0, None, None
    return pa, p0, bilerp(hf, ly, lx, TAG), bilerp(t1, ly, lx, TAG)


def glue(o0, o1, f0, f1, fidx, J, Hd, Wd, Jm=None, tag_shared=False, accumulate=False, divide_by=1.0,
         det=None, tag=None, write_tag=True, entry="scale"):
    """One glue call as the kernels compute it.  o0 [N,C0,h,w] with C0 = 2Jm (or Jm + 1 with a shared tag map),
    o1 [N,Jm,2h,2w], f0 / f1 the mirrored pass (None without flip), fidx the flip index.  ``det`` is the array the
    call writes (and, with accumulate, reads), ``tag`` the tag array; they are updated in place as the kernels would
    and returned, and made NaN-filled when not given.  write_tag=False is a call with tag == NULL."""
    o0, o1 = np.asarray(o0, _F32), np.asarray(o1, _F32)
    flip = f0 is not None
    N, _, h, w = o0.shape
    Jm = J if Jm is None else Jm
    if det is None:
        det = np.full((N, J, Hd, Wd), np.nan, _F32)
    if tag is None and write_tag:
        tag = np.full((N, 1 if tag_shared else J, Hd, Wd, 2 if flip else 1), np.nan, _F32)
    a, b = _split(o0, o1, np.asarray(f0, _F32) if flip else None, np.asarray(f1, _F32) if flip else None,
                  fidx, J, Jm, tag_shared)
    paths = [glue_path(N, J, h, w, Hd, Wd, flip, Jm, tag_shared, accumulate, divide_by, write_tag, entry, j)
             for j in range(J)]
    for path in sorted(set(paths)):
        js = np.array([j for j in range(J) if paths[j] == path])
        aj = tuple(x[:, js] for x in a)
        bj = tuple(x[:, js] for x in b) if flip else None
        if path == "x4":
            d, t0, t1 = _x4(aj, bj, h, w)
        elif path == "quad":
            d, t0, t1 = _quad(*_mid_maps(aj, bj, h, w, tile=True))
        else:
            ha, t0, hf, t1 = _mid_maps(aj, bj, h, w, tile=path != "unprojected")
            if path == "generic":
                ha, t0, hf, t1 = _generic(ha, t0, hf, t1, h, w, Hd, Wd)
            d = mul32(add32(ha, hf), 0.5) if flip else ha
            if accumulate:
                d = add32(det[:, js], d)
            if divide_by != 1.0:
                d = (d / _F32(divide_by)).astype(_F32)
        det[:, js] = d
        if write_tag:
            tv = np.stack([t0, t1], -1) if flip else t0[..., None]
            if not tag_shared:
                tag[:, js] = tv
            elif js[0] == 0:                              # a shared map is written by the j == 0 blocks only
                tag[:, 0] = tv[:, 0]
    return det, tag


# ---------------------------------------------------------------- float64 twin and the per-path bound
ROUNDINGS = {
    # fp32 roundings on the longest chain of each path: (det, tag)
    "x4": (12, 8),            # up x 2 + up y 2, + o1, * 0.5, proj y 2, proj x 2, + (flip), * 0.5
    "quad": (12, 8),          # bilerp 4, + o1, * 0.5, GL_Q 4, +, * 0.5
    "generic": (14, 8),       # bilerp 4, + o1, * 0.5, GL_P 4, +, * 0.5, + accumulated, / divide_by
    "unprojected": (10, 4),   # bilerp 4, + o1, * 0.5, +, * 0.5, + accumulated, / divide_by
}


def _bil64(p, ly, lx):
    y0, y1, yl0, yl1 = ly
    x0, x1, xl0, xl1 = lx
    g = lambda yy, xx: p[..., yy[:, None], xx[None, :]]
    xl0, xl1 = xl0.astype(_F64)[None, :], xl1.astype(_F64)[None, :]
    r0 = xl0 * g(y0, x0) + xl1 * g(y0, x1)
    r1 = xl0 * g(y1, x0) + xl1 * g(y1, x1)
    return yl0.astype(_F64)[:, None] * r0 + yl1.astype(_F64)[:, None] * r1


def _up2_64(x, axis, ext):
    n = x.shape[axis]
    t = lambda i: np.take(x, np.clip(i, 0, n - 1), axis=axis)
    m = np.arange(-1, 2 * n + 1) if ext else np.arange(2 * n)
    i = m // 2
    ev = 0.25 * t(i - 1) + 0.75 * t(i)
    od = 0.75 * t(i) + 0.25 * t(i + 1)
    sel = (m % 2 == 0).reshape([-1 if k == axis % x.ndim else 1 for k in range(x.ndim)])
    return np.where(sel, ev, od)


def _proj4_64(m, axis):
    axis %= m.ndim
    n2 = m.shape[axis] - 2
    t = lambda k: np.take(m, k + 1, axis=axis)
    k = np.arange(n2)
    ev = 0.25 * t(k - 1) + 0.75 * t(k)
    od = 0.75 * t(k) + 0.25 * t(k + 1)
    out = np.stack([ev, od], axis=axis + 1)
    shp = list(m.shape)
    shp[axis] = 2 * n2
    return out.reshape(shp)


def glue_f64(o0, o1, f0, f1, fidx, J, Hd, Wd, Jm=None, tag_shared=False, accumulate=False, divide_by=1.0,
             det_in=None, entry="scale", has_tag=True):
    """The operation of glue() in float64: the same source indices, constant weights and fp32 lambdas per path, every
    product and sum in float64.  Returns det [N,J,Hd,Wd] and the tag planes [N,J,Hd,Wd,T] per joint (the shared map
    repeated), both float64."""
    o0, o1 = np.asarray(o0, _F64), np.asarray(o1, _F64)
    flip = f0 is not None
    N, _, h, w = o0.shape
    H2, W2 = 2 * h, 2 * w
    Jm = J if Jm is None else Jm
    a, b = _split(o0, o1, None if not flip else np.asarray(f0, _F64), None if not flip else np.asarray(f1, _F64),
                  fidx, J, Jm, tag_shared)
    det = np.zeros((N, J, Hd, Wd), _F64)
    tag = np.zeros((N, J, Hd, Wd, 2 if flip else 1), _F64)
    for j in range(J):
        path = glue_path(N, J, h, w, Hd, Wd, flip, Jm, tag_shared, accumulate, divide_by, has_tag, entry, j)
        aj = tuple(x[:, j] for x in a)
        bj = tuple(x[:, j] for x in b) if flip else None
        if path == "x4":
            ry, rx = np.clip(np.arange(-1, H2 + 1), 0, H2 - 1), np.clip(np.arange(-1, W2 + 1), 0, W2 - 1)
            mids = lambda p: _up2_64(_up2_64(p, -1, True), -2, True)
            sa = (mids(aj[0]) + aj[2][..., ry[:, None], rx[None, :]]) * 0.5
            sb = ((mids(bj[0]) + bj[2][..., ry[:, None], rx[None, :]]) * 0.5)[..., ::-1]
            proj = lambda m: _proj4_64(_proj4_64(m, -2), -1)
            det[:, j] = (proj(sa) + proj(sb)) * 0.5
            tag[:, j] = np.stack([proj(mids(aj[1])), proj(mids(bj[1])[..., ::-1])], -1)
            continue
        ly, lx = lerp_coord(H2, _scale(h, H2), h), lerp_coord(W2, _scale(w, W2), w)
        ha, t0 = (_bil64(aj[0], ly, lx) + aj[2]) * 0.5, _bil64(aj[1], ly, lx)
        hf = t1 = None
        if flip:
            hf, t1 = ((_bil64(bj[0], ly, lx) + bj[2]) * 0.5)[..., ::-1], _bil64(bj[1], ly, lx)[..., ::-1]
        if path == "quad":
            up = lambda s: _up2_64(_up2_64(s, -1, False), -2, False)
            det[:, j] = (up(ha) + up(hf)) * 0.5
            tag[:, j] = np.stack([up(t0), up(t1)], -1)
            continue
        if path == "generic":
            py, px = lerp_coord(Hd, _scale(H2, Hd), H2), lerp_coord(Wd, _scale(W2, Wd), W2)
            ha, t0 = _bil64(ha, py, px), _bil64(t0, py, px)
            if flip:
                hf, t1 = _bil64(hf, py, px), _bil64(t1, py, px)
        v = (ha + hf) * 0.5 if flip else ha
        if accumulate:
            v = np.asarray(det_in, _F64)[:, j] + v
        det[:, j] = v / float(_F32(divide_by))
        tag[:, j] = np.stack([t0, t1], -1) if flip else t0[..., None]
    return det, tag


def glue_bound(o0, o1, f0, f1, fidx, J, Hd, Wd, det_in=None, **kw):
    """Per output: k * 2^-24 * sum|terms| + k * 2^-149 with k the roundings of the output's path (ROUNDINGS) and
    sum|terms| the float64 glue of the absolute values (every weight is >= 0).  Returns (det_bound, tag_bound)."""
    ab = lambda x: None if x is None else np.abs(np.asarray(x, _F64))
    d, t = glue_f64(ab(o0), ab(o1), ab(f0), ab(f1), fidx, J, Hd, Wd, det_in=ab(det_in), **kw)
    N, _, h, w = np.shape(o0)
    kd = np.zeros(J)
    kt = np.zeros(J)
    for j in range(J):
        p = glue_path(N, J, h, w, Hd, Wd, f0 is not None, kw.get("Jm"), kw.get("tag_shared", False),
                      kw.get("accumulate", False), kw.get("divide_by", 1.0), kw.get("has_tag", True),
                      kw.get("entry", "scale"), j)
        kd[j], kt[j] = ROUNDINGS[p]
    kd, kt = kd[None, :, None, None], kt[None, :, None, None, None]
    return kd * (1 + 1e-6) * U32 * d + kd * SUB_ULP, kt * (1 + 1e-6) * U32 * t + kt * SUB_ULP


# ---------------------------------------------------------------- the cases the GPU test runs (shared with the CPU test)
def multiscale_calls(scales, proj, hw):
    """the calls of one multi-scale step (valid.py:205-225 as LitePosePipeline.step_multiscale launches it): per scale,
    largest first, (h, w, accumulate, divide_by, write_tag); returns (calls, Hd, Wd).  Image sides as
    test_gpu_parser.test_glue_multiscale_ratios_vs_oracle builds them (multiples of 64, scale 1 exactly hw)."""
    sides = {s: (hw[0], hw[1]) if s == 1 else (int(round(hw[0] * s / 64)) * 64, int(round(hw[1] * s / 64)) * 64)
             for s in scales}
    order = sorted(scales, reverse=True)
    calls = [(sides[s][0] // 4, sides[s][1] // 4, i > 0, float(len(order)) if i == len(order) - 1 else 1.0, s == 1)
             for i, s in enumerate(order)]
    Hd, Wd = (hw[0], hw[1]) if proj else (sides[order[0]][0] // 2, sides[order[0]][1] // 2)
    return calls, Hd, Wd


def _case(name, N, J, h, w, Hd, Wd, flip=True, Jm=None, tag_shared=False, entry="f32", calls=None):
    return dict(name=name, N=N, J=J, Jm=J if Jm is None else Jm, tag_shared=tag_shared, Hd=Hd, Wd=Wd, flip=flip,
                entry=entry, calls=calls or [(h, w, False, 1.0, True)])


def _ms(name, scales, proj, hw, N=2):
    calls, Hd, Wd = multiscale_calls(scales, proj, hw)
    return _case(name, N, 14, 0, 0, Hd, Wd, entry="scale", calls=calls)


CASES = [
    # x4: the evaluation config (flip + PROJECT2IMAGE to 4h x 4w)
    _case("x4_16", 2, 14, 16, 16, 64, 64),
    _case("x4_bench", 1, 14, 128, 128, 512, 512),                  # the bench's per-image shape
    _case("x4_7x129", 3, 14, 7, 129, 28, 516),                     # a partial 128-wide block
    _case("x4_1x1_j17", 2, 17, 1, 1, 4, 4),
    _case("x4_1x300", 1, 14, 1, 300, 4, 1200),
    _case("x4_33x5", 1, 14, 33, 5, 132, 20),
    # quad: x4 not allowed
    _case("quad_nj_over_65535", 4682, 14, 1, 1, 4, 4),             # N * J > 65535
    _case("quad_center_ignored", 2, 14, 16, 12, 64, 48, Jm=15, entry="scale"),
    _case("quad_shared_tag", 2, 14, 16, 12, 64, 48, tag_shared=True, entry="scale"),   # joints 1.. take generic
    # generic projection
    _case("generic_shared_tag_noflip", 2, 14, 8, 8, 32, 32, flip=False, tag_shared=True, entry="scale"),   # no flip
    _case("generic_no_tag", 2, 14, 8, 12, 32, 48, entry="scale", calls=[(8, 12, False, 1.0, False)]),   # tag NULL
    _case("generic_61x93", 2, 14, 16, 24, 61, 93),
    _case("generic_noflip_x4", 2, 14, 16, 16, 64, 64, flip=False),
    _case("generic_shrink_4p6", 1, 14, 370, 370, 160, 161),        # just inside glue_tile_side's limit, both axes
    _ms("ms_075_1_125", [0.75, 1, 1.25], True, (192, 256)),
    _ms("ms_1_15_25", [1, 1.5, 2.5], True, (128, 128)),
    _ms("ms_05_1_2_noproj", [0.5, 1, 2], False, (128, 192)),
    _ms("ms_1_2", [1, 2], True, (64, 64)),
    # unprojected
    _case("unproj_flip", 2, 14, 16, 24, 32, 48),
    _case("unproj_noflip", 2, 14, 16, 24, 32, 48, flip=False),
    _case("unproj_shared_tag", 2, 14, 9, 11, 18, 22, tag_shared=True, Jm=15, entry="scale"),
]

KINDS = ("randn", "heat", "wide", "midpoint")


def flip_index(J):
    """a permutation for the mirrored pass: the CrowdPose one for 14 joints, else reversed pairs"""
    if J == 14:
        return [1, 0, 3, 2, 5, 4, 7, 6, 9, 8, 11, 10, 12, 13]
    return list(range(J))[::-1]


def make_input(kind, shape, rng):
    """fp32 arrays of one input kind: randn; heat (non-negative, heat-map-like); wide (+-2^-140 .. 2^60 with fp32
    subnormals and -0.0); midpoint (+-[1, 2) at full precision: 0.75 x and the pair sums land on fp32 midpoints)"""
    if kind == "randn":
        return rng.standard_normal(shape).astype(_F32)
    if kind == "heat":
        return (rng.random(shape) ** 4).astype(_F32)
    if kind == "wide":
        e = rng.uniform(-140, 60, shape)
        x = (np.sign(rng.standard_normal(shape)) * np.exp2(e) * rng.uniform(1, 2, shape)).astype(_F32)
        x[rng.random(shape) < 0.03] = _F32(-0.0)
        return x
    if kind == "midpoint":
        k = rng.integers(0, 2 ** 23, shape)
        return (np.where(rng.random(shape) < 0.5, -1, 1) * (1 + k * 2.0 ** -23)).astype(_F32)
    raise ValueError(kind)


def case_inputs(case, kind, seed):
    """per call: o0, o1, f0, f1 (f0 / f1 None without flip)"""
    rng = np.random.default_rng(seed)
    N, Jm = case["N"], case["Jm"]
    C0 = Jm + 1 if case["tag_shared"] else 2 * Jm
    out = []
    for h, w, _, _, _ in case["calls"]:
        o = [make_input(kind, (N, C0, h, w), rng), make_input(kind, (N, Jm, 2 * h, 2 * w), rng)]
        f = [make_input(kind, (N, C0, h, w), rng), make_input(kind, (N, Jm, 2 * h, 2 * w), rng)] if case["flip"] \
            else [None, None]
        out.append(o + f)
    return out


def run_case(case, inputs):
    """the emulated det / tag after every call of the case"""
    det = tag = None
    J, fidx = case["J"], flip_index(case["J"])
    for (h, w, acc, div, wt), (o0, o1, f0, f1) in zip(case["calls"], inputs):
        if tag is None and wt:
            tag = np.full((o0.shape[0], 1 if case["tag_shared"] else J, case["Hd"], case["Wd"],
                           2 if case["flip"] else 1), np.nan, _F32)
        det, _ = glue(o0, o1, f0, f1, fidx, J, case["Hd"], case["Wd"], Jm=case["Jm"], tag_shared=case["tag_shared"],
                      accumulate=acc, divide_by=div, det=det, tag=tag if wt else None, write_tag=wt,
                      entry=case["entry"])
    return det, tag


def case_paths(case):
    """the set of branches the case's calls take (over all joints)"""
    out = set()
    for h, w, acc, div, wt in case["calls"]:
        for j in range(case["J"]):
            out.add(glue_path(case["N"], case["J"], h, w, case["Hd"], case["Wd"], case["flip"], case["Jm"],
                              case["tag_shared"], acc, div, wt, case["entry"], j))
    return out
