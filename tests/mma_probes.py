"""Probe operands that measure the tensor cores' fp16 -> fp32 accumulation through lp_head_pw_dual_f16 (test
infrastructure, numpy only).

The head GEMM with C1 = C2 = 16 and fp32 output stores, for every pixel p and output channel c,
    out[p, c] = mma(mma(+0, a1[p], w1[c]), a2[p], w2[c])
with one wgmma K = 16 step per source: the first starts from an accumulator of +0, the second carries the first's
result as its addend.  A probe is one activation row [a1 | a2] (32 fp16 values); every probe row is reduced against
every row of PROBE_WEIGHTS, so each row is measured at 16 product scales and signs.  Each group of rows decides one
parameter of the model in mma_emul (the row names say which)."""
import numpy as np

_F16 = np.float16


def _w_rows():
    """[16, 32] fp16: uniform rows of scale 1, 2^-12, 2^12, -1, 2^-24 (a subnormal), 1 + 2^-10 and 3, an alternating
    +-1 row, and eight random normal rows"""
    rng = np.random.default_rng(7)
    rows = [np.full(32, v) for v in (1.0, 2.0 ** -12, 2.0 ** 12, -1.0, 2.0 ** -24, 1.0 + 2.0 ** -10, 3.0)]
    rows.append(np.where(np.arange(32) % 2 == 0, 1.0, -1.0))
    for _ in range(8):
        rows.append(rng.standard_normal(32) * 2.0 ** rng.integers(-6, 4))
    return np.stack(rows).astype(_F16)


PROBE_WEIGHTS = _w_rows()


def probe_rows():
    """(names [P], a [P, 32] fp16): the named probe rows, [a1 | a2]"""
    names, rows = [], []

    def add(name, first=(), second=()):
        r = np.zeros(32)
        for i, v in first:
            r[i] = v
        for i, v in second:
            r[16 + i] = v
        rows.append(r)
        names.append(name)

    big = 2.0 ** 15
    for j in range(1, 40):
        s = big * 2.0 ** -j
        if s < 2.0 ** -24:
            break
        # F and how aligned terms lose bits: a small term next to a large one, with and without the large one cancelled
        for sg in (1, -1):
            add("F_pair j=%d sg=%d" % (j, sg), [(0, 1.0), (1, sg * 2.0 ** -j)] if j <= 24 else [(0, big), (1, sg * s)])
            add("F_pair_neg j=%d sg=%d" % (j, sg), [(0, -1.0), (5, sg * 2.0 ** -j)] if j <= 24 else [(0, -big), (5, sg * s)])
            add("F_cancel j=%d sg=%d" % (j, sg), [(0, big), (1, -big), (2, sg * s)])
            add("F_cancel_late j=%d sg=%d" % (j, sg), [(3, sg * s), (14, big), (15, -big)])
            # c in the alignment: the second step's products cancel, the first step's small result is its addend
            add("c_align_cancel j=%d sg=%d" % (j, sg), [(0, sg * s)], [(0, big), (1, -big)])
            # c in the alignment: a large c against small products of the second step
            add("c_align_small j=%d sg=%d" % (j, sg), [(0, big)], [(0, sg * s), (7, sg * s)])
        # final rounding: 1 + (1 + 2^-10) 2^-j lands between fp32 neighbours for j >= 14
        if big * 2.0 ** -j * (1 + 2.0 ** -10) >= 2.0 ** -14:
            for sg in (1, -1):
                add("round j=%d sg=%d" % (j, sg), [(0, big), (1, sg * big * (1 + 2.0 ** -10) * 2.0 ** -j)])
                add("round_c j=%d sg=%d" % (j, sg), [(0, big)], [(1, sg * big * (1 + 2.0 ** -10) * 2.0 ** -j)])
    # B: +L at i, -L at j, small terms everywhere else; which small terms survive depends on the blocks i and j fall in
    for big_, small in ((2.0 ** 10, 2.0 ** -20), (2.0 ** 15, 2.0 ** -23), (2.0 ** 2, 2.0 ** -22)):
        for i in range(16):
            for j in range(16):
                if i != j:
                    add("B i=%d j=%d L=%g" % (i, j, big_),
                        [(t, big_ if t == i else (-big_ if t == j else small)) for t in range(16)])
    # B: a large term at i and a small one at j, nothing else
    for i in range(16):
        for j in range(16):
            if i != j:
                add("B_pair i=%d j=%d" % (i, j), [(i, 1.0), (j, -2.0 ** -20)], [(0, -1.0)])
    # the exponent a product brings to E: significands multiplying to >= 2 (1.5 * 1.5, 1.75 * 1.5 against the weight
    # row of 3s) next to a term one bit below 2^(ea + eb - 24); a subnormal weight (2^-24, exponent read as -14)
    for m in (1, 3, 5, 7):
        add("lead_carry 1.5 m=%d" % m, [(0, 1.5), (1, -1.5), (2, m * 2.0 ** -24)])
        add("lead_carry 1.75 m=%d" % m, [(0, 1.75), (3, -1.75), (9, m * 2.0 ** -24)])
    for j in range(14, 20):
        add("lead_sub j=%d" % j, [(0, big), (1, -big), (2, big * 2.0 ** -j)])
    # the sign of zero
    add("zero 1-1", [(0, 1.0), (1, -1.0)])
    add("zero 1-1 both", [(0, 1.0), (1, -1.0)], [(0, 1.0), (1, -1.0)])
    add("zero -0 products", [(t, -0.0) for t in range(16)], [(t, -0.0) for t in range(16)])
    add("zero +0 products")
    add("zero -tiny lost", [(0, big), (1, -big), (2, -2.0 ** -24)])
    add("zero -tiny lost c", [(0, -2.0 ** -24)], [(0, big), (1, -big)])
    add("zero 1-1 then -0", [(0, 1.0), (1, -1.0)], [(t, -0.0) for t in range(16)])
    # fp16 subnormal operands
    for m in (1, 3, 511, 1023):
        sub = m * 2.0 ** -24
        add("subnormal m=%d" % m, [(0, sub)])
        add("subnormal_sum m=%d" % m, [(t, sub) for t in range(16)], [(t, -sub) for t in range(0, 16, 3)])
        add("subnormal_big m=%d" % m, [(0, 1.0), (1, sub)], [(0, sub), (1, -1.0)])
        add("subnormal_c m=%d" % m, [(0, sub)], [(0, 2.0 ** -14), (1, -2.0 ** -14)])
    return names, np.stack(rows).astype(_F16)


def fuzz_rows(p, k, seed):
    """[p, k] fp16 random rows in four kinds (a quarter each): randn; wide exponents (2^-24 .. 2^15, random signs);
    cancelling (the second half of each row repeats the first negated, slightly perturbed); fp16 subnormals mixed with
    normals"""
    rng = np.random.default_rng(seed)
    q = p // 4
    out = np.empty((p, k))
    out[:q] = rng.standard_normal((q, k))
    sgn = rng.choice([-1.0, 1.0], (q, k))
    out[q:2 * q] = sgn * (1 + rng.random((q, k))) * 2.0 ** rng.integers(-24, 15, (q, k))
    h = rng.standard_normal((q, k // 2)) * 2.0 ** rng.integers(-8, 8, (q, 1))
    pert = np.where(rng.random((q, k // 2)) < 0.2, rng.standard_normal((q, k // 2)) * 2.0 ** -12, 0.0)
    out[2 * q:3 * q] = np.concatenate([h, -(h + pert) * np.where(rng.random((q, 1)) < 0.5, 1, -1)], 1)
    r = p - 3 * q
    out[3 * q:] = np.where(rng.random((r, k)) < 0.5, rng.integers(-1023, 1024, (r, k)) * 2.0 ** -24,
                           rng.standard_normal((r, k)) * 2.0 ** -10)
    return out.astype(_F16)


def fuzz_weights(n, k, seed):
    """[n, k] fp16 weight rows: half randn / sqrt(k), half wide exponents (2^-16 .. 2^4, random signs)"""
    rng = np.random.default_rng(seed)
    w = rng.standard_normal((n, k)) / np.sqrt(k)
    h = n // 2
    w[h:] = rng.choice([-1.0, 1.0], (n - h, k)) * (1 + rng.random((n - h, k))) * 2.0 ** rng.integers(-16, 4, (n - h, k))
    return w.astype(_F16)
