"""-m gpu: lp_pw1x1_f16 (the streaming pointwise kernel) at the 1x1 shapes of a LitePose-S 512x512 batch-32 pass.

1. Against an fp32 reference of the same op on fp16-rounded inputs (tolerance as in test_gpu_kernels).
2. Exact equality of one launch with the same problem split over several launches: row ranges (ragged, one 64-row
   tile, fewer rows than SMs) and column slices packed on their own (other NC instantiations, other tile counts per
   CTA).  Every output element accumulates the same K=16 slices in the same order whatever the split, then adds bias
   and residual the same way, so the values must match exactly (compared as floats: +0 == -0).
3. The same launch twice gives the same output."""
import pytest
import torch
import torch.nn.functional as F

from litepose_b200 import _lib
from gpu_util import pack_pw, q16, stream, tol_check

pytestmark = pytest.mark.gpu

# (M, K, N, act, res): the eight stride-2 / stage-3 launches of one pass at batch 32, plus a residual projection
BENCH_SHAPES = [
    (2097152, 16, 96, 2, False),
    (524288, 96, 16, 0, False),
    (131072, 96, 32, 0, False),
    (131072, 32, 192, 2, False),
    (32768, 192, 48, 0, False),
    (32768, 48, 288, 2, False),
    (32768, 120, 720, 2, False),
    (32768, 720, 120, 0, True),
]


def _inputs(m, k, n, res, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(m, k, generator=g).half().cuda()
    wt = q16(torch.randn(n, k, generator=g) / (k ** 0.5))
    b = torch.randn(n, generator=g) * 0.1
    r = torch.randn(m, n, generator=g).half().cuda() if res else None
    return a, wt, b, r


def _run(a, wp, bp, r, m, k, n, act, out=None):
    lib = _lib.load()
    if out is None:
        out = torch.full((m, n), float("nan"), dtype=torch.float16, device="cuda")
    _lib.check(lib.lp_pw1x1_f16(a.data_ptr(), wp.data_ptr(), bp.data_ptr(), None if r is None else r.data_ptr(),
                                out.data_ptr(), m, k, n, act, stream()), "pw1x1")
    return out


def _same(x, y, what):
    assert x.shape == y.shape, what
    bad = ~(x == y)
    assert not bad.any(), "%s: %d elements differ, first at %s" % (what, int(bad.sum()), bad.nonzero()[0].tolist())


@pytest.mark.parametrize("m,k,n,act,res", BENCH_SHAPES)
def test_pw_bench_shapes_vs_fp32(m, k, n, act, res):
    a, wt, b, r = _inputs(m, k, n, res, m + k + n)
    wp, bp = pack_pw(wt, b)
    out = _run(a, wp, bp, r, m, k, n, act)
    torch.cuda.synchronize()
    ref = a.float() @ wt.cuda().t() + b.cuda()
    ref = F.relu6(ref) if act == 2 else (F.relu(ref) if act == 1 else ref)
    if res:
        ref = ref + r.float()
    tol_check(out, ref, what="pw %dx%dx%d" % (m, k, n))


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("k,n", [(120, 720), (16, 96), (96, 16), (192, 48), (720, 120)])
def test_pw_row_split_is_exact(k, n, act, res):
    m = 20000
    a, wt, b, r = _inputs(m, k, n, res, 7 * k + n)
    wp, bp = pack_pw(wt, b)
    full = _run(a, wp, bp, r, m, k, n, act)
    parts = torch.full_like(full, float("nan"))
    # one 64-row tile, fewer rows than SMs, a ragged middle, a ragged tail
    bounds = [0, 64, 64 + 100, 64 + 100 + 12345, m]
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        _run(a[lo:hi], wp, bp, None if r is None else r[lo:hi], hi - lo, k, n, act, out=parts[lo:hi])
    torch.cuda.synchronize()
    _same(full, parts, "row split k%d n%d act%d res%d" % (k, n, act, res))


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("m,width", [(32768, 80), (32768, 144), (3000, 240), (1000, 16)])
def test_pw_column_split_is_exact(m, width, act, res):
    k, n = 120, 720
    a, wt, b, r = _inputs(m, k, n, res, m + width)
    wp, bp = pack_pw(wt, b)
    full = _run(a, wp, bp, r, m, k, n, act)
    for j in range(n // width):
        cols = slice(j * width, (j + 1) * width)
        wpj, bpj = pack_pw(wt[cols].contiguous(), b[cols].contiguous())
        rj = None if r is None else r[:, cols].contiguous()
        part = _run(a, wpj, bpj, rj, m, k, width, act)
        torch.cuda.synchronize()
        _same(full[:, cols], part, "column slice %d x %d act%d res%d" % (j, width, act, res))


@pytest.mark.parametrize("m,k,n,res", [(2097152, 16, 96, False), (32768, 120, 720, False), (50000, 96, 16, True),
                                       (64, 960, 160, True)])
def test_pw_repeat_is_identical(m, k, n, res):
    a, wt, b, r = _inputs(m, k, n, res, 3)
    wp, bp = pack_pw(wt, b)
    x = _run(a, wp, bp, r, m, k, n, 2)
    y = _run(a, wp, bp, r, m, k, n, 2)
    torch.cuda.synchronize()
    _same(x, y, "repeat %dx%dx%d" % (m, k, n))
