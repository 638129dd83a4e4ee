"""-m gpu: the tensor cores' fp16 -> fp32 accumulation measured, then every GEMM kernel held to it value for value.

(a) The probe rows of mma_probes.py and a random fuzz (wide exponents, cancellation, subnormals; K = 32, 64 and 256)
    through lp_head_pw_dual_f16 with fp32 output, which stores the raw accumulators: the device equals mma_emul.MODEL
    as bits on every output, and each parameter of the model is decided by its named probe group (every other value
    of that parameter disagrees with the device on that group).
(b) lp_pw1x1_f16 (resident and streaming weights, NC = 1..10, every activation, with and without a residual),
    lp_head_pw_dual_f16 (fp32 and fp16 output) and lp_fusion_deconv_f16 (both kernels, each in its own slice order)
    equal the emulator run over the kernel's K = 16 slices in issue order, with the kernel's epilogue.  Values are
    compared as floats (+0 == -0).
(c) LitePoseEngine.run equals net_emul.forward exactly (XS, S, M; fp32 / fp16 input and output; plain and mirrored
    pass; a 64 x 512 frame whose last deconv levels take the row kernel): the stem output, every block output, every
    deconv level and both head outputs, so a mismatch names the first op at fault.  Between them the cases run every op
    kind of the engine's plans."""
import numpy as np
import pytest
import torch

import conv_ref as cr
import mma_emul as me
import mma_probes as mp
from litepose_b200 import _lib
from gpu_util import pack_pw, stream

pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def assert_equal_values(got, want, what):
    got = np.asarray(got)
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    neq = got != want
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


def run_head(a1, a2, w1, w2, fp32, n=1, h=None, w=64):
    """lp_head_pw_dual_f16 on rows a1 [P, C1], a2 [P, C2] laid out as an [n, h, w] map; -> [P, Co] (pixel-major)"""
    lib = _lib.load()
    p, c1 = a1.shape
    c2 = a2.shape[1]
    co = w1.shape[0]
    if h is None:
        h = (p + n * w - 1) // (n * w)
    rows = n * h * w
    assert rows >= p

    def pad(x):
        y = np.zeros((rows, x.shape[1]), np.float16)
        y[:p] = x
        return _dev(y.reshape(n, h, w, -1))

    d1, d2 = pad(a1), pad(a2)
    wp = np.zeros(lib.lp_head_packed_elems(c1, c2, co), np.uint16)
    h1 = np.ascontiguousarray(w1, np.float16).view(np.uint16)      # held: .ctypes.data does not keep them alive
    h2 = np.ascontiguousarray(w2, np.float16).view(np.uint16)
    _lib.check(lib.lp_head_pack(h1.ctypes.data, h2.ctypes.data, c1, c2, co, wp.ctypes.data), "head_pack")
    wd = _dev(wp)
    out = torch.full((n, co, h, w), float("nan"), dtype=torch.float32 if fp32 else torch.float16, device="cuda")
    _lib.check(lib.lp_head_pw_dual_f16(d1.data_ptr(), d2.data_ptr(), wd.data_ptr(), out.data_ptr(), 1 if fp32 else 0,
                                       n, h, w, c1, c2, co, stream()), "head_pw_dual")
    torch.cuda.synchronize()
    return out.cpu().numpy().transpose(0, 2, 3, 1).reshape(rows, co)[:p]


# ---------------------------------------------------------------- (a) measurement
_probe_cache = {}


def _probe_out():
    if "out" not in _probe_cache:
        names, a = mp.probe_rows()
        w = mp.PROBE_WEIGHTS
        _probe_cache["out"] = (np.array(names), a, w, run_head(a[:, :16], a[:, 16:], w[:, :16], w[:, 16:], True))
    return _probe_cache["out"]


def _emul_probes(a, w, m=me.MODEL):
    return me.head_dual(a[:, :16], a[:, 16:], w[:, :16], w[:, 16:], True, m)


def _bit_mismatches(got, want):
    return np.asarray(got, np.float32).view(np.int32) != np.asarray(want, np.float32).view(np.int32)


def test_probes_equal_model_as_bits():
    names, a, w, got = _probe_out()
    bad = _bit_mismatches(got, _emul_probes(a, w))
    rows = np.nonzero(bad.any(1))[0]
    assert not len(rows), "%d probe outputs differ; first rows: %s" % (
        bad.sum(), ["%s (weight row %d: device %r, model %r)" % (names[r], np.nonzero(bad[r])[0][0],
                                                              got[r, np.nonzero(bad[r])[0][0]],
                                                              _emul_probes(a[r:r + 1], w)[0, np.nonzero(bad[r])[0][0]])
                    for r in rows[:5]])


def test_probes_fp16_output_equal_model():
    names, a, w, _ = _probe_out()
    got = run_head(a[:, :16], a[:, 16:], w[:, :16], w[:, 16:], False)
    want = me.head_dual(a[:, :16], a[:, 16:], w[:, :16], w[:, 16:], False)
    assert not _bit_mismatches(got.astype(np.float32), want.astype(np.float32)).any()


# parameter -> (probe group, the other values of the parameter); each must disagree with the device on the group
DECIDED_BY = {
    "B": ("B ", [dict(B=8), dict(B=4), dict(B=8, wide=True), dict(B=4, wide=True)]),
    "F": ("F_cancel ", [dict(F=24), dict(F=26)]),
    "align": ("F_cancel ", [dict(align="floor"), dict(align="rne")]),
    "c_align": ("c_align_cancel ", [dict(c_align=False)]),
    "norm": ("round ", [dict(norm="rne")]),
    "ftz": ("subnormal ", [dict(ftz=True)]),
    "lead": ("lead", [dict(lead="true"), dict(lead="clamp"), dict(lead="carry")]),
}


@pytest.mark.parametrize("param", sorted(DECIDED_BY))
def test_each_parameter_is_decided_by_its_probe(param):
    names, a, w, got = _probe_out()
    prefix, alts = DECIDED_BY[param]
    sel = np.array([n.startswith(prefix) for n in names])
    assert sel.sum() > 0
    assert not _bit_mismatches(got[sel], _emul_probes(a[sel], w)).any(), "%s: the model misses its own probe" % param
    for alt in alts:
        m = me.MODEL._replace(**alt)
        assert _bit_mismatches(got[sel], _emul_probes(a[sel], w, m)).any(), (
            "%s: probe group %r does not reject %s" % (param, prefix, alt))


def test_zero_results_are_positive():
    """1 - 1, -0 products onto +0, and tiny negative terms cut away all give +0 on the device"""
    names, a, w, got = _probe_out()
    sel = np.array([n.startswith("zero") for n in names])
    z = got[sel]
    assert (z[z == 0].view(np.int32) == 0).all()


# (rows, C1, C2, Co, seed): K = 32 (two steps), K = 64 with a partial slice per source, K = 256 (16 steps)
FUZZ = [(16384, 16, 16, 64, 1), (4096, 24, 40, 48, 3), (4096, 128, 128, 64, 2)]


@pytest.mark.parametrize("p,c1,c2,co,seed", FUZZ)
def test_fuzz_equals_model_as_bits(p, c1, c2, co, seed):
    a = mp.fuzz_rows(p, c1 + c2, seed)
    w = mp.fuzz_weights(co, c1 + c2, seed + 100)
    got = run_head(a[:, :c1], a[:, c1:], w[:, :c1], w[:, c1:], True)
    want = me.head_dual(a[:, :c1], a[:, c1:], w[:, :c1], w[:, c1:], True)
    bad = _bit_mismatches(got, want)
    assert not bad.any(), "%d of %d outputs differ, first %s: device %r model %r" % (
        bad.sum(), bad.size, np.argwhere(bad)[0], got[bad][0], want[bad][0])


# ---------------------------------------------------------------- (b) the GEMM kernels
def _pw_run(a, wt, b, r, act):
    lib = _lib.load()
    m, k = a.shape
    n = wt.shape[0]
    wpk, bpk = pack_pw(torch.from_numpy(wt), torch.from_numpy(b))
    out = torch.full((m, n), float("nan"), dtype=torch.float16, device="cuda")
    ad, rd = _dev(a), None if r is None else _dev(r)               # held until the kernel has run
    _lib.check(lib.lp_pw1x1_f16(ad.data_ptr(), wpk.data_ptr(), bpk.data_ptr(), None if rd is None else rd.data_ptr(),
                                out.data_ptr(), m, k, n, act, stream()), "pw1x1")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _pw_inputs(m, k, n, res, seed, wide=False):
    """randn activations (wide: a quarter of the rows with exponents over the fp16 range and subnormals), fan-in
    weights, a bias comparable to the accumulator, an optional residual"""
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((m, k))
    if wide:
        q = m // 4
        a[:q] *= 2.0 ** rng.integers(-20, 8, (q, k))
    wt = rng.standard_normal((n, k)) / k ** 0.5
    b = (rng.standard_normal(n) * np.where(np.arange(n) % 3 == 0, 4.0, 0.3)).astype(np.float32)
    r = rng.standard_normal((m, n)).astype(np.float16) if res else None
    return a.astype(np.float16), wt.astype(np.float16), b, r


# (m, k, n, act, res): PW_EDGE_SHAPES of test_gpu_dw_exact, the eight BENCH_SHAPES of test_gpu_pw_stream with M
# reduced (same K, N, activation, residual), and N = 16 NC for NC = 1..10 (resident weights) plus streaming weights
PW_SHAPES = [
    (1, 8, 8, 0, False), (63, 8, 24, 2, True), (65, 72, 24, 1, True), (64, 72, 168, 2, False), (65, 72, 168, 0, True),
    (1, 96, 1024, 0, True), (300, 32, 1024, 2, False), (63, 448, 256, 0, True), (1, 960, 160, 0, False),
    (65, 960, 160, 2, True), (4096, 24, 8, 1, True),
    (8192, 16, 96, 2, False), (4096, 96, 16, 0, False), (4096, 96, 32, 0, False), (4096, 32, 192, 2, False),
    (2048, 192, 48, 0, False), (2048, 48, 288, 2, False), (1024, 120, 720, 2, False), (1024, 720, 120, 0, True),
] + [(1000 + 13 * nc, 40 + 16 * (nc % 3), 16 * nc, nc % 3, nc % 2 == 0) for nc in range(1, 11)] + [
    (500, 960, 16 * nc, nc % 3, nc % 2 == 1) for nc in (1, 4, 10)]


@pytest.mark.parametrize("m,k,n,act,res", PW_SHAPES)
def test_pw1x1_equals_model(m, k, n, act, res):
    a, wt, b, r = _pw_inputs(m, k, n, res, m + 7 * k + n, wide=m >= 1000)
    got = _pw_run(a, wt, b, r, act)
    assert_equal_values(got, me.pw1x1(a, wt, b, r, act), "pw1x1 m%d k%d n%d act%d res%d" % (m, k, n, act, res))


# (n, h, w, C1, C2, Co)
HEAD_SHAPES = [(2, 16, 16, 16, 16, 17), (1, 24, 40, 32, 32, 34), (2, 12, 20, 24, 40, 14), (1, 8, 72, 72, 96, 17),
               (1, 16, 16, 192, 64, 256), (2, 5, 7, 8, 16, 30)]


@pytest.mark.parametrize("fp32", [True, False])
@pytest.mark.parametrize("n,h,w,c1,c2,co", HEAD_SHAPES)
def test_head_pw_dual_equals_model(n, h, w, c1, c2, co, fp32):
    rng = np.random.default_rng(n + h + w + c1 + c2 + co)
    p = n * h * w
    a1 = np.maximum(rng.standard_normal((p, c1)), 0).astype(np.float16)
    a2 = np.maximum(rng.standard_normal((p, c2)) * 2.0 ** rng.integers(-12, 4, (p, 1)), 0).astype(np.float16)
    w1 = (rng.standard_normal((co, c1)) / c1 ** 0.5).astype(np.float16)
    w2 = (rng.standard_normal((co, c2)) / c2 ** 0.5).astype(np.float16)
    got = run_head(a1, a2, w1, w2, fp32, n, h, w)
    assert_equal_values(got, me.head_dual(a1, a2, w1, w2, fp32),
                        "head n%d %dx%d c1 %d c2 %d co %d fp32 %d" % (n, h, w, c1, c2, co, fp32))


def run_deconv(xr, xw, wr, ww, b):
    lib = _lib.load()
    n, h, w, cr_ = xr.shape
    cw, co = xw.shape[3], wr.shape[1]
    wp = np.zeros(lib.lp_deconv_packed_elems(cr_, cw, co), np.uint16)
    bp = np.zeros(lib.lp_deconv_packed_bias_elems(co), np.float32)
    _lib.check(lib.lp_deconv_pack(wr.view(np.uint16).ctypes.data, ww.view(np.uint16).ctypes.data, b.ctypes.data, cr_,
                                  cw, co, wp.ctypes.data, bp.ctypes.data), "deconv_pack")
    out = torch.full((n, 2 * h, 2 * w, co), float("nan"), dtype=torch.float16, device="cuda")
    rd, rwd, wd, bd = _dev(xr), _dev(xw), _dev(wp.view(np.float16)), _dev(bp)     # held until the kernel has run
    _lib.check(lib.lp_fusion_deconv_f16(rd.data_ptr(), rwd.data_ptr(), wd.data_ptr(), bd.data_ptr(), out.data_ptr(), n,
                                        h, w, cr_, cw, co, stream()), "deconv")
    torch.cuda.synchronize()
    return out.cpu().numpy()


# the deconv cases of conv_ref, the largest row-kernel frames shrunk to keep the emulation cheap
DECONV_CASES = [c for c in cr.DECONV_ROWS_CASES if c[0] * c[1] * c[2] <= 40000] + [(2, 6, 128, 24, 16, 32),
                                                                                  (1, 12, 300, 8, 16, 8)]
DECONV_CASES += cr.DECONV_TILED_CASES


@pytest.mark.parametrize("n,h,w,cr_,cw,co", DECONV_CASES)
def test_deconv_equals_model(n, h, w, cr_, cw, co):
    rows = cr.uses_rows_kernel(cr_, cw, co, w)
    assert rows == ((n, h, w, cr_, cw, co) not in cr.DECONV_TILED_CASES)
    xr, xw, wr, ww, b = cr.deconv_inputs(n, h, w, cr_, cw, co, 3 * n + h + w + cr_ + cw + co)
    got = run_deconv(xr, xw, wr, ww, b)
    want = me.deconv(xr, xw, wr, ww, b, rows)
    assert_equal_values(got, want, "deconv %s n%d %dx%d cr%d cw%d co%d" % ("rows" if rows else "tiled", n, h, w, cr_,
                                                                            cw, co))


# ---------------------------------------------------------------- (c) the whole forward, bit for bit
# (arch, n, h, w, input dtype, fp32 output, mirrored pass): XS and S at batch 2 over every input / output / flip
# combination between them, M, and a 64 x 512 frame whose last two deconv levels take the row kernel
NET_CASES = [
    ("XS", 2, 128, 128, "fp16", True, False),
    ("XS", 2, 128, 128, "fp32", False, True),
    ("S", 2, 128, 128, "fp32", True, True),
    ("S", 2, 128, 128, "fp16", False, False),
    ("M", 1, 128, 128, "fp16", True, True),
    ("XS", 1, 64, 512, "fp16", True, False),
]
NET_OPS = {"stem_fused", "block_s1", "block_s2", "inv", "dw7_project", "dw7", "pc", "deconv rows", "deconv tiled",
           "head_fused"}
_ops_run = {}


def _net(arch_name, h):
    from litepose_b200 import synth
    from litepose_b200.config import get_arch, get_cfg
    from litepose_b200.lib.models.pose_mobilenet import get_pose_net
    arch = get_arch(arch_name)
    torch.manual_seed(0)
    model = synth.randomize_bn_(get_pose_net(get_cfg(input_size=h), False, arch), 1).eval()
    return arch, {k: v.detach().cpu() for k, v in model.state_dict().items()}


def _op_names(plan):
    names = set()
    for op in plan["ops"]:
        if op.name == "deconv":
            names.add("deconv rows" if cr.uses_rows_kernel(*op.args[8:11], op.args[7]) else "deconv tiled")
        else:
            names.add(op.name)
    return names


@pytest.mark.parametrize("case", NET_CASES, ids=["-".join(map(str, c)) for c in NET_CASES])
def test_engine_forward_equals_net_emul(case, dw_precision):
    import net_emul
    from litepose_b200 import engine, synth
    arch_name, n, h, w, dt, out_fp32, flip = case
    dw_precision(-1)
    arch, sd = _net(arch_name, h)
    x = synth.make_frames(n, h, seed=h + w + n, width=w)
    x = x.half() if dt == "fp16" else x
    eng = engine.LitePoseEngine(sd, arch, "cuda")
    got = eng.run(x.cuda(), flip=flip, out_fp32=out_fp32)
    torch.cuda.synchronize()
    plan = next(iter(eng.plans.values()))
    _ops_run[case] = _op_names(plan)
    keep = plan["keep"]
    fused_stem = "stem_fused" in _ops_run[case]
    inner = [keep[0]] + [t for t in keep[1 if fused_stem else 3:] if t.dim() == 4]
    trace = []
    want = net_emul.forward(sd, arch, x.numpy(), flip, out_fp32, trace)
    assert len(inner) == len(trace), (len(inner), [nm for nm, _ in trace])
    for t, (nm, wt) in zip(inner, trace):       # the first tensor that differs names the op at fault
        assert_equal_values(t.cpu().numpy(), wt, "%s %s" % ("-".join(map(str, case)), nm))
    assert len(got) == len(want) == 2
    for i, (g, wt) in enumerate(zip(got, want)):
        g = g.cpu().numpy()
        assert g.dtype == (np.float32 if out_fp32 else np.float16) and g.shape == wt.shape, (g.dtype, g.shape, wt.shape)
        assert_equal_values(g, wt, "%s output %d" % ("-".join(map(str, case)), i))


def test_engine_forward_cases_reach_every_op():
    """the forward cases above run every op kind of the engine's plans, both deconv kernels included (a case not run
    in this session contributes the plan it would run, built on the host)"""
    import torch as _t
    from litepose_b200 import engine
    reached = set()
    for case in NET_CASES:
        if case in _ops_run:
            reached |= _ops_run[case]
            continue
        arch_name, n, h, w, dt, out_fp32, flip = case
        arch, sd = _net(arch_name, h)
        eng = engine.LitePoseEngine(sd, arch, "cpu")
        reached |= _op_names(eng._build_plan(n, h, w, _t.float16 if dt == "fp16" else _t.float32, out_fp32,
                                             alloc=engine._Bump()))
    assert NET_OPS <= reached, sorted(NET_OPS - reached)
