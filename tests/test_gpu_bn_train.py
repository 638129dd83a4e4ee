"""-m gpu: the super-network's BN recalibration pass on the sm_90a kernels.

(a) lp_bn_stats_f16 / lp_bn_apply_f16 equal tests/bn_train_emul.py bit for bit, with the same bits on a second run:
    C from 8 to 720 (not all multiples of 64), M = 2, M around and past the 2048-pixel range of a statistics CTA, every
    activation with and without a residual, inputs with -0 and fp16 subnormals.
(b) lp_stem_conv3x3_s2_act and lp_fusion_deconv_act_f16: with the old activation equal to the existing entry points,
    with none equal to the restatement (both deconv kernels, one branch and two).
(c) lp_recalibrate_bn over the golden architectures and three batches equals bn_train_emul bit for bit in outputs and
    every buffer, untouched suffixes included; the eval forward after it equals a fresh module loaded with the
    recalibrated state dict; network_to_half recalibrates within tolerance of its module tree; a stem output that
    overflows fp16 raises and changes no buffer; model(x) in training mode still runs autograd."""
import copy

import numpy as np
import pytest
import torch

import bn_train_emul as bte
import conv_ref as cr
import mma_emul as me
import recal_cases as rc
from litepose_b200 import _lib
from litepose_b200.subnet import derive_supernet_subnet

pytestmark = pytest.mark.gpu
F16 = np.float16


@pytest.fixture(autouse=True)
def default_dw_precision():
    _lib.load().lp_set_dw_precision(-1)
    yield
    _lib.load().lp_set_dw_precision(-1)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16 if a.dtype == F16 else np.uint32)


def _x(m, c, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((m, c)) * np.exp(rng.standard_normal(c))).astype(F16)
    x[::7, ::3] = F16(-0.0)
    x[1::11, 1::5] = (rng.standard_normal(x[1::11, 1::5].shape) * 3e-6).astype(F16)   # fp16 subnormals
    return x


STATS_CASES = [(2, 8), (2, 720), (777, 24), (2048, 64), (2049, 200), (5000, 40), (9000, 720), (4100, 136)]


@pytest.mark.parametrize("m,c", STATS_CASES)
def test_stats_and_apply_exact(m, c):
    lib = _lib.load()
    rng = np.random.default_rng(m + c)
    x = _x(m, c, m * 3 + c)
    gamma = rng.uniform(0.5, 1.5, c).astype(np.float32)
    beta = (rng.standard_normal(c) * 0.1).astype(np.float32)
    rm = (rng.standard_normal(c) * 0.1).astype(np.float32)
    rv = rng.uniform(0.5, 1.5, c).astype(np.float32)
    mom, eps = 0.1, 1e-5
    dev = {k: torch.from_numpy(v).cuda() for k, v in dict(gamma=gamma, beta=beta, rm=rm, rv=rv).items()}
    xd = torch.from_numpy(x.view(np.int16)).cuda().view(torch.float16)
    ws = torch.empty(lib.lp_bn_stats_workspace_bytes(m, c), dtype=torch.uint8, device="cuda")
    want = bte.stats(x, gamma, beta, rm, rv, mom, eps)
    runs = []
    for _ in range(2):
        out = torch.full((4, c), float("nan"), device="cuda")
        flag = torch.zeros(1, dtype=torch.int32, device="cuda")
        _lib.check(lib.lp_bn_stats_f16(xd.data_ptr(), m, c, dev["gamma"].data_ptr(), dev["beta"].data_ptr(),
                                       dev["rm"].data_ptr(), dev["rv"].data_ptr(), mom, eps, out[0].data_ptr(),
                                       out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), flag.data_ptr(),
                                       ws.data_ptr(), ws.numel(), _stream()), "lp_bn_stats_f16")
        runs.append((out.cpu().numpy(), int(flag.item())))
    assert np.array_equal(_bits(runs[0][0]), _bits(runs[1][0]))
    for i in range(4):
        assert np.array_equal(_bits(runs[0][0][i]), _bits(want[i])), (m, c, i)
    assert runs[0][1] == int(want[4]) == 0
    scale, shift = runs[0][0][0], runs[0][0][1]
    res = _x(m, c, m + 5)
    rd = torch.from_numpy(res.view(np.int16)).cuda().view(torch.float16)
    sd, hd = torch.from_numpy(scale).cuda(), torch.from_numpy(shift).cuda()
    for act in (_lib.ACT_NONE, _lib.ACT_RELU, _lib.ACT_RELU6):
        for with_res in (False, True):
            got = []
            for in_place in (False, True):
                src = xd.clone()
                y = src if in_place else torch.empty_like(xd)
                _lib.check(lib.lp_bn_apply_f16(src.data_ptr(), sd.data_ptr(), hd.data_ptr(),
                                               rd.data_ptr() if with_res else None, y.data_ptr(), m, c, act, _stream()),
                           "lp_bn_apply_f16")
                got.append(y.cpu().numpy().view(F16))
            ref = bte.apply(x, scale, shift, act, res if with_res else None)
            assert np.array_equal(_bits(got[0]), _bits(ref)), (m, c, act, with_res)
            assert np.array_equal(_bits(got[1]), _bits(ref)), (m, c, act, with_res, "in place")


def test_stats_flags_non_finite():
    lib = _lib.load()
    m, c = 100, 16
    x = _x(m, c, 1)
    x[3, 5] = F16(np.inf)
    xd = torch.from_numpy(x.view(np.int16)).cuda().view(torch.float16)
    ones = torch.ones(c, device="cuda")
    out = torch.empty((4, c), device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.lp_bn_stats_workspace_bytes(m, c), dtype=torch.uint8, device="cuda")
    _lib.check(lib.lp_bn_stats_f16(xd.data_ptr(), m, c, ones.data_ptr(), ones.data_ptr(), ones.data_ptr(),
                                   ones.data_ptr(), 0.1, 1e-5, out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
                                   out[3].data_ptr(), flag.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "stats")
    assert int(flag.item()) == 1


@pytest.mark.parametrize("fp32", [True, False])
def test_stem_act(fp32):
    lib = _lib.load()
    rng = np.random.default_rng(3)
    n, h, w = 2, 32, 48
    x = (rng.standard_normal((n, 3, h, w)) * 2).astype(np.float32 if fp32 else F16)
    wt = (rng.standard_normal((32, 27)) * 0.3).astype(F16)
    bias = (rng.standard_normal(32) * 0.1).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    wd = torch.from_numpy(wt.view(np.int16)).cuda()
    bd = torch.from_numpy(bias).cuda()
    outs = {}
    for name, call in (("old", lambda y: lib.lp_stem_conv3x3_s2(xd.data_ptr(), int(fp32), 0, wd.data_ptr(),
                                                                  bd.data_ptr(), y.data_ptr(), n, h, w, _stream())),
                       ("relu6", lambda y: lib.lp_stem_conv3x3_s2_act(xd.data_ptr(), int(fp32), 0, wd.data_ptr(),
                                                                        bd.data_ptr(), y.data_ptr(), n, h, w,
                                                                        _lib.ACT_RELU6, _stream())),
                       ("none", lambda y: lib.lp_stem_conv3x3_s2_act(xd.data_ptr(), int(fp32), 0, wd.data_ptr(), None,
                                                                       y.data_ptr(), n, h, w, _lib.ACT_NONE,
                                                                       _stream()))):
        y = torch.empty((n, h // 2, w // 2, 32), dtype=torch.float16, device="cuda")
        _lib.check(call(y), name)
        outs[name] = y.cpu().numpy()
    assert np.array_equal(_bits(outs["old"]), _bits(outs["relu6"]))
    assert np.array_equal(_bits(outs["none"]), _bits(bte.stem_raw(x, wt)))


DECONV = [cr.DECONV_ROWS_CASES[1], cr.DECONV_ROWS_CASES[2], cr.DECONV_TILED_CASES[0], cr.DECONV_TILED_CASES[2]]


@pytest.mark.parametrize("case", DECONV)
@pytest.mark.parametrize("branches", [1, 2])
def test_deconv_act(case, branches):
    lib = _lib.load()
    n, h, w, c_r, c_w, co = case
    if branches == 1:
        c_w = 0
    xr, xw, wr, ww, bias = cr.deconv_inputs(n, h, w, c_r, c_w, co, seed=sum(case) + branches)
    wp = np.zeros(lib.lp_deconv_packed_elems(c_r, c_w, co), np.uint16)
    bp = np.zeros(lib.lp_deconv_packed_bias_elems(co), np.float32)
    _lib.check(lib.lp_deconv_pack(wr.view(np.uint16).ctypes.data, ww.view(np.uint16).ctypes.data if c_w else None,
                                  bias.ctypes.data, c_r, c_w, co, wp.ctypes.data, bp.ctypes.data), "pack")
    dev = [torch.from_numpy(a.view(np.int16) if a.dtype == F16 else a.view(np.int16)).cuda() for a in (xr, xw, wp)]
    bpd = torch.from_numpy(bp).cuda()
    outs = {}
    for name, act in (("old", None), ("relu", _lib.ACT_RELU), ("none", _lib.ACT_NONE)):
        y = torch.empty((n, 2 * h, 2 * w, co), dtype=torch.float16, device="cuda")
        args = [dev[0].data_ptr(), dev[1].data_ptr() if c_w else None, dev[2].data_ptr(), bpd.data_ptr(),
                y.data_ptr(), n, h, w, c_r, c_w, co]
        rc_ = lib.lp_fusion_deconv_f16(*args, _stream()) if act is None else \
            lib.lp_fusion_deconv_act_f16(*args, act, _stream())
        _lib.check(rc_, name)
        outs[name] = y.cpu().numpy()
    assert np.array_equal(_bits(outs["old"]), _bits(outs["relu"]))
    assert np.array_equal(_bits(outs["old"]), _bits(me.deconv(xr, xw, wr, ww, bias,
                                                               cr.uses_rows_kernel(c_r, c_w, co, w))))
    assert np.array_equal(_bits(outs["none"]), _bits(bte.deconv_raw(xr, xw, wr, ww, bias)))


# ---------------------------------------------------------------- the whole pass
@pytest.mark.parametrize("name", rc.ARCHS)
def test_recalibrate_equals_emulation(golden_dir, name):
    z, arch = rc.golden(golden_dir, name)
    inp = rc.inputs(golden_dir)
    model = rc.supernet(golden_dir, arch).cuda().eval()
    used = rc.used(model, arch)
    sub = derive_supernet_subnet(model.state_dict(), arch)
    params = {n: (0.1, 1e-5) for n in used}
    rm0, rv0 = np.asarray(inp["running_mean"]), np.asarray(inp["running_var"])
    running = {n: (rm0[o:o + c], rv0[o:o + c]) for n, (o, c) in used.items()}
    mask = np.ones(rm0.shape, bool)
    for n, (o, c) in used.items():
        mask[o:o + c] = False
    for i in range(3):
        x = inp["batches"][i].astype(np.float32)
        outs = model.lp_recalibrate_bn(torch.from_numpy(x).cuda())
        assert not model.training
        want, new, bad = bte.forward(sub, x, running, params)
        assert not bad
        running = new
        rm, rv, nbt = rc.state(model)
        for n, (o, c) in used.items():
            assert np.array_equal(_bits(rm[o:o + c]), _bits(new[n][0])), (name, i, n, "mean")
            assert np.array_equal(_bits(rv[o:o + c]), _bits(new[n][1])), (name, i, n, "var")
        assert np.array_equal(_bits(rm[mask]), _bits(rm0[mask])) and np.array_equal(_bits(rv[mask]), _bits(rv0[mask]))
        assert np.array_equal(nbt, z["num_batches_tracked"][i])
        for g, w_ in zip(outs, want):
            assert not g.requires_grad
            assert np.array_equal(_bits(g.cpu().numpy()), _bits(w_)), (name, i)
        for key in ("running_mean", "running_var"):
            got = rm if key == "running_mean" else rv
            assert rc.tol_used(got, z[key][i]) <= rc.TOL_FACTOR
    for k, g in zip(("out0", "out1"), outs):
        u = rc.tol_used(g.cpu().numpy(), z[k])
        print("%s %s: %.3f of the tolerance" % (name, k, u))
        assert u <= rc.TOL_FACTOR
    # the eval engine sees the new statistics: equal to a fresh module loaded with them
    x = torch.from_numpy(inp["batches"][0].astype(np.float32)).cuda()
    with torch.no_grad():
        after = model(x)
        fresh = rc.supernet(golden_dir, arch)
        fresh.load_state_dict(model.state_dict())
        ref = fresh.cuda().eval()(x)
    for a, b in zip(after, ref):
        assert torch.equal(a, b)


def test_network_to_half_recalibrates(golden_dir):
    _, arch = rc.golden(golden_dir, "search_XS")
    inp = rc.inputs(golden_dir)
    base = rc.supernet(golden_dir, arch).cuda()
    half = copy.deepcopy(base).half()
    for m in half.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.float()
    tree = copy.deepcopy(half).train()
    x = torch.from_numpy(inp["batches"][0]).cuda()
    outs = half.lp_recalibrate_bn(x)
    with torch.no_grad():
        want = tree(x)
    for g, w_ in zip(outs, want):
        assert g.dtype == torch.float16
        assert rc.tol_used(g.float().cpu().numpy(), w_.float().cpu().numpy()) <= rc.TOL_FACTOR
    for a, b in zip(rc.state(half)[:2], rc.state(tree)[:2]):
        assert rc.tol_used(a, b) <= rc.TOL_FACTOR


def test_non_finite_raises_and_changes_nothing(golden_dir):
    _, arch = rc.golden(golden_dir, "search_XS")
    model = rc.supernet(golden_dir, arch).cuda()
    before = rc.state(model)
    # conv weights start at std 0.001: with every pixel at 1e9 the raw stem sums (fp32) overflow fp16
    x = torch.full((2, 3, 64, 64), 1e9, device="cuda")
    with pytest.raises(_lib.LitePoseError, match="first.0.1"):
        model.lp_recalibrate_bn(x)
    after = rc.state(model)
    for a, b in zip(before, after):
        assert np.array_equal(a, b)


def test_train_mode_forward_keeps_autograd(golden_dir):
    _, arch = rc.golden(golden_dir, "search_XS")
    model = rc.supernet(golden_dir, arch).cuda().train()
    outs = model(torch.from_numpy(rc.inputs(golden_dir)["batches"][0]).float().cuda())
    assert all(o.requires_grad for o in outs)
