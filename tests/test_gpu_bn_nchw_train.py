"""-m gpu: the NCHW train-mode BatchNorm kernels (lp_bn_nchw_fwd / _bwd) bit for bit against bn_nchw_train_emul, and
litepose_b200.train_bn's autograd function and converter against PyTorch and on real training steps, with
litepose_b200.train_dw's converter on as well."""
import copy
import random

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import bn_nchw_train_emul as bte
from litepose_b200 import _lib, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models import pose_mobilenet, pose_supermobilenet
from litepose_b200.lib.models.pose_supermobilenet import SuperBatchNorm2d
from litepose_b200.train_bn import (ACT_NONE, ACT_RELU, ACT_RELU6, BatchNormAct2d, batch_norm_act,
                                    convert_batchnorm)
from litepose_b200.train_dw import convert_depthwise

pytestmark = pytest.mark.gpu

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False

_CODE = {torch.float32: _lib.LP_DT_F32, torch.float16: _lib.LP_DT_F16}
ACTS = [ACT_NONE, ACT_RELU, ACT_RELU6]
MOM, EPS = 0.1, 1e-5


def _st():
    return torch.cuda.current_stream().cuda_stream


def kfwd(x, g, b, rm, rv, act):
    """-> y, saved; rm / rv updated in place"""
    lib = _lib.load()
    n, c, h, w = x.shape
    y = torch.empty_like(x)
    saved = torch.empty(4, c, device="cuda")
    nb = lib.lp_bn_nchw_workspace_bytes(n, c, h, w)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    _lib.check(lib.lp_bn_nchw_fwd(x.data_ptr(), g.data_ptr(), b.data_ptr(), rm.data_ptr(), rv.data_ptr(), MOM, EPS,
                                  y.data_ptr(), saved.data_ptr(), n, c, h, w, act, _CODE[x.dtype], ws.data_ptr(), nb,
                                  _st()), "fwd")
    return y, saved


def kbwd(x, dy, g, saved, act):
    lib = _lib.load()
    n, c, h, w = x.shape
    dx = torch.empty_like(x)
    dg, db = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    nb = lib.lp_bn_nchw_workspace_bytes(n, c, h, w)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    _lib.check(lib.lp_bn_nchw_bwd(x.data_ptr(), dy.data_ptr(), g.data_ptr(), saved.data_ptr(), dx.data_ptr(),
                                  dg.data_ptr(), db.data_ptr(), n, c, h, w, act, _CODE[x.dtype], ws.data_ptr(), nb,
                                  _st()), "bwd")
    return dx, dg, db


def _inputs(n, c, h, w, dt, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(n, c, h, w, device="cuda", generator=g) * 2 +
         torch.randn(1, c, 1, 1, device="cuda", generator=g)).to(dt)
    gamma = torch.rand(c, device="cuda", generator=g) + 0.5
    beta = torch.randn(c, device="cuda", generator=g) * 0.5
    rm = torch.randn(c, device="cuda", generator=g) * 0.1
    rv = torch.rand(c, device="cuda", generator=g) * 0.5 + 0.75
    dy = torch.randn(n, c, h, w, device="cuda", generator=g).to(dt)
    return x, gamma, beta, rm, rv, dy


def _np(t):
    return t.detach().cpu().numpy()


def _same(got, want, what):
    got = _np(got)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    eq = (got == want) | (np.isnan(got) & np.isnan(want))
    assert eq.all(), "%s: %d of %d differ, first at %s" % (what, (~eq).sum(), eq.size, np.argwhere(~eq)[0])


def _check_all(n, c, h, w, dt, act, seed, channels=None):
    x, g, b, rm, rv, dy = _inputs(n, c, h, w, dt, seed)
    rm0, rv0 = _np(rm), _np(rv)
    y, saved = kfwd(x, g, b, rm, rv, act)
    dx, dg, db = kbwd(x, dy, g, saved, act)
    what = "act %d %s %s" % (act, dt, (n, c, h, w))
    cs = list(range(c)) if channels is None else channels
    sl = slice(None) if channels is None else cs
    xn, dn = _np(x)[:, sl], _np(dy)[:, sl]        # a channel's results depend on that channel's values only
    gn, bn_ = _np(g)[sl], _np(b)[sl]
    ey, es, em, ev = bte.fwd(xn, gn, bn_, rm0[sl], rv0[sl], MOM, EPS, act)
    _same(y[:, sl], ey, "y " + what)
    _same(saved[:, sl], es, "saved " + what)
    _same(rm[sl], em, "running_mean " + what)
    _same(rv[sl], ev, "running_var " + what)
    edx, edg, edb = bte.bwd(xn, dn, gn, es, act)
    _same(dx[:, sl], edx, "dx " + what)
    _same(dg[sl], edg, "dgamma " + what)
    _same(db[sl], edb, "dbeta " + what)


# small and odd planes (every channel checked), the 14 distinct BN shapes of LitePose-S at 448^2, batch 16 (a sample
# of channels checked), and N * C past one grid row
SMALL = [(2, 3, 9, 11), (5, 2, 1, 1), (3, 5, 61, 53), (16, 3, 7, 7), (16, 6, 11, 11)]
LITEPOSE = [(16, 32, 224, 224), (16, 16, 224, 224), (16, 96, 224, 224), (16, 96, 112, 112), (16, 16, 112, 112),
            (16, 24, 112, 112), (16, 96, 56, 56), (16, 32, 56, 56), (16, 192, 56, 56), (16, 192, 28, 28),
            (16, 48, 28, 28), (16, 288, 28, 28), (16, 120, 28, 28), (16, 720, 28, 28)]
WIDE = (2, 40000, 3, 5)
COMBOS = [(dt, act) for dt in (torch.float32, torch.float16) for act in ACTS]


@pytest.mark.parametrize("dt,act", COMBOS, ids=["%s-act%d" % (str(d)[6:], a) for d, a in COMBOS])
def test_entry_points_equal_emulator(dt, act):
    for i, shape in enumerate(SMALL):
        _check_all(*shape, dt, act, 10 * act + i)
    ci = COMBOS.index((dt, act))
    for j in range(ci, len(LITEPOSE), len(COMBOS)):
        n, c, h, w = LITEPOSE[j]
        _check_all(n, c, h, w, dt, act, j, channels=[0, c // 3, c - 1])
    if ci % 3 == 0:
        _check_all(*WIDE, dt, act, ci, channels=[0, 32768, 39999])


@pytest.mark.parametrize("act", ACTS)
def test_fp16_is_fp32_rounded(act):
    x, g, b, rm, rv, dy = _inputs(4, 24, 57, 70, torch.float16, act)
    rm2, rv2 = rm.clone(), rv.clone()
    y16, s16 = kfwd(x, g, b, rm, rv, act)
    y32, s32 = kfwd(x.float(), g, b, rm2, rv2, act)
    assert torch.equal(y16.view(torch.int16), y32.half().view(torch.int16)) and torch.equal(s16, s32)
    assert torch.equal(rm, rm2) and torch.equal(rv, rv2)
    b16, b32 = kbwd(x, dy, g, s16, act), kbwd(x.float(), dy.float(), g, s32, act)
    assert torch.equal(b16[0].view(torch.int16), b32[0].half().view(torch.int16))
    assert torch.equal(b16[1], b32[1]) and torch.equal(b16[2], b32[2])


def test_same_bits_every_call_and_stream():
    x, g, b, rm, rv, dy = _inputs(16, 96, 112, 112, torch.float32, 5)
    r0 = (rm.clone(), rv.clone())

    def run():
        m, v = r0[0].clone(), r0[1].clone()
        y, s = kfwd(x, g, b, m, v, ACT_RELU6)
        return [y, s, m, v] + list(kbwd(x, dy, g, s, ACT_RELU6))

    ref = run()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for rep in range(3):
        with torch.cuda.stream(side if rep == 2 else torch.cuda.current_stream()):
            got = run()
        torch.cuda.synchronize()
        for a, b_ in zip(got, ref):
            assert torch.equal(a.view(torch.int32), b_.view(torch.int32))


# ---------------------------------------------------------------- the autograd function against PyTorch
def _torch_act(y, act):
    return F.relu(y) if act == ACT_RELU else F.relu6(y) if act == ACT_RELU6 else y


@pytest.mark.parametrize("act", ACTS)
def test_autograd_within_bound_of_fp64(act):
    n, c, h, w = 4, 12, 23, 19
    x, g, b, rm, rv, dy = _inputs(n, c, h, w, torch.float32, 7 + act)
    xr, gr, br = x.clone().requires_grad_(True), g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    m, v = rm.clone(), rv.clone()
    y = batch_norm_act(xr, gr, br, m, v, MOM, EPS, act)
    y.backward(dy)
    xn, gn, bn_, dn = _np(x), _np(g), _np(b), _np(dy)
    ey, es, em, ev = bte.fwd(xn, gn, bn_, _np(rm), _np(rv), MOM, EPS, act)
    ex, _, _, _ = bte.exact_fwd(xn, gn, bn_, EPS, act)
    assert (np.abs(_np(y).astype(np.float64) - ex) <= bte.bound_fwd(xn, gn, bn_, EPS)).all()
    dx64, dg64, db64 = bte.exact_bwd(xn, dn, gn, EPS, es, act)
    ldx, ldg, ldb = bte.bound_bwd(xn, dn, gn, EPS, es, act)
    for got, exact, lim, what in ((xr.grad, dx64, ldx, "dx"), (gr.grad, dg64, ldg, "dgamma"),
                                  (br.grad, db64, ldb, "dbeta")):
        err = np.abs(_np(got).astype(np.float64) - exact)
        assert (err <= lim).all(), (what, float((err - lim).max()))
    _same(y, ey, "y")                                     # and exactly the kernels
    _same(m, em, "running_mean")
    _same(v, ev, "running_var")
    edx, edg, edb = bte.bwd(xn, dn, gn, es, act)
    _same(xr.grad, edx, "dx")
    _same(gr.grad, edg, "dgamma")
    _same(br.grad, edb, "dbeta")


@pytest.mark.parametrize("act", ACTS)
def test_modules_match_pytorch(act):
    """outputs, gradients, running statistics and num_batches_tracked of nn.BatchNorm2d / SuperBatchNorm2d (+ the
    activation) over three steps, converted against unconverted"""
    a = {ACT_RELU: [nn.ReLU(inplace=True)], ACT_RELU6: [nn.ReLU6(inplace=True)]}.get(act, [])
    for cls, cin in ((nn.BatchNorm2d, 16), (SuperBatchNorm2d, 12)):
        ref = synth.randomize_bn_(nn.Sequential(cls(16), *copy.deepcopy(a)), act + 1).cuda().train()
        conv = convert_batchnorm(copy.deepcopy(ref))
        assert type(conv[0]) is not cls
        for step in range(3):
            x, _, _, _, _, dy = _inputs(8, cin, 15, 17, torch.float32, 10 * step + act)
            outs = []
            for m in (ref, conv):
                xr = x.clone().requires_grad_(True)
                y = m(xr)
                y.backward(dy)
                outs.append((y.detach(), xr.grad))
            torch.testing.assert_close(outs[1][0], outs[0][0], rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(outs[1][1], outs[0][1], rtol=1e-4, atol=1e-5)
        for p, q in zip(ref.parameters(), conv.parameters()):
            torch.testing.assert_close(q.grad, p.grad, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(conv[0].running_mean, ref[0].running_mean, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(conv[0].running_var, ref[0].running_var, rtol=1e-5, atol=1e-6)
        assert int(conv[0].num_batches_tracked) == int(ref[0].num_batches_tracked)
        assert int(conv[0].num_batches_tracked) == (3 if cls is nn.BatchNorm2d else 0)


def test_nan_and_inf_propagate_as_in_pytorch():
    x, g, b, rm, rv, dy = _inputs(2, 4, 6, 6, torch.float32, 3)
    x[0, 1, 2, 2] = float("nan")
    x[1, 2, 0, 0] = float("inf")
    for act in ACTS:
        outs = []
        for fused in (True, False):
            xr = x.clone().requires_grad_(True)
            m, v = rm.clone(), rv.clone()
            if fused:
                y = batch_norm_act(xr, g, b, m, v, MOM, EPS, act)
            else:
                y = _torch_act(F.batch_norm(xr, m, v, g, b, True, MOM, EPS), act)
            y.backward(dy)
            outs.append((y.detach(), xr.grad, m, v))
        for a, b_ in zip(*outs):
            assert torch.equal(torch.isnan(a), torch.isnan(b_)), act
            assert torch.equal(torch.isinf(a), torch.isinf(b_)), act
        assert torch.isnan(outs[0][0][:, 1]).all() and not torch.isnan(outs[0][0][:, 0]).any()
    # a NaN gradient propagates where the activation passes it, and is masked where it does not
    xr = x[:, :1].clone().requires_grad_(True)
    y = batch_norm_act(xr, g[:1], b[:1], rm[:1].clone(), rv[:1].clone(), MOM, EPS, ACT_RELU)
    d = dy[:, :1].clone()
    d[y.detach() > 0] = float("nan")
    y.backward(d)
    assert torch.isnan(xr.grad).all()


def test_no_host_synchronisation():
    x, g, b, rm, rv, dy = _inputs(4, 8, 16, 16, torch.float32, 2)
    xr, gr, br = x.requires_grad_(True), g.requires_grad_(True), b.requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = batch_norm_act(xr, gr, br, rm, rv, MOM, EPS, ACT_RELU6)
        y.backward(dy)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_backward_launches_only_what_is_needed():
    lib = _lib.load()
    x, g, b, rm, rv, dy = _inputs(2, 8, 20, 20, torch.float32, 3)
    for need_x, need_p, launches in ((True, False, 3), (False, True, 2), (True, True, 3), (False, False, 0)):
        xr, gr, br = x.clone().requires_grad_(need_x), g.clone().requires_grad_(need_p), b.clone().requires_grad_(need_p)
        y = batch_norm_act(xr, gr, br, rm, rv, MOM, EPS, ACT_RELU6)
        if not y.requires_grad:
            continue
        torch.cuda.synchronize()
        before = lib.lp_launch_count()
        y.backward(dy)
        torch.cuda.synchronize()
        assert lib.lp_launch_count() - before == launches, (need_x, need_p)
        assert (xr.grad is not None) == need_x and (gr.grad is not None) == need_p
    y = batch_norm_act(x.requires_grad_(True), g, b, rm, rv, MOM, EPS, ACT_RELU)
    gx = torch.autograd.grad(y, (x,), dy, create_graph=True)[0]
    with pytest.raises(RuntimeError):
        gx.sum().backward()                 # once_differentiable: no double backward


def test_refusals():
    x, g, b, rm, rv, _ = _inputs(2, 4, 3, 3, torch.float32, 1)
    for args, msg in (((x.bfloat16(), g, b, rm, rv), "bfloat16"), ((x.double(), g, b, rm, rv), "float64"),
                      ((x.half(), g.half(), b, rm, rv), "fp32"), ((x, g, b, rm.half(), rv), "fp32"),
                      ((x[:1, :, :1, :1], g, b, rm, rv), "more than 1 value"), ((x, g[:3], b, rm, rv), "do not fit")):
        with pytest.raises(ValueError, match=msg):
            batch_norm_act(*args, MOM, EPS, ACT_RELU)
    with pytest.raises(ValueError, match="momentum None"):
        batch_norm_act(x, g, b, rm, rv, None, EPS, ACT_RELU)
    m = convert_batchnorm(nn.BatchNorm2d(4)).cuda().train()
    m.momentum = None
    with pytest.raises(ValueError, match="momentum None"):
        m(x)


def test_eval_after_training_runs_the_engine_on_the_updated_statistics():
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_mobilenet.get_pose_net(get_cfg(input_size=128), False, get_arch("XS")), 1)
    conv = convert_batchnorm(convert_depthwise(copy.deepcopy(model))).cuda().eval()
    ref = copy.deepcopy(model).cuda().eval()
    x = synth.make_frames(2, 128, seed=4).cuda()
    with torch.no_grad():
        before = [o.clone() for o in conv(x)]
        for a, b in zip(ref(x), before):
            assert torch.equal(a, b)                 # eval of a converted model: the engine, unchanged
    # a train-mode forward updates the running statistics in place; eval then runs the engine on them, without a
    # train() / eval() switch in between (the version counters tell the engine's cache)
    conv.train()
    conv(synth.make_frames(4, 128, seed=5).cuda())
    for m in conv.modules():
        m.training = False
    with torch.no_grad():
        after = conv(x)
        fresh = copy.deepcopy(conv).eval()
        fresh.lp_invalidate()
        for a, b in zip(after, fresh(x)):
            assert torch.equal(a, b)
        assert any(not torch.equal(a, b) for a, b in zip(after, before))


def test_supernet_reorganize_and_recalibrate_unchanged():
    cfg = get_cfg(input_size=256)
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_supermobilenet.get_pose_net(cfg), 1).cuda()
    conv = convert_batchnorm(copy.deepcopy(model))
    model.re_organize_weights()
    conv.re_organize_weights()
    x = synth.make_frames(2, 256, seed=3).cuda()
    for m in (model, conv):
        random.seed(5)
        m.lp_recalibrate_bn(x)
    sd1, sd2 = model.state_dict(), conv.state_dict()
    assert list(sd1) == list(sd2) and all(torch.equal(sd1[k], sd2[k]) for k in sd1)


# ---------------------------------------------------------------- whole training steps against fp64
LR = 1e-3
FLOOR = 1e-6          # of max |fp64 gradient| of the tensor: the fp32 rounding level a 0-distance cuDNN step can hide
# The step is chaotic at the ReLU / ReLU6 boundaries: a pre-activation within rounding of 0 or 6 lands on either side,
# and each such flip moves a gradient by a whole incoming gradient.  The cuDNN step itself on an input perturbed by
# one unit in the last place moves single gradient tensors by up to ~5x its unperturbed distance from fp64 (measured
# on LitePose-S, H100), although the BatchNorm kernels are as accurate as cuDNN's layer by layer.  So the converted
# step's distance summed over all tensors is held to 2x the cuDNN step's, and each tensor's to 4x the largest distance
# of the cuDNN step and PERTURB cuDNN steps on inputs perturbed that way.  In the fp16 steps cuDNN's own fp16
# depthwise convolution can overflow (it does in the drawn super-network architecture); a tensor or statistic that no
# cuDNN step computes finitely is only required to be finite.
PERTURB = 6
HALF_LOSS_SCALE = 2.0 ** -6   # a static loss scale for the fp16 steps: the unscaled loss overflows cuDNN's fp16 wgrad


def _half_model(model):
    """network_to_half: the model in fp16 with its BatchNorms kept in fp32 (BN_convert_float)"""
    model = model.half()
    for m in model.modules():
        if isinstance(m, nn.modules.batchnorm._BatchNorm):
            m.float()
    return model


def _train_step(model, x, seed, dt, autocast=False, loss_scale=1.0):
    random.seed(seed)
    model.zero_grad(set_to_none=True)
    with torch.autocast("cuda", torch.float16, enabled=autocast):
        outs = model(x.cuda().to(dt))
    wts = [torch.linspace(-1, 1, o.numel(), device="cuda", dtype=torch.float64).reshape(o.shape) for o in outs]
    loss = sum((o.double() * t).sum() for o, t in zip(outs, wts)) * loss_scale
    loss.backward()
    grads = {n: p.grad.detach().double().clone() for n, p in model.named_parameters() if p.grad is not None}
    # Adam on fp32 master copies of the parameters (fp64 for the fp64 model), as FP16_Optimizer steps an fp16 model
    names = [n for n, _ in model.named_parameters()]
    masters = []
    for _, p in model.named_parameters():
        m = p.detach().to(torch.float64 if p.dtype == torch.float64 else torch.float32).clone()
        m.grad = None if p.grad is None else p.grad.detach().to(m.dtype)
        masters.append(m)
    torch.optim.Adam(masters, lr=LR).step()
    stats = {n: b.detach().double().clone() for n, b in model.named_buffers() if "running" in n}
    return grads, {n: m.double() for n, m in zip(names, masters)}, stats


def _perturbed(x, k, rel):
    g = torch.Generator().manual_seed(100 + k)
    return x * (1 + rel * (torch.randint(0, 2, x.shape, generator=g).to(x.dtype) * 2 - 1))


def _compare_step(model, x, seed, mode="fp32"):
    """gradients, post-Adam parameters and running statistics of the converted step (depthwise + BatchNorm kernels)
    against an fp64 step: summed over the gradient tensors within 2x the cuDNN step's distance, each tensor within 4x
    the perturbed cuDNN steps' (see PERTURB)"""
    dt = torch.float16 if mode == "half" else torch.float32
    ac = mode == "autocast"
    ls = 1.0 if mode == "fp32" else HALF_LOSS_SCALE
    rel = 2.0 ** -23 if mode == "fp32" else 2.0 ** -10      # one unit in the last place of what the step computes in
    prep = _half_model if mode == "half" else (lambda m: m)
    m64 = copy.deepcopy(model).double().cuda().train()
    conv = prep(convert_batchnorm(convert_depthwise(copy.deepcopy(model))).cuda()).train()
    g64, p64, s64 = _train_step(m64, x, seed, torch.float64, loss_scale=ls)
    gr, pr, sr = _train_step(prep(copy.deepcopy(model).cuda()).train(), x, seed, dt, ac, ls)
    gps = [_train_step(prep(copy.deepcopy(model).cuda()).train(), _perturbed(x, k, rel), seed, dt, ac, ls)[0]
           for k in range(PERTURB)]
    gc, pc, sc = _train_step(conv, x, seed, dt, ac, ls)
    assert list(gc) == list(g64) == list(gr)
    tot_c = tot_r = 0.0
    for name in g64:
        scale = g64[name].abs().max().item()
        ec = (gc[name] - g64[name]).abs().max().item()
        assert np.isfinite(ec), name
        dists = [(g[name] - g64[name]).abs().max().item() for g in [gr] + gps]
        finite = [d for d in dists if np.isfinite(d)]
        if not finite:
            continue        # no cuDNN step computes this one finitely: finite is all we ask
        env = max(finite)
        assert ec <= 4 * env + FLOOR * scale + 1e-30, "%s: converted %.3e, cuDNN %.3e, perturbed cuDNN %.3e " \
            "(max |g| %.3e)" % (name, ec, dists[0], env, scale)
        if np.isfinite(dists[0]):
            tot_c, tot_r = tot_c + ec, tot_r + dists[0]
    assert tot_c <= 2 * tot_r, (tot_c, tot_r)
    for name in g64:
        # Adam's first step moves a parameter by lr * g / (|g| + eps): a gradient error dg moves it by at most
        # lr * min(2, 2 |dg| / (|g| + eps)) (the gradients' own bound is held above).  Not for the fp16 model, whose
        # parameters start rounded to fp16 and so apart from the fp64 model's.
        if mode == "half" or not np.isfinite(gr[name].abs().max().item()):
            continue
        lim = LR * torch.clamp(2 * (gc[name] - g64[name]).abs() / (g64[name].abs() + 1e-8), max=2) + 1e-7
        assert ((pc[name] - p64[name]).abs() <= lim).all(), "%s after Adam" % name
    for name in s64:
        ec = (sc[name] - s64[name]).abs().max().item()
        er = (sr[name] - s64[name]).abs().max().item()
        assert np.isfinite(ec), name
        lim = 2 * er + 1e-6 * s64[name].abs().max().item() + 1e-30
        assert not np.isfinite(er) or ec <= lim, "%s: converted %.3e, cuDNN %.3e" % (name, ec, er)


def _litepose_s():
    torch.manual_seed(0)
    return synth.randomize_bn_(pose_mobilenet.get_pose_net(get_cfg(input_size=256), False, get_arch("S")), 1)


def _supernet():
    cfg = get_cfg(input_size=256)
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_supermobilenet.get_pose_net(cfg), 1)
    random.seed(4)
    arch = model.arch_manager.random_sample()
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            st["block_setting"][bi] = [6, (7, 5, 3)[(si + bi) % 3]]
    model.arch_manager.is_search, model.arch_manager.search_arch = True, arch
    return model


@pytest.mark.parametrize("mode", ["fp32", "half", "autocast"])
def test_train_step_litepose_s(mode):
    _compare_step(_litepose_s(), synth.make_frames(4, 256, seed=1), 0, mode)


@pytest.mark.parametrize("mode", ["fp32", "half", "autocast"])
def test_train_step_supernet_random_sample(mode):
    _compare_step(_supernet(), synth.make_frames(2, 256, seed=2), 0, mode)


def test_converted_step_runs_the_kernels_and_fuses_the_activations():
    model = convert_batchnorm(_litepose_s()).cuda().train()
    lib = _lib.load()
    before = lib.lp_launch_count()
    outs = model(synth.make_frames(2, 256, seed=1).cuda())
    sum(o.sum() for o in outs).backward()
    torch.cuda.synchronize()
    # 112 BatchNorms, 3 launches forward and 3 backward each
    assert lib.lp_launch_count() - before == 112 * 6
    assert all(type(m) is BatchNormAct2d for m in model.modules() if isinstance(m, nn.BatchNorm2d))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_data_parallel_two_gpus():
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_mobilenet.get_pose_net(get_cfg(input_size=128), False, get_arch("XS")), 1)
    dp = nn.DataParallel(convert_batchnorm(copy.deepcopy(model)).cuda().train(), device_ids=[0, 1])
    x = synth.make_frames(4, 128, seed=6).cuda()
    outs = dp(x)
    sum(o.sum() for o in outs).backward()
    for n, p in dp.module.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    assert all(type(m) is BatchNormAct2d for m in dp.module.modules() if isinstance(m, nn.BatchNorm2d))
