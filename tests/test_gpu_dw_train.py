"""-m gpu: the NCHW depthwise training kernels (lp_dw_nchw_fwd / _dgrad / _wgrad) bit for bit against dw_train_emul, and
litepose_b200.train_dw's autograd function and converter on real training steps."""
import copy
import random

import numpy as np
import pytest
import torch
import torch.nn as nn

import dw_train_emul as dte
from litepose_b200 import _lib, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models import pose_mobilenet, pose_supermobilenet
from litepose_b200.train_dw import DepthwiseConv2d, convert_depthwise, depthwise_conv2d

pytestmark = pytest.mark.gpu

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False

_NP = {torch.float32: np.float32, torch.float16: np.float16}
_CODE = {torch.float32: _lib.LP_DT_F32, torch.float16: _lib.LP_DT_F16}


def _st():
    return torch.cuda.current_stream().cuda_stream


def kfwd(x, w, s):
    n, c, h, wd = x.shape
    k = w.shape[-1]
    y = torch.empty(n, c, dte.out_size(h, s), dte.out_size(wd, s), dtype=x.dtype, device="cuda")
    _lib.check(_lib.load().lp_dw_nchw_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), n, c, h, wd, k, s, _CODE[x.dtype],
                                          _st()), "fwd")
    return y


def kdgrad(dy, w, s, h, wd):
    n, c = dy.shape[:2]
    k = w.shape[-1]
    dx = torch.empty(n, c, h, wd, dtype=dy.dtype, device="cuda")
    _lib.check(_lib.load().lp_dw_nchw_dgrad(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), n, c, h, wd, k, s,
                                            _CODE[dy.dtype], _st()), "dgrad")
    return dx


def kwgrad(x, dy, k, s):
    lib = _lib.load()
    n, c, h, wd = x.shape
    nb = lib.lp_dw_nchw_wgrad_workspace_bytes(n, c, h, wd, k, s)
    ws = torch.empty(max(nb, 4), dtype=torch.uint8, device="cuda")
    dw = torch.empty(c, k, k, dtype=x.dtype, device="cuda")
    _lib.check(lib.lp_dw_nchw_wgrad(x.data_ptr(), dy.data_ptr(), dw.data_ptr(), n, c, h, wd, k, s, _CODE[x.dtype],
                                    ws.data_ptr(), nb, _st()), "wgrad")
    return dw


def _inputs(n, c, h, w, k, s, dt, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, c, h, w, device="cuda", generator=g).to(dt)
    wt = (torch.randn(c, k, k, device="cuda", generator=g) / k).to(dt)
    dy = torch.randn(n, c, dte.out_size(h, s), dte.out_size(w, s), device="cuda", generator=g).to(dt)
    return x, wt, dy


def _same(got, want, what):
    got = got.cpu().numpy()
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    eq = (got == want) | (np.isnan(got) & np.isnan(want))
    assert eq.all(), "%s: %d of %d differ, first at %s" % (what, (~eq).sum(), eq.size, np.argwhere(~eq)[0])


# small and odd planes (every element checked), then the LitePose-S depthwise shapes (stage 0 at 512^2 and 256^2
# inputs, stages 1 - 3, batch 16 and 32; a sample of planes / channels checked) and N * C beyond one grid row
SMALL = [(2, 3, 131, 37), (3, 5, 4, 3), (1, 7, 1, 1), (2, 4, 33, 65)]
LITEPOSE = [(32, 96, 256, 256), (16, 96, 128, 128), (32, 192, 64, 64), (16, 288, 32, 32), (32, 720, 16, 16),
            (16, 96, 64, 64)]
WIDE = (2, 40000, 3, 5)
COMBOS = [(k, s, dt) for k in (3, 5, 7) for s in (1, 2) for dt in (torch.float32, torch.float16)]


def _check_all(n, c, h, w, k, s, dt, seed, planes=None, channels=None):
    x, wt, dy = _inputs(n, c, h, w, k, s, dt, seed)
    y, dx, dw = kfwd(x, wt, s), kdgrad(dy, wt, s, h, w), kwgrad(x, dy, k, s)
    what = "k%d s%d %s %s" % (k, s, dt, (n, c, h, w))
    xn, wn, dn = x.cpu().numpy(), wt.cpu().numpy(), dy.cpu().numpy()
    if planes is None:
        _same(y, dte.fwd(xn, wn, s), "fwd " + what)
        _same(dx, dte.dgrad(dn, wn, s, h, w), "dgrad " + what)
        _same(dw, dte.wgrad(xn, dn, k, s), "wgrad " + what)
        return
    for (i, j) in planes:             # one (n, c) plane: it depends on x[i, j], dy[i, j] and w[j] only
        _same(y[i:i + 1, j:j + 1], dte.fwd(xn[i:i + 1, j:j + 1], wn[j:j + 1], s), "fwd %s plane %s" % (what, (i, j)))
        _same(dx[i:i + 1, j:j + 1], dte.dgrad(dn[i:i + 1, j:j + 1], wn[j:j + 1], s, h, w),
              "dgrad %s plane %s" % (what, (i, j)))
    for j in channels:                # one channel's weight gradient: every image of that channel
        _same(dw[j:j + 1], dte.wgrad(xn[:, j:j + 1], dn[:, j:j + 1], k, s), "wgrad %s channel %d" % (what, j))


@pytest.mark.parametrize("k,s,dt", COMBOS, ids=["k%d-s%d-%s" % (k, s, str(d)[6:]) for k, s, d in COMBOS])
def test_entry_points_equal_emulator(k, s, dt):
    for i, shape in enumerate(SMALL):
        _check_all(*shape, k, s, dt, 100 * k + 10 * s + i)
    ci = COMBOS.index((k, s, dt))
    n, c, h, w = LITEPOSE[ci % len(LITEPOSE)]
    _check_all(n, c, h, w, k, s, dt, ci, planes=[(0, 0), (n - 1, c - 1), (n // 2, c // 3)], channels=[0, c - 1])
    if ci % 4 == 0:
        n, c, h, w = WIDE
        _check_all(n, c, h, w, k, s, dt, ci, planes=[(0, 0), (1, 32767), (1, 39999)], channels=[0, 32768, 39999])


@pytest.mark.parametrize("k,s", [(3, 2), (5, 1), (7, 2), (7, 1)])
def test_fp16_is_fp32_rounded(k, s):
    x, wt, dy = _inputs(4, 24, 57, 70, k, s, torch.float16, k + s)
    up = [t.float() for t in (x, wt, dy)]
    assert torch.equal(kfwd(x, wt, s).view(torch.int16), kfwd(up[0], up[1], s).half().view(torch.int16))
    assert torch.equal(kdgrad(dy, wt, s, 57, 70).view(torch.int16), kdgrad(up[2], up[1], s, 57, 70).half().view(torch.int16))
    assert torch.equal(kwgrad(x, dy, k, s).view(torch.int16), kwgrad(up[0], up[2], k, s).half().view(torch.int16))


def test_same_bits_every_call_and_stream():
    n, c, h, w, k, s = 32, 96, 128, 128, 7, 1
    x, wt, dy = _inputs(n, c, h, w, k, s, torch.float32, 5)
    ref = [kfwd(x, wt, s), kdgrad(dy, wt, s, h, w), kwgrad(x, dy, k, s)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for rep in range(3):
        with torch.cuda.stream(side if rep == 2 else torch.cuda.current_stream()):
            got = [kfwd(x, wt, s), kdgrad(dy, wt, s, h, w), kwgrad(x, dy, k, s)]
        torch.cuda.synchronize()
        for a, b in zip(got, ref):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---------------------------------------------------------------- autograd
@pytest.mark.parametrize("k,s", [(3, 1), (5, 2), (7, 1), (7, 2)])
def test_autograd_within_bound_of_fp64(k, s):
    n, c, h, w = 3, 16, 45, 38
    x, wt, dy = _inputs(n, c, h, w, k, s, torch.float32, 11 * k + s)
    xr = x.clone().requires_grad_(True)
    wr = wt.reshape(c, 1, k, k).clone().requires_grad_(True)
    y = depthwise_conv2d(xr, wr, s)
    y.backward(dy)
    xn, wn, dn = x.cpu().numpy(), wt.cpu().numpy(), dy.cpu().numpy()
    ex = dte.exact_fwd(xn, wn, s)
    dx64, dw64 = dte.exact_grads(xn, wn, dn, s)
    for got, exact, bound, what in ((y, ex, dte.bound_fwd(xn, wn, s), "y"),
                                    (xr.grad, dx64, dte.bound_dgrad(xn, wn, dn, s), "dx"),
                                    (wr.grad.reshape(c, k, k), dw64, dte.bound_wgrad(xn, wn, dn, s), "dw")):
        err = np.abs(got.detach().double().cpu().numpy() - exact)
        assert (err <= bound).all(), (what, float((err - bound).max()))
    # and exactly the kernels
    _same(y.detach(), dte.fwd(xn, wn, s), "y")
    _same(xr.grad, dte.dgrad(dn, wn, s, h, w), "dx")
    _same(wr.grad.reshape(c, k, k), dte.wgrad(xn, dn, k, s), "dw")


def test_backward_launches_only_what_is_needed():
    lib = _lib.load()
    x, wt, dy = _inputs(2, 8, 20, 20, 5, 2, torch.float32, 3)
    w4 = wt.reshape(8, 1, 5, 5)
    for need_x, need_w, launches in ((True, False, 1), (False, True, 2), (True, True, 3)):
        xr, wr = x.clone().requires_grad_(need_x), w4.clone().requires_grad_(need_w)
        y = depthwise_conv2d(xr, wr, 2)
        torch.cuda.synchronize()
        before = lib.lp_launch_count()
        y.backward(dy)
        torch.cuda.synchronize()
        assert lib.lp_launch_count() - before == launches, (need_x, need_w)
        assert (xr.grad is not None) == need_x and (wr.grad is not None) == need_w
    y = depthwise_conv2d(x.requires_grad_(True), w4.requires_grad_(True), 2)
    g = torch.autograd.grad(y, (x,), dy, create_graph=True)[0]
    with pytest.raises(RuntimeError):
        g.sum().backward()                 # once_differentiable: no double backward


def test_non_contiguous_and_channels_last():
    x, wt, dy = _inputs(2, 12, 30, 26, 7, 1, torch.float32, 9)
    base_w = torch.randn(24, 1, 9, 9, device="cuda")
    w_sl = base_w[::2, :, 1:8, 1:8].clone().requires_grad_(False)
    xs = x.transpose(2, 3).contiguous().transpose(2, 3).requires_grad_(True)   # same values, column-major planes
    wb = base_w.clone().requires_grad_(True)
    w_view = wb[::2, :, 1:8, 1:8]
    assert not xs.is_contiguous() and not w_view.is_contiguous()
    y = depthwise_conv2d(xs, w_view, 1)
    assert y.is_contiguous()
    _same(y.detach(), dte.fwd(x.cpu().numpy(), w_sl.cpu().numpy(), 1), "y")
    y.backward(dy.transpose(2, 3).contiguous().transpose(2, 3))
    _same(xs.grad, dte.dgrad(dy.cpu().numpy(), w_sl.cpu().numpy(), 1, 30, 26), "dx")
    gw = wb.grad[::2, :, 1:8, 1:8].reshape(12, 7, 7)
    _same(gw, dte.wgrad(x.cpu().numpy(), dy.cpu().numpy(), 7, 1), "dw through the slice")
    assert wb.grad[1::2].abs().sum() == 0 and wb.grad[:, :, 0].abs().sum() == 0
    xc = x.to(memory_format=torch.channels_last)
    yc = depthwise_conv2d(xc, w_sl, 1)
    assert yc.is_contiguous() and torch.equal(yc, y.detach())


def test_autocast_and_half_modules():
    x, wt, dy = _inputs(2, 16, 24, 24, 5, 1, torch.float32, 2)
    m = convert_depthwise(nn.Conv2d(16, 16, 5, 1, 2, groups=16, bias=False)).cuda()
    m.weight.data.copy_(wt.reshape(16, 1, 5, 5))
    xr = x.clone().requires_grad_(True)
    with torch.autocast("cuda", torch.float16):
        y = m(xr)
    assert y.dtype == torch.float16
    assert torch.equal(y, kfwd(x.half(), wt.half(), 1))
    y.backward(dy.half())
    assert xr.grad.dtype == torch.float32 and m.weight.grad.dtype == torch.float32
    assert torch.equal(xr.grad, kdgrad(dy.half(), wt.half(), 1, 24, 24).float())
    assert torch.equal(m.weight.grad.reshape(16, 5, 5), kwgrad(x.half(), dy.half(), 5, 1).float())
    # network_to_half: an fp16 model and fp16 input run the fp16 kernels
    mh = copy.deepcopy(m).half()
    assert torch.equal(mh(x.half()), kfwd(x.half(), wt.half(), 1))


def test_dtype_refusals():
    x = torch.randn(1, 4, 8, 8, device="cuda")
    w = torch.randn(4, 1, 3, 3, device="cuda")
    for xx, ww, msg in ((x.bfloat16(), w.bfloat16(), "bfloat16"), (x.double(), w.double(), "float64"),
                        (x.half(), w, "one dtype"), (x, w[:, :, :2, :2], "does not fit"),
                        (x, torch.randn(4, 1, 9, 9, device="cuda"), "does not fit")):
        with pytest.raises(ValueError, match=msg):
            depthwise_conv2d(xx, ww, 1)
    with pytest.raises(ValueError, match="stride"):
        depthwise_conv2d(x, w, 3)
    with torch.autocast("cuda", torch.bfloat16):
        with pytest.raises(ValueError, match="autocast"):
            depthwise_conv2d(x, w, 1)


# ---------------------------------------------------------------- whole training steps against fp64
LR = 1e-3
FLOOR = 1e-6          # of max |fp64 gradient| of the tensor: the fp32 rounding level a 0-distance cuDNN step can hide


def _train_step(model, x, seed, dt):
    random.seed(seed)
    model.zero_grad(set_to_none=True)
    outs = model(x.cuda().to(dt))
    wts = [torch.linspace(-1, 1, o.numel(), device="cuda", dtype=torch.float64).reshape(o.shape) for o in outs]
    loss = sum((o.double() * t).sum() for o, t in zip(outs, wts))
    loss.backward()
    opt = torch.optim.Adam(model.parameters(), lr=LR)
    grads = {n: p.grad.detach().double().clone() for n, p in model.named_parameters() if p.grad is not None}
    opt.step()
    return grads, {n: p.detach().double().clone() for n, p in model.named_parameters()}


def _compare_step(model, x, seed):
    m64 = copy.deepcopy(model).double().cuda().train()
    ref = copy.deepcopy(model).cuda().train()
    conv = convert_depthwise(copy.deepcopy(model)).cuda().train()
    g64, p64 = _train_step(m64, x, seed, torch.float64)
    gr, pr = _train_step(ref, x, seed, torch.float32)
    lib = _lib.load()
    before = lib.lp_launch_count()
    gc, pc = _train_step(conv, x, seed, torch.float32)
    assert lib.lp_launch_count() > before
    assert list(gc) == list(g64) == list(gr)
    worst = []
    for name in g64:
        scale = g64[name].abs().max().item()
        ec = (gc[name] - g64[name]).abs().max().item()
        er = (gr[name] - g64[name]).abs().max().item()
        lim = 2 * er + FLOOR * scale + 1e-30
        worst.append((ec / lim, name, ec, er, scale))
        assert ec <= lim, "%s: converted %.3e, cuDNN %.3e (max |g| %.3e)" % (name, ec, er, scale)
    for name in g64:
        # Adam's first step moves a parameter by lr * g / (|g| + eps): a gradient error dg moves it by at most
        # lr * min(2, 2 |dg| / (|g| + eps)) (the gradients' own bound is held above)
        lim = LR * torch.clamp(2 * (gc[name] - g64[name]).abs() / (g64[name].abs() + 1e-8), max=2) + 1e-7
        assert ((pc[name] - p64[name]).abs() <= lim).all(), "%s after Adam" % name
    return max(worst)


def test_train_step_litepose_s():
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_mobilenet.get_pose_net(get_cfg(input_size=256), False, get_arch("S")), 1)
    x = synth.make_frames(4, 256, seed=1)
    _compare_step(model, x, 0)


def test_train_step_supernet_random_sample():
    """a random_sample() architecture (the sampler draws k = 7 only) with some blocks set to k = 5 and 3, as searched
    candidates have them: both functional call sites, the 7x7 slice and its Linear5x5 / Linear3x3 transforms"""
    cfg = get_cfg(input_size=256)
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_supermobilenet.get_pose_net(cfg), 1)
    random.seed(4)
    arch = model.arch_manager.random_sample()
    for si, st in enumerate(arch["backbone_setting"]):
        for bi in range(st["num_blocks"]):
            st["block_setting"][bi] = [6, (7, 5, 3)[(si + bi) % 3]]
    model.arch_manager.is_search, model.arch_manager.search_arch = True, arch
    x = synth.make_frames(2, 256, seed=2)
    _compare_step(model, x, 0)


def test_eval_after_conversion_runs_the_engine_unchanged():
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_mobilenet.get_pose_net(get_cfg(input_size=128), False, get_arch("XS")), 1)
    ref = copy.deepcopy(model).cuda().eval()
    conv = convert_depthwise(copy.deepcopy(model)).cuda().eval()
    x = synth.make_frames(2, 128, seed=4).cuda()
    with torch.no_grad():
        for a, b in zip(ref(x), conv(x)):
            assert torch.equal(a, b)
        for a, b in zip(ref(x.half()), conv(x.half())):
            assert torch.equal(a, b)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_data_parallel_two_gpus():
    torch.manual_seed(0)
    model = synth.randomize_bn_(pose_mobilenet.get_pose_net(get_cfg(input_size=128), False, get_arch("XS")), 1)
    dp = nn.DataParallel(convert_depthwise(copy.deepcopy(model)).cuda().train(), device_ids=[0, 1])
    x = synth.make_frames(4, 128, seed=6).cuda()
    outs = dp(x)
    sum(o.sum() for o in outs).backward()
    for n, p in dp.module.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    assert all(type(m) is DepthwiseConv2d for n, m in dp.module.named_modules() if isinstance(m, nn.Conv2d) and m.groups > 1)
