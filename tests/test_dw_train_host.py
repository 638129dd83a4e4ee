"""CPU: the NCHW depthwise training kernels' restatement (dw_train_emul) against fp64 F.conv2d within its stated bound,
the C ABI's host-side checks, and convert_depthwise on the drop-in models: exactly the depthwise convs converted, the
same Parameter objects and state dict, and CPU train-mode forward / backward bit-identical to the unconverted module."""
import copy
import pickle
import random

import numpy as np
import pytest
import torch
import torch.nn as nn

import dw_train_emul as dte
from litepose_b200 import _lib, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models import pose_mobilenet, pose_simplenet, pose_supermobilenet
from litepose_b200.train_dw import DepthwiseConv2d, convert_depthwise, depthwise_conv2d, is_eligible

# odd sizes, H or W below k, 1 x 1 planes, a plane taller than one wgrad range with a ragged column tile
SHAPES = [(2, 3, 9, 11), (1, 2, 4, 3), (2, 2, 1, 1), (1, 2, 2, 6), (1, 1, 131, 37)]


def _inputs(n, c, h, w, k, s, seed, dt=np.float32):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, c, h, w)).astype(dt)
    wt = (rng.standard_normal((c, k, k)) / k).astype(dt)
    dy = rng.standard_normal((n, c, dte.out_size(h, s), dte.out_size(w, s))).astype(dt)
    return x, wt, dy


def _within(got, exact, bound, what):
    err = np.abs(got.astype(np.float64) - exact)
    assert np.all(err <= bound), "%s: max excess %.3e" % (what, float(np.max(err - bound)))


@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
@pytest.mark.parametrize("s", [1, 2])
@pytest.mark.parametrize("k", [3, 5, 7])
def test_emulator_within_bound_of_fp64(k, s, fp16):
    dt = np.float16 if fp16 else np.float32
    for i, (n, c, h, w) in enumerate(SHAPES):
        x, wt, dy = _inputs(n, c, h, w, k, s, 10 * k + s + i, dt)
        what = "k%d s%d %s %s" % (k, s, dt.__name__, (n, c, h, w))
        y = dte.fwd(x, wt, s)
        assert y.dtype == dt and y.shape == dy.shape
        _within(y, dte.exact_fwd(x, wt, s), dte.bound_fwd(x, wt, s, fp16), "fwd " + what)
        dx64, dw64 = dte.exact_grads(x, wt, dy, s)
        dx = dte.dgrad(dy, wt, s, h, w)
        assert dx.dtype == dt and dx.shape == x.shape
        _within(dx, dx64, dte.bound_dgrad(x, wt, dy, s, fp16), "dgrad " + what)
        dw = dte.wgrad(x, dy, k, s)
        assert dw.dtype == dt and dw.shape == wt.shape
        _within(dw, dw64, dte.bound_wgrad(x, wt, dy, s, fp16), "wgrad " + what)


def test_emulator_fp16_is_fp32_rounded():
    """the fp16 results are the fp32 results on the up-converted inputs, rounded once to fp16"""
    for k, s in ((3, 2), (7, 1)):
        x, wt, dy = _inputs(2, 3, 9, 11, k, s, 3, np.float16)
        up = [a.astype(np.float32) for a in (x, wt, dy)]
        assert np.array_equal(dte.fwd(x, wt, s), dte.fwd(up[0], up[1], s).astype(np.float16))
        assert np.array_equal(dte.dgrad(dy, wt, s, 9, 11), dte.dgrad(up[2], up[1], s, 9, 11).astype(np.float16))
        assert np.array_equal(dte.wgrad(x, dy, k, s), dte.wgrad(up[0], up[2], k, s).astype(np.float16))


def test_emulator_padding_taps_multiply_the_weight():
    """a padding tap is a +0 input: an inf weight makes the border outputs NaN, as F.conv2d's zero padding does"""
    x, wt, _ = _inputs(1, 1, 6, 6, 3, 1, 4)
    wt[0, 0, 0] = np.inf
    with np.errstate(invalid="ignore"):
        y = dte.fwd(x, wt, 1)
    assert np.isnan(y[0, 0, 0, 0]) and np.isnan(y[0, 0, 0, 3]) and not np.isnan(y[0, 0, 3, 3])


def test_wgrad_ranges_depend_on_the_shape_only():
    lib = _lib.load()
    # 32 x 96 x 256^2 at stride 2: Ho = Wo = 128, one range down and four across per image
    assert lib.lp_dw_nchw_wgrad_workspace_bytes(32, 96, 256, 256, 7, 2) == 32 * 4 * 96 * 49 * 4
    assert dte.wgrad_partials(*_inputs(2, 1, 131, 37, 3, 1, 1)[::2], 3, 1).shape == (2 * 2 * 2, 1, 9)
    assert lib.lp_dw_nchw_wgrad_workspace_bytes(1, 8, 300, 65, 3, 1) == 1 * 3 * 3 * 8 * 9 * 4
    assert lib.lp_dw_nchw_wgrad_workspace_bytes(1, 8, 16, 16, 9, 1) == 0


def test_train_header_matches_binding_and_footprint_table():
    """every symbol include/litepose_b200_train.h declares is exported and bound (_lib.TRAIN_SIGNATURES), none is also
    in the inference header's table, and every launching one has a footprint case"""
    import os
    import re
    import dw_train_footprint_cases as tfc
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(root, "include", "litepose_b200_train.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(lp_[a-z0-9_]+)\s*\(", hdr))
    lib = _lib.load()
    assert declared == set(_lib.TRAIN_SIGNATURES) and len(declared) == 4
    assert all(hasattr(lib, s) for s in declared) and not declared & set(_lib.SIGNATURES)
    assert tfc.launching_symbols() == tfc.covered_symbols() == {"lp_dw_nchw_fwd", "lp_dw_nchw_dgrad",
                                                                "lp_dw_nchw_wgrad"}
    ids = [c.id for c in tfc.CASES]
    assert len(ids) == len(set(ids))


def test_entry_point_refusals():
    lib = _lib.load()
    assert lib.lp_dw_nchw_fwd(None, None, None, 1, 8, 16, 16, 9, 1, 0, None) == 1
    assert b"kernel size 9" in lib.lp_last_error()
    assert lib.lp_dw_nchw_dgrad(None, None, None, 1, 8, 16, 16, 3, 3, 0, None) == 1
    assert b"stride 3" in lib.lp_last_error()
    assert lib.lp_dw_nchw_wgrad(None, None, None, 1, 8, 16, 16, 3, 1, 2, None, 0, None) == 1
    assert b"dtype 2" in lib.lp_last_error()
    assert lib.lp_dw_nchw_fwd(None, None, None, 1, 8, 0, 16, 3, 1, 0, None) == 1
    # N * C == 0 launches nothing (and needs no pointers)
    assert lib.lp_dw_nchw_fwd(None, None, None, 0, 8, 16, 16, 3, 1, 0, None) == 0
    assert lib.lp_dw_nchw_dgrad(None, None, None, 4, 0, 16, 16, 5, 2, 1, None) == 0


def test_depthwise_conv2d_refuses_cpu_tensors():
    with pytest.raises(ValueError, match="CUDA tensors"):
        depthwise_conv2d(torch.zeros(1, 4, 8, 8), torch.zeros(4, 1, 3, 3))


def test_eligibility():
    ok = nn.Conv2d(8, 8, 7, 2, 3, groups=8, bias=False)
    assert is_eligible(ok)
    for bad in (nn.Conv2d(8, 8, 7, 2, 3, groups=8, bias=True), nn.Conv2d(8, 8, 3, 1, 1, groups=4, bias=False),
                nn.Conv2d(8, 16, 3, 1, 1, groups=8, bias=False), nn.Conv2d(8, 8, 9, 1, 4, groups=8, bias=False),
                nn.Conv2d(8, 8, 3, 3, 1, groups=8, bias=False), nn.Conv2d(8, 8, 3, 1, 2, 2, groups=8, bias=False),
                nn.Conv2d(8, 8, 3, 1, 0, groups=8, bias=False),
                nn.Conv2d(8, 8, 3, 1, 1, groups=8, bias=False, padding_mode="reflect"),
                nn.Conv2d(8, 8, (3, 5), 1, (1, 2), groups=8, bias=False), DepthwiseConv2d(8, 8, 3, 1, 1, groups=8,
                                                                                            bias=False)):
        assert not is_eligible(bad), bad
    assert type(convert_depthwise(ok)) is DepthwiseConv2d


# ---------------------------------------------------------------- the converter on the drop-in models
def _models():
    torch.manual_seed(0)
    yield "S", pose_mobilenet.get_pose_net(get_cfg(input_size=448), False, get_arch("S")), 1 + 34 + 4
    torch.manual_seed(0)
    yield "XS", pose_mobilenet.get_pose_net(get_cfg(input_size=256), False, get_arch("XS")), 1 + 34 + 4
    torch.manual_seed(0)
    yield "simplenet", pose_simplenet.get_pose_net(get_cfg(input_size=256), False, get_arch("XS")), 1 + 34 + 2
    torch.manual_seed(0)
    yield "supernet", pose_supermobilenet.get_pose_net(get_cfg(input_size=256)), 1 + 34 + 4


MODELS = list(_models())


def _depthwise_names(model):
    return sorted(n for n, m in model.named_modules() if isinstance(m, nn.Conv2d) and m.groups > 1)


@pytest.mark.parametrize("name,model,count", MODELS, ids=[m[0] for m in MODELS])
def test_convert_exactly_the_depthwise_convs(name, model, count):
    model = copy.deepcopy(model)
    before = dict(model.named_parameters())
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    want = _depthwise_names(model)
    assert convert_depthwise(model) is model
    got = sorted(n for n, m in model.named_modules() if type(m) is DepthwiseConv2d)
    assert got == want and len(got) == count, (len(got), count)
    assert all(isinstance(m, nn.Conv2d) for n, m in model.named_modules() if n in got)
    after = dict(model.named_parameters())
    assert list(after) == list(before) and all(after[k] is before[k] for k in before)
    sd2 = model.state_dict()
    assert list(sd2) == list(sd) and all(torch.equal(sd2[k], sd[k]) for k in sd)


def _step(model, x, seed):
    random.seed(seed)
    outs = model(x)
    loss = sum((o.float() * torch.linspace(-1, 1, o.numel()).reshape(o.shape)).sum() for o in outs)
    loss.backward()
    return [o.detach() for o in outs], {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("name,model,count", MODELS, ids=[m[0] for m in MODELS])
def test_cpu_train_step_unchanged(name, model, count):
    """the CPU path is the module tree: converted and unconverted give the same bits, forward and backward"""
    ref = synth.randomize_bn_(copy.deepcopy(model), 1).train()
    conv = convert_depthwise(copy.deepcopy(ref))
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1))
    o1, g1 = _step(ref, x, 7)
    o2, g2 = _step(conv, x, 7)
    assert all(torch.equal(a, b) for a, b in zip(o1, o2)) and len(o1) == len(o2) == 2
    assert list(g1) == list(g2) and all(torch.equal(g1[k], g2[k]) for k in g1)
    for n, m in conv.named_modules():     # the running statistics moved the same way
        if isinstance(m, nn.BatchNorm2d):
            r = ref.get_submodule(n)
            assert torch.equal(m.running_mean, r.running_mean) and torch.equal(m.running_var, r.running_var)


def test_deepcopy_and_pickle_keep_the_conversion():
    model = convert_depthwise(copy.deepcopy(MODELS[3][1]))
    for twin in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
        kinds = [(n, type(m)) for n, m in twin.named_modules()]
        assert kinds == [(n, type(m)) for n, m in model.named_modules()]
        sd, sd2 = model.state_dict(), twin.state_dict()
        assert all(torch.equal(sd[k], sd2[k]) for k in sd)
