"""CPU: the NCHW train-mode BatchNorm kernels' restatement (bn_nchw_train_emul) against fp64 within its stated bound, the
C ABI's host-side checks and its agreement with the header and the footprint table, and convert_batchnorm on the
drop-in models: exactly the eligible BatchNorms and the activations that follow them converted, the same Parameter
objects, state dict and isinstance, and every activation applied once on the paths that do not run the kernels."""
import copy
import os
import pickle
import random
import re

import numpy as np
import pytest
import torch
import torch.nn as nn

import bn_nchw_train_emul as bte
from litepose_b200 import _lib, synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models import pose_mobilenet, pose_simplenet, pose_supermobilenet
from litepose_b200.lib.models.pose_supermobilenet import SuperBatchNorm2d
from litepose_b200.train_bn import (ACT_NONE, ACT_RELU, ACT_RELU6, BatchNormAct2d, FusedReLU, FusedReLU6,
                                    SuperBatchNormAct2d, batch_norm_act, convert_batchnorm, is_eligible)

ACTS = [ACT_NONE, ACT_RELU, ACT_RELU6]
# odd planes, 1 x 1 planes, a channel past one reduction range (8192 values) with a ragged last range, H*W < 256
SHAPES = [(2, 3, 9, 11), (5, 2, 1, 1), (3, 2, 61, 53), (16, 3, 7, 7)]


def _inputs(n, c, h, w, seed, dt=np.float32):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((n, c, h, w)) * 2 + rng.standard_normal((1, c, 1, 1))).astype(dt)
    gamma = rng.uniform(0.5, 1.5, c).astype(np.float32)
    beta = (rng.standard_normal(c) * 0.5).astype(np.float32)
    rm = (rng.standard_normal(c) * 0.1).astype(np.float32)
    rv = rng.uniform(0.75, 1.25, c).astype(np.float32)
    dy = rng.standard_normal((n, c, h, w)).astype(dt)
    return x, gamma, beta, rm, rv, dy


def _within(got, exact, bound, what):
    err = np.abs(np.asarray(got, np.float64) - exact)
    assert np.all(err <= bound), "%s: max excess %.3e" % (what, float(np.max(err - bound)))


@pytest.mark.parametrize("fp16", [False, True], ids=["fp32", "fp16"])
@pytest.mark.parametrize("act", ACTS, ids=["none", "relu", "relu6"])
def test_emulator_within_bound_of_fp64(act, fp16):
    dt = np.float16 if fp16 else np.float32
    for i, (n, c, h, w) in enumerate(SHAPES):
        x, gamma, beta, rm, rv, dy = _inputs(n, c, h, w, 10 * act + i, dt)
        what = "act %d %s %s" % (act, dt.__name__, (n, c, h, w))
        y, saved, nm, nv = bte.fwd(x, gamma, beta, rm, rv, 0.1, 1e-5, act)
        assert y.dtype == dt and y.shape == x.shape and saved.shape == (4, c)
        ex, mean, var_u, _ = bte.exact_fwd(x, gamma, beta, 1e-5, act)
        _within(y, ex, bte.bound_fwd(x, gamma, beta, 1e-5, fp16), "y " + what)
        _within(nm, 0.9 * rm.astype(np.float64) + 0.1 * mean, 1e-6 * (np.abs(rm) + np.abs(mean)), "mean " + what)
        _within(nv, 0.9 * rv.astype(np.float64) + 0.1 * var_u, 1e-6 * (np.abs(rv) + var_u), "var " + what)
        dx, dg, db = bte.bwd(x, dy, gamma, saved, act)
        assert dx.dtype == dt and dg.dtype == db.dtype == np.float32
        dx64, dg64, db64 = bte.exact_bwd(x, dy, gamma, 1e-5, saved, act)
        ldx, ldg, ldb = bte.bound_bwd(x, dy, gamma, 1e-5, saved, act, fp16)
        _within(dx, dx64, ldx, "dx " + what)
        _within(dg, dg64, ldg, "dgamma " + what)
        _within(db, db64, ldb, "dbeta " + what)


def test_emulator_fp16_is_fp32_rounded():
    """an fp16 call is the fp32 call on the up-converted inputs, its x-shaped results rounded once to fp16"""
    x, gamma, beta, rm, rv, dy = _inputs(3, 4, 13, 17, 3, np.float16)
    for act in ACTS:
        y16, s16, m16, v16 = bte.fwd(x, gamma, beta, rm, rv, 0.1, 1e-5, act)
        y32, s32, m32, v32 = bte.fwd(x.astype(np.float32), gamma, beta, rm, rv, 0.1, 1e-5, act)
        assert np.array_equal(y16, y32.astype(np.float16)) and np.array_equal(s16, s32)
        assert np.array_equal(m16, m32) and np.array_equal(v16, v32)
        b16, b32 = bte.bwd(x, dy, gamma, s16, act), bte.bwd(x.astype(np.float32), dy.astype(np.float32), gamma, s32, act)
        assert np.array_equal(b16[0], b32[0].astype(np.float16))
        assert np.array_equal(b16[1], b32[1]) and np.array_equal(b16[2], b32[2])


def test_emulator_nan_and_masked_gradients():
    """NaN passes the activation; a NaN gradient where the mask is 0 contributes +0, as threshold_backward selects it"""
    x, gamma, beta, rm, rv, dy = _inputs(2, 2, 5, 5, 4)
    y, saved, _, _ = bte.fwd(x, gamma, beta, rm, rv, 0.1, 1e-5, ACT_RELU)
    v = bte.act_fn(np.nan, ACT_RELU6)
    assert np.isnan(v) and bte.act_fn(np.inf, ACT_RELU6) == 6 and bte.act_fn(-np.inf, ACT_RELU) == 0
    off = np.argwhere(y == 0)[0]
    dy[tuple(off)] = np.nan
    dx, dg, db = bte.bwd(x, dy, gamma, saved, ACT_RELU)
    assert np.isfinite(dx).all() and np.isfinite(dg).all() and np.isfinite(db).all()
    dx, dg, db = bte.bwd(x, dy, gamma, saved, ACT_NONE)
    assert np.isnan(dx[:, off[1]]).all() and np.isnan(db[off[1]]) and not np.isnan(db[1 - off[1]])


def test_workspace_depends_on_the_shape_only():
    lib = _lib.load()
    for n, c, h, w in SHAPES + [(16, 96, 224, 224), (16, 720, 14, 14)]:
        assert lib.lp_bn_nchw_workspace_bytes(n, c, h, w) == bte.workspace_bytes(n, c, h, w)
    assert bte.nparts(16, 224, 224) == 98 and bte.nparts(3, 61, 53) == 2
    assert lib.lp_bn_nchw_workspace_bytes(1, 8, 1, 1) == 0          # one value per channel
    assert lib.lp_bn_nchw_workspace_bytes(1, 8, 0, 4) == 0


def test_train_bn_header_matches_binding_and_footprint_table():
    """every symbol include/litepose_b200_train_bn.h declares is exported and bound (_lib.TRAIN_BN_SIGNATURES), none is
    also in the other two tables, and every launching one has a footprint case"""
    import bn_nchw_train_footprint_cases as bfc
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(root, "include", "litepose_b200_train_bn.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(lp_[a-z0-9_]+)\s*\(", hdr))
    lib = _lib.load()
    assert declared == set(_lib.TRAIN_BN_SIGNATURES) and len(declared) == 3
    assert all(hasattr(lib, s) for s in declared)
    assert not declared & set(_lib.SIGNATURES) and not declared & set(_lib.TRAIN_SIGNATURES)
    assert bfc.launching_symbols() == bfc.covered_symbols() == {"lp_bn_nchw_fwd", "lp_bn_nchw_bwd"}
    ids = [c.id for c in bfc.CASES]
    assert len(ids) == len(set(ids))


def test_entry_point_refusals():
    lib = _lib.load()
    fwd, bwd = lib.lp_bn_nchw_fwd, lib.lp_bn_nchw_bwd
    assert fwd(None, None, None, None, None, 0.1, 1e-5, None, None, 2, 8, 4, 4, 0, 2, None, 0, None) == 1
    assert b"dtype 2" in lib.lp_last_error()
    assert fwd(None, None, None, None, None, 0.1, 1e-5, None, None, 2, 8, 4, 4, 3, 0, None, 0, None) == 1
    assert b"act 3" in lib.lp_last_error()
    assert fwd(None, None, None, None, None, 0.1, 1e-5, None, None, 1, 8, 1, 1, 0, 0, None, 0, None) == 1
    assert b"one value per channel" in lib.lp_last_error()
    assert fwd(None, None, None, None, None, 0.1, 1e-5, None, None, 2, 8, 0, 4, 0, 0, None, 0, None) == 1
    assert b"bad shape" in lib.lp_last_error()
    assert fwd(None, None, None, None, None, 1.5, 1e-5, None, None, 2, 8, 4, 4, 0, 0, None, 0, None) == 1
    assert b"momentum" in lib.lp_last_error()
    assert fwd(None, None, None, None, None, 0.1, 1e-5, None, None, 2, 8, 4, 4, 0, 0, None, 0, None) == 1
    assert b"null pointer" in lib.lp_last_error()
    assert bwd(None, None, None, None, None, None, None, 2, 8, 4, 4, 0, 1, None, 0, None) == 0   # nothing wanted
    assert bwd(None, None, None, None, 8, None, None, 2, 8, 4, 4, 0, 1, None, 0, None) == 1
    assert b"null pointer" in lib.lp_last_error()
    # C == 0 launches nothing and needs no pointers
    assert fwd(None, None, None, None, None, 0.1, 1e-5, None, None, 2, 0, 4, 4, 0, 0, None, 0, None) == 0
    # workspace capacity and alignment, checked before anything is launched (host pointers are never dereferenced)
    p = 4096
    assert fwd(p, p, p, p, p, 0.1, 1e-5, p, p, 2, 8, 4, 4, 0, 0, p, 16, None) == 5
    assert b"workspace of 16 bytes" in lib.lp_last_error()
    assert fwd(p, p, p, p, p, 0.1, 1e-5, p, p, 2, 8, 4, 4, 0, 0, p + 4, 1 << 20, None) == 2
    assert fwd(p + 2, p, p, p, p, 0.1, 1e-5, p, p, 2, 8, 4, 4, 0, 0, p, 1 << 20, None) == 2
    assert b"aligned" in lib.lp_last_error()


def test_batch_norm_act_refuses_cpu_tensors():
    x, w = torch.zeros(2, 4, 3, 3), torch.ones(4)
    with pytest.raises(ValueError, match="CUDA tensor"):
        batch_norm_act(x, w, torch.zeros(4), torch.zeros(4), torch.ones(4), 0.1, 1e-5, ACT_RELU)


def test_eligibility():
    assert is_eligible(nn.BatchNorm2d(8)) and is_eligible(SuperBatchNorm2d(8))
    for bad in (nn.BatchNorm2d(8, affine=False), nn.BatchNorm2d(8, track_running_stats=False),
                nn.BatchNorm2d(8, momentum=None), nn.SyncBatchNorm(8), nn.BatchNorm1d(8), BatchNormAct2d(8)):
        assert not is_eligible(bad), bad
    seq = convert_batchnorm(nn.Sequential(nn.BatchNorm2d(8), nn.ReLU6(), nn.BatchNorm2d(8, momentum=None), nn.ReLU(),
                                          nn.BatchNorm2d(8), nn.Identity(), nn.ReLU()))
    assert [type(m) for m in seq] == [BatchNormAct2d, FusedReLU6, nn.BatchNorm2d, nn.ReLU, BatchNormAct2d, nn.Identity,
                                      nn.ReLU]
    assert seq[0].lp_act == ACT_RELU6 and seq[4].lp_act == ACT_NONE
    assert convert_batchnorm(seq) is seq and seq[0].lp_act == ACT_RELU6      # idempotent


# ---------------------------------------------------------------- the converter on the drop-in models
def _models():
    torch.manual_seed(0)
    yield "S", pose_mobilenet.get_pose_net(get_cfg(input_size=448), False, get_arch("S"))
    torch.manual_seed(0)
    yield "XS", pose_mobilenet.get_pose_net(get_cfg(input_size=256), False, get_arch("XS"))
    torch.manual_seed(0)
    yield "simplenet", pose_simplenet.get_pose_net(get_cfg(input_size=256), False, get_arch("XS"))
    torch.manual_seed(0)
    yield "supernet", pose_supermobilenet.get_pose_net(get_cfg(input_size=256))


MODELS = list(_models())


def _bn_act_pairs(model):
    """(BatchNorm name, the activation type that directly follows it in its nn.Sequential, or None)"""
    out = {}
    for sn, seq in model.named_modules():
        if isinstance(seq, nn.Sequential):
            kids = list(seq.named_children())
            for i, (cn, m) in enumerate(kids):
                if isinstance(m, nn.BatchNorm2d):
                    nxt = kids[i + 1][1] if i + 1 < len(kids) else None
                    out[(sn + "." if sn else "") + cn] = type(nxt) if type(nxt) in (nn.ReLU, nn.ReLU6) else None
    return out


def test_litepose_s_counts():
    """LitePose-S: 112 BatchNorms, 70 followed by a ReLU6 and 7 by a ReLU"""
    pairs = _bn_act_pairs(MODELS[0][1])
    kinds = list(pairs.values())
    assert len(kinds) == 112 and kinds.count(nn.ReLU6) == 70 and kinds.count(nn.ReLU) == 7


@pytest.mark.parametrize("name,model", MODELS, ids=[m[0] for m in MODELS])
def test_convert_exactly_the_batchnorms(name, model):
    model = copy.deepcopy(model)
    pairs = _bn_act_pairs(model)
    before = dict(model.named_parameters())
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    kinds = {n: type(m) for n, m in model.named_modules()}
    assert convert_batchnorm(model) is model
    mods = dict(model.named_modules())
    assert sorted(n for n, m in mods.items() if isinstance(m, (BatchNormAct2d, SuperBatchNormAct2d))) == sorted(pairs)
    for n, act in pairs.items():
        m = mods[n]
        assert type(m) is {nn.BatchNorm2d: BatchNormAct2d, SuperBatchNorm2d: SuperBatchNormAct2d}[kinds[n]]
        assert isinstance(m, kinds[n])
        assert m.lp_act == {None: ACT_NONE, nn.ReLU: ACT_RELU, nn.ReLU6: ACT_RELU6}[act]
    fused = [n for n, m in mods.items() if type(m) in (FusedReLU, FusedReLU6)]
    assert len(fused) == sum(a is not None for a in pairs.values())
    assert all(isinstance(mods[n], kinds[n]) for n in fused)
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


def _same_step(ref, conv, x):
    o1, g1 = _step(ref, x, 7)
    o2, g2 = _step(conv, x, 7)
    assert all(torch.equal(a, b) for a, b in zip(o1, o2)) and len(o1) == len(o2) == 2
    assert list(g1) == list(g2) and all(torch.equal(g1[k], g2[k]) for k in g1)
    sd1, sd2 = ref.state_dict(), conv.state_dict()
    assert all(torch.equal(sd1[k], sd2[k]) for k in sd1)      # running statistics and num_batches_tracked


@pytest.mark.parametrize("name,model", MODELS, ids=[m[0] for m in MODELS])
def test_cpu_train_step_unchanged(name, model):
    """the CPU path is the module tree with every activation applied once: converted and unconverted give the same
    bits, forward, backward and running statistics"""
    ref = synth.randomize_bn_(copy.deepcopy(model), 1).train()
    conv = convert_batchnorm(copy.deepcopy(ref))
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1))
    _same_step(ref, conv, x)


def test_activation_applied_after_the_batchnorm_is_replaced():
    """a converted BatchNorm swapped for a fresh module (as convert_sync_batchnorm swaps it): its activation applies"""
    ref = synth.randomize_bn_(copy.deepcopy(MODELS[1][1]), 1).train()
    conv = convert_batchnorm(copy.deepcopy(ref))
    for m in (ref, conv):
        for seq in (m.first[0], m.stage[0][0].inv, m.deconv_bnrelu[0]):
            bn = seq[1] if len(seq) > 2 else seq[0]
            fresh = nn.BatchNorm2d(bn.num_features)
            fresh.load_state_dict(bn.state_dict())
            seq[1 if len(seq) > 2 else 0] = fresh
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(3))
    _same_step(ref, conv, x)


def test_fused_activation_skips_only_an_unchanged_tagged_output():
    x = torch.linspace(-8, 8, 33)
    relu, relu6 = FusedReLU(), FusedReLU6()
    assert torch.equal(relu(x), torch.relu(x)) and torch.equal(relu6(x), torch.clamp(x, 0, 6))
    t = x.clone()
    t._lp_act = (ACT_RELU, t._version)
    assert relu(t) is t and torch.equal(relu6(t), torch.clamp(x, 0, 6))       # a ReLU output still needs the 6 cap
    t6 = x.clone()
    t6._lp_act = (ACT_RELU6, t6._version)
    assert relu(t6) is t6 and relu6(t6) is t6
    t6.add_(1)                                                                # changed in place: the tag is stale
    assert torch.equal(relu6(t6), torch.clamp(x + 1, 0, 6))


def test_eval_mode_uses_the_running_statistics():
    bn = synth.randomize_bn_(nn.Sequential(nn.BatchNorm2d(6), nn.ReLU6()), 2)
    ref = copy.deepcopy(bn).eval()
    conv = convert_batchnorm(copy.deepcopy(bn)).eval()
    x = torch.randn(3, 6, 5, 5) * 4
    assert torch.equal(ref(x), conv(x))


def test_re_organize_weights_on_a_converted_supernet():
    model = synth.randomize_bn_(copy.deepcopy(MODELS[3][1]), 4)
    conv = convert_batchnorm(copy.deepcopy(model))
    model.re_organize_weights()
    conv.re_organize_weights()
    sd1, sd2 = model.state_dict(), conv.state_dict()
    assert all(torch.equal(sd1[k], sd2[k]) for k in sd1)


def test_permute_bn_sees_through_the_conversion():
    bn = synth.randomize_bn_(nn.Sequential(nn.BatchNorm2d(4)), 5)[0]
    conv = convert_batchnorm(nn.Sequential(copy.deepcopy(bn)))[0]
    idx = torch.tensor([3, 1, 0, 2])
    for m in (bn, conv):
        pose_supermobilenet.SuperLitePose._permute_bn(m, idx)
    assert torch.equal(bn.running_mean, conv.running_mean) and torch.equal(bn.running_var, conv.running_var)
    assert not torch.equal(bn.running_mean, synth.randomize_bn_(nn.Sequential(nn.BatchNorm2d(4)), 5)[0].running_mean)


def test_deepcopy_and_pickle_keep_the_conversion():
    model = convert_batchnorm(copy.deepcopy(MODELS[3][1]))
    for twin in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
        kinds = [(n, type(m), getattr(m, "lp_act", None)) for n, m in twin.named_modules()]
        assert kinds == [(n, type(m), getattr(m, "lp_act", None)) for n, m in model.named_modules()]
