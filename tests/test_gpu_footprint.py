"""-m gpu: where the kernels read and write.  Every launching entry point runs on guarded buffers (footprint_util):
each tensor in its own allocation between 1 MiB guards, the payload 16 bytes past a 512-byte boundary (or at the
smallest alignment, or an odd element offset, the entry point documents), inputs flush against NaN / 0xA5 / 0x7F7F...
poison, outputs and their guards filled with a sentinel NaN.  After each call:
  (a) the outputs equal the reference of the entry point's own test (footprint_cases), bit for bit as values;
  (b) every guard byte of every buffer (inputs, weights, outputs, workspaces, descriptors) is unchanged;
  (c) every input payload byte is unchanged (in-place contracts are outputs with an initial payload);
  (d) no output element still holds the sentinel, except where the header promises "untouched" - there it survives;
  (e) the call returned LP_OK.
The detector self-tests show the harness sees a one-row / one-image overrun and a one-row / one-pixel over-read, all
well inside the guards.  The engine test runs whole LitePose plans with every buffer guarded and 16-byte skewed,
launched back to back as LitePoseEngine.run launches them."""
import json
import os

import numpy as np
import pytest
import torch

import dw_emul as de
import footprint_cases as fc
import mma_emul as me
from footprint_util import Guarded, Plain, compare
from litepose_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def default_dw_precision():
    _lib.load().lp_set_dw_precision(-1)
    yield
    _lib.load().lp_set_dw_precision(-1)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ok(rcs, what):
    assert all(rc == _lib.LP_OK for rc in rcs), "%s returned %s: %s" % (what, rcs, _lib.load().lp_last_error())


@pytest.mark.parametrize("case", fc.CASES, ids=[c.id for c in fc.CASES])
def test_footprint(case):
    _lib.load().lp_set_dw_precision(case.prec)
    g = Guarded()
    _ok(case.run(g), case.id)
    if case.ref is not None:
        want = case.ref()
    else:
        p = Plain()
        _ok(case.run(p), case.id + " (plain tensors)")
        want = p.outputs()
    errs = g.verify(want, case.untouched)
    assert not errs, "%s:\n  %s" % (case.id, "\n  ".join(errs))


# ---------------------------------------------------------------- the harness sees what it claims to see
def _pw_call(g, a, wt, b, m_call, out_rows):
    wp, bp = fc.pack_pw(wt, b)
    ad, wd, bd = g.inp("a", a), g.inp("w", wp), g.inp("bias", bp)
    out = g.out("out", (out_rows, wt.shape[0]), np.float16)
    return _lib.load().lp_pw1x1_f16(ad.data_ptr(), wd.data_ptr(), bd.data_ptr(), None, out.data_ptr(), m_call,
                                    a.shape[1], wt.shape[0], 0, _stream())


def test_detects_pw1x1_overrun():
    """M = rows + 1 against an output sized for rows: the extra row lands in the back guard"""
    rows = 129
    a, wt, b, _ = fc.pw_inputs(rows + 1, 72, 24, False, 5)
    g = Guarded()
    _ok([_pw_call(g, a, wt, b, rows + 1, rows)], "pw1x1")
    errs = g.verify({"out": me.pw1x1(a[:rows], wt, b)})
    assert any(e.startswith("out: back guard modified: %d bytes" % (24 * 2)) for e in errs), errs
    assert not [e for e in errs if not e.startswith("out: back guard")], errs


def test_detects_pw1x1_over_read():
    """an input one row shorter than the call reads: the poisoned neighbour shows up in the last output row"""
    rows = 129
    a, wt, b, _ = fc.pw_inputs(rows, 72, 24, False, 6)
    g = Guarded()
    _ok([_pw_call(g, a[:rows - 1], wt, b, rows, rows)], "pw1x1")
    errs = g.verify({"out": me.pw1x1(a, wt, b)})
    assert len(errs) == 1 and errs[0].startswith("out: 24 of %d elements differ" % (24 * rows)), errs
    assert "first at (%d, 0)" % (rows - 1) in errs[0], errs


def _dw_call(g, x, wt, b, n_call, n_out, hwc):
    h, w, c = hwc
    xd, wd, bd = g.inp("x", x), g.inp("w", wt), g.inp("bias", b)
    y = g.out("y", (n_out, h, w, c), np.float16)
    return _lib.load().lp_dwconv_f16(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), y.data_ptr(), n_call, c, h, w, 3, 1,
                                     de.ACT_NONE, _stream())          # no activation: a NaN is not clamped away


def test_detects_dwconv_overrun():
    """one more image than the output holds: that image lands in the back guard"""
    n, c, h, w = 2, 40, 9, 13
    x, wt, b = de.make_inputs(n + 1, c, h, w, 3, "signed", 8)
    g = Guarded()
    _ok([_dw_call(g, x, wt, b, n + 1, n, (h, w, c))], "dwconv")
    errs = g.verify({"y": de.dwconv(x[:n], wt, b, 3, 1, de.ACT_NONE, de.default_prec(3))})
    assert any(e.startswith("y: back guard modified") for e in errs), errs
    assert not [e for e in errs if not e.startswith("y: back guard")], errs


def test_detects_dwconv_over_read():
    """an input one pixel shorter than the call reads: NaN reaches the outputs whose window holds the last pixel"""
    n, c, h, w = 2, 40, 9, 13
    x, wt, b = de.make_inputs(n, c, h, w, 3, "signed", 9)
    g = Guarded()
    flat = x.reshape(-1)[:-c]                     # the last pixel of the last image is missing
    _ok([_dw_call(g, flat, wt, b, n, n, (h, w, c))], "dwconv")
    errs = g.verify({"y": de.dwconv(x, wt, b, 3, 1, de.ACT_NONE, de.default_prec(3))})
    assert len(errs) == 1 and "elements differ" in errs[0] and errs[0].startswith("y: "), errs
    assert "first at (1, 7, 11, 0)" in errs[0], errs     # the first output whose 3x3 window holds pixel (8, 12)


# ---------------------------------------------------------------- the engine's plan, every buffer guarded
def _nets():
    from litepose_b200 import engine, subnet, synth
    from litepose_b200.config import get_arch, get_cfg
    from litepose_b200.lib.models import pose_mobilenet, pose_simplenet, pose_supermobilenet
    torch.manual_seed(0)
    xs = synth.randomize_bn_(pose_mobilenet.get_pose_net(get_cfg(input_size=128), False, get_arch("XS")), 1)
    torch.manual_seed(0)
    sn = synth.randomize_bn_(pose_simplenet.get_pose_net(get_cfg(input_size=128), False, get_arch("XS")), 1)
    torch.manual_seed(0)
    sup = synth.randomize_bn_(pose_supermobilenet.get_pose_net(get_cfg(input_size=128)), 1)
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "model_supernet_random_seed1.npz"))
    sub = subnet.derive_supernet_subnet({k: v.detach() for k, v in sup.state_dict().items()}, json.loads(str(z["arch"])))
    return {
        "XS": lambda: engine.LitePoseEngine(xs.state_dict(), get_arch("XS"), "cuda"),
        "simplenet_XS": lambda: engine.LitePoseEngine(sn.state_dict(), get_arch("XS"), "cuda"),
        "supernet_seed1": lambda: engine.LitePoseEngine(sub.state_dict, sub.arch, "cuda", residual=sub.residual,
                                                        strides=sub.strides),
    }


_net_cache = {}


def _engine(name):
    if not _net_cache:
        _net_cache.update({k: None for k in ("XS", "simplenet_XS", "supernet_seed1")})
        _net_cache["_make"] = _nets()
    if _net_cache[name] is None:
        _net_cache[name] = _net_cache["_make"][name]()
    return _net_cache[name]


def _device_tensors(node, out):
    if torch.is_tensor(node):
        if node.is_cuda:
            out.append(node)
    elif isinstance(node, dict):
        for k in sorted(node, key=str):
            _device_tensors(node[k], out)
    elif isinstance(node, (list, tuple)):
        for v in node:
            _device_tensors(v, out)
    return out


# (net, n, h, w, input dtype, fp32 output, mirrored pass): 208 x 144 is ragged against the tiles at every level
ENGINE = [("XS", 2, 208, 144, "fp16", True, False), ("XS", 2, 208, 144, "fp32", False, True),
          ("XS", 1, 208, 144, "fp32", True, False), ("simplenet_XS", 2, 208, 144, "fp32", True, True),
          ("simplenet_XS", 2, 208, 144, "fp16", False, False), ("supernet_seed1", 2, 208, 144, "fp16", True, True),
          ("supernet_seed1", 1, 208, 144, "fp32", False, False)]


@pytest.mark.parametrize("net,n,h,w,dt,out_fp32,flip", ENGINE, ids=["-".join(map(str, c)) for c in ENGINE])
def test_engine_plan_guarded(net, n, h, w, dt, out_fp32, flip):
    from litepose_b200 import synth
    eng = _engine(net)
    tdt = torch.float16 if dt == "fp16" else torch.float32
    x = synth.make_frames(n, h, seed=h + w + n, width=w).to(tdt)
    want = [o.cpu().numpy() for o in eng.run(x.cuda(), flip=flip, out_fp32=out_fp32)]
    params = _device_tensors(eng.P, [])
    before = [p.cpu().numpy().tobytes() for p in params]

    g = Guarded()
    names = []

    def alloc(shape, dtype):
        names.append("buf%d" % len(names))
        return g.scratch(names[-1], tuple(shape), {torch.float16: np.float16, torch.float32: np.float32}[dtype])

    plan = eng._build_plan(n, h, w, tdt, out_fp32, alloc=alloc)
    xd = g.inp("x", x.numpy())
    plan["in_ptr"].value = xd.data_ptr()
    plan["flip"].value = 1 if flip else 0
    eng._launch_all(plan, _stream())                 # no synchronisation between the ops, as in run()
    errs = g.verify({})
    outs = [o.cpu().numpy() for o in plan["outs"]]
    for i, (got, ref) in enumerate(zip(outs, want)):
        assert got.dtype == ref.dtype and got.shape == ref.shape, (i, got.dtype, got.shape, ref.dtype, ref.shape)
        errs += compare("output %d" % i, got, ref)
    changed = [i for i, (p, b) in enumerate(zip(params, before)) if p.cpu().numpy().tobytes() != b]
    if changed:
        errs.append("engine.P: %d of %d device tensors modified (first: #%d, shape %s)"
                    % (len(changed), len(params), changed[0], tuple(params[changed[0]].shape)))
    assert len(outs) == len(want) == 2
    assert not errs, "%s:\n  %s" % (net, "\n  ".join(errs))
