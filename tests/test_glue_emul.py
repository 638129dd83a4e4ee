"""CPU: the glue restatement (tests/glue_emul.py) checks itself before the GPU test holds the kernels to it: the exact
fp32 FMA against fractions.Fraction, every path against its float64 twin within the path's rounding bound, the
emulation against the reference's goldens, the x2 / x4 lambdas, and glue_path over the GPU case list."""
import hashlib
import os

import numpy as np
import pytest
import torch

import glue_emul as ge
from litepose_b200.config import flip_index_for, get_cfg


def test_fma32_matches_fraction_random():
    rng = np.random.default_rng(0)
    n = 4000
    e = rng.integers(-150, 40, (3, n))
    v = (np.sign(rng.standard_normal((3, n))) * rng.uniform(1, 2, (3, n)) * np.exp2(e)).astype(np.float32)
    v[:, :50] = np.float32(0.25)                          # the glue's constant weights
    v[1, 50:100] = np.float32(0.75)
    got = ge.fma32(v[0], v[1], v[2])
    for i in range(n):
        ref = ge.fma32_exact(v[0, i], v[1, i], v[2, i])
        assert got[i].view(np.uint32) == ref.view(np.uint32), (v[:, i], got[i], ref)


def test_fma32_midpoints_and_subnormals():
    """constructed cases: products that land exactly on an fp32 midpoint (tie to even), one ulp of the float64 sum
    beyond it (double rounding would tie the wrong way), subnormal results and signed zeros"""
    cases = []
    one = np.float32(1)
    u = np.float32(2.0 ** -24)
    for k in range(1, 40):
        a = np.float32(1 + k * 2.0 ** -23)
        cases += [(a, np.float32(0.75), np.float32(0)), (a, np.float32(0.75), u), (a, np.float32(0.75), -u),
                  (a, a, np.float32(-1)), (a, np.float32(0.25), np.float32(2.0 ** -60)),
                  (a, np.float32(0.75), np.float32(2.0 ** -80)), (a, np.float32(0.75), np.float32(-2.0 ** -80)),
                  (one + u * 2, one + u * 2, -one - u * 4)]
    for k in range(1, 30):
        s = np.float32(k * 2.0 ** -149)                   # subnormals
        cases += [(s, np.float32(0.75), np.float32(0)), (s, np.float32(0.25), s), (s, np.float32(0.75), -s),
                  (np.float32(2.0 ** -126), np.float32(0.75 + k * 2.0 ** -24), np.float32(-2.0 ** -127))]
    cases += [(np.float32(-0.0), np.float32(0.25), np.float32(-0.0)), (np.float32(-0.0), np.float32(0.75), np.float32(0)),
              (np.float32(1), np.float32(0), np.float32(-0.0)), (np.float32(-1), np.float32(0), np.float32(-0.0))]
    a, b, c = (np.array(x, np.float32) for x in zip(*cases))
    got = ge.fma32(a, b, c)
    ref = np.array([ge.fma32_exact(*x) for x in cases], np.float32)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    # the round-to-odd step is needed: rounding the float64 sum directly is wrong on some of these
    naive = (a.astype(np.float64) * b + c).astype(np.float32)
    assert not np.array_equal(naive.view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("n", [1, 2, 5, 16, 128])
def test_x2_x4_lambdas_are_quarters(n):
    """the fp32 lambdas of a x2 up-sample (lerp_coord with scale h / 2h, and the x2 projection H2 / 4h) are exactly
    0.25 / 0.75, and (1, 0) at the clamped first sample"""
    for scale in (ge._scale(n, 2 * n), ge._scale(2 * n, 4 * n)):
        i0, i1, l0, l1 = ge.lerp_coord(2 * n, scale, n)
        assert scale == np.float32(0.5)
        assert l0[0] == 1 and l1[0] == 0 and i0[0] == 0
        pairs = set(zip(l0[1:].tolist(), l1[1:].tolist()))
        assert pairs <= {(0.25, 0.75), (0.75, 0.25)}, pairs
        assert (i1 - i0 <= 1).all() and i1.max() <= n - 1


@pytest.mark.parametrize("case", ge.CASES, ids=[c["name"] for c in ge.CASES])
def test_emul_vs_f64_within_path_bound(case):
    """every path against the float64 glue, call by call, within k * 2^-24 * sum|terms| + k * 2^-149"""
    J, fidx = case["J"], ge.flip_index(case["J"])
    for kind in ("randn", "wide"):
        inputs = ge.case_inputs(case, kind, 3)
        det = None
        for (h, w, acc, div, wt), (o0, o1, f0, f1) in zip(case["calls"], inputs):
            prev = None if det is None else det.copy()
            kw = dict(Jm=case["Jm"], tag_shared=case["tag_shared"], accumulate=acc, divide_by=div, entry=case["entry"])
            det, tag = ge.glue(o0, o1, f0, f1, fidx, J, case["Hd"], case["Wd"], det=det, write_tag=wt, **kw)
            d64, t64 = ge.glue_f64(o0, o1, f0, f1, fidx, J, case["Hd"], case["Wd"], det_in=prev, has_tag=wt, **kw)
            bd, bt = ge.glue_bound(o0, o1, f0, f1, fidx, J, case["Hd"], case["Wd"], det_in=prev, has_tag=wt, **kw)
            err = np.abs(det.astype(np.float64) - d64)
            assert (err <= bd).all(), (kind, h, w, float((err / bd).max()))
            if wt:
                tg = tag if not case["tag_shared"] else np.repeat(tag, J, axis=1)[:, :1]
                t64 = t64 if not case["tag_shared"] else t64[:, :1]
                bt = bt if not case["tag_shared"] else bt[:, :1]
                assert (np.abs(tg.astype(np.float64) - t64) <= bt).all(), kind


def test_glue_path_reaches_every_branch():
    """the GPU case list reaches all four branches, and each case takes the branch its name starts with (ms cases:
    generic, plus unprojected for the largest scale without projection; quad_shared_tag: quad for joint 0 only)"""
    prefix = {"x4": "x4", "quad": "quad", "generic": "generic", "ms": "generic", "unproj": "unprojected"}
    seen = set()
    for c in ge.CASES:
        p = ge.case_paths(c)
        seen |= p
        assert prefix[c["name"].split("_")[0]] in p, (c["name"], p)
    assert seen == {"x4", "quad", "generic", "unprojected"}
    # selection details restated from glue_launch
    assert ge.glue_path(1, 14, 16, 16, 64, 64, entry="f32") == "x4"
    assert ge.glue_path(1, 14, 16, 16, 64, 64, accumulate=True) == "generic"
    assert ge.glue_path(1, 14, 16, 16, 64, 64, has_tag=False) == "generic"
    assert ge.glue_path(1, 14, 16, 16, 64, 64, Jm=15) == "quad"
    assert [ge.glue_path(1, 14, 16, 16, 64, 64, tag_shared=True, j=j) for j in (0, 1)] == ["quad", "generic"]
    assert ge.glue_path(4682, 14, 1, 1, 4, 4, entry="f32") == "quad"
    assert ge.glue_path(4681, 14, 1, 1, 4, 4, entry="f32") == "x4"
    assert ge.glue_path(1, 14, 16, 16, 32, 32) == "unprojected"
    assert ge.glue_tile_side(370, 370, 160, 160) == 8
    with pytest.raises(ValueError):
        ge.glue_path(1, 14, 371, 16, 160, 64)


# ---------------------------------------------------------------- against the reference's own outputs
def _check_golden(det, tag, z, name, stats):
    """the glue tests' tolerance, and the largest error in ulps of max|ref| (np.spacing of the largest output)"""
    ed, et = z["final_heatmaps"], z["tags"]
    assert det.shape == ed.shape and tag.shape == et.shape, name
    assert np.abs(det - ed).max() <= 1e-5 * max(1.0, np.abs(ed).max()), name
    assert np.abs(tag - et).max() <= 1e-5 * max(1.0, np.abs(et).max()), name
    stats[name] = tuple(float(np.abs(a - e).max() / np.spacing(np.float32(np.abs(e).max()))) for a, e in
                        ((det, ed), (tag, et)))


def test_emul_vs_reference_goldens(golden_dir):
    """the emulation against the unmodified reference's glue (oracle/make_golden.py) within the tolerance the GPU
    glue tests use.  Measured largest error in ulps of max|ref| (det, tag): flip1_proj1 (x4) 1.5, 2; flip0_proj1
    (generic) 1, 1.5; flip1_proj0 (unprojected) 1.5, 1; ms_1_2_proj1 1, 2; ms_05_1_proj0 1, 1.5; cfg center_ignored
    (quad) 1.5, 2; center_kept (x4) 1.25, 2; shared_tag (quad + generic) 2, 2; shared_tag_noproj (unprojected) 1, 1.
    Element-wise ulp distances are larger (tens of ulps) only on outputs far below max|ref|, where the two
    evaluation orders cancel differently."""
    from oracle.make_golden import (GLUE_CFG_CASES, GLUE_CFG_SIZE, MULTISCALE_CASES, FakeScaleModel, glue_cfg,
                                    multiscale_inputs)
    stats = {}
    for flip, proj in ((1, 1), (0, 1), (1, 0)):
        z = np.load(os.path.join(golden_dir, "glue_flip%d_proj%d.npz" % (flip, proj)))
        cfg = get_cfg(input_size=64, flip_test=bool(flip), project2image=bool(proj))
        n, j2, h, w = z["a0"].shape
        Hd, Wd = (64, 64) if proj else (2 * h, 2 * w)
        det, tag = ge.glue(z["a0"], z["a1"], z["b0"] if flip else None, z["b1"] if flip else None,
                           flip_index_for(cfg), j2 // 2, Hd, Wd, entry="f32")
        _check_golden(det, tag, z, "flip%d_proj%d" % (flip, proj), stats)
    for name, scales, proj, flip, size, seed in MULTISCALE_CASES:
        z = np.load(os.path.join(golden_dir, "glue_%s.npz" % name))
        cfg = get_cfg(input_size=size, flip_test=flip, project2image=proj)
        cfg.TEST.SCALE_FACTOR = list(scales)
        base, images = multiscale_inputs(cfg, size)
        fake = FakeScaleModel(cfg.DATASET.NUM_JOINTS, seed)
        order = sorted(scales, reverse=True)
        for s in order:
            for _ in range(2 if flip else 1):
                fake(images[s])
        dig = hashlib.sha256(b"".join(o.numpy().tobytes() for outs in fake.log for o in outs)).hexdigest()
        assert dig == str(z["in_digest"])
        first = images[order[0]]
        Hd, Wd = (base[1], base[0]) if proj else (first.shape[2] // 2, first.shape[3] // 2)
        det, tag = None, None
        per = 2 if flip else 1
        for i, s in enumerate(order):
            a, b = fake.log[i * per], fake.log[i * per + 1] if flip else [None, None]
            nn = lambda t: None if t is None else t.numpy()
            if s == 1 and tag is None:
                tag = np.full((a[0].shape[0], 14, Hd, Wd, 2 if flip else 1), np.nan, np.float32)
            det, _ = ge.glue(nn(a[0]), nn(a[1]), nn(b[0]), nn(b[1]), flip_index_for(cfg), 14, Hd, Wd,
                             accumulate=i > 0, divide_by=float(len(order)) if i == len(order) - 1 else 1.0,
                             det=det, tag=tag if s == 1 else None, write_tag=s == 1)
        _check_golden(det, tag, z, name, stats)
    for name, center, ignore, per_joint, proj, seed in GLUE_CFG_CASES:
        z = np.load(os.path.join(golden_dir, "glue_cfg_%s.npz" % name))
        cfg = glue_cfg(center, ignore, per_joint, proj)
        jm = cfg.DATASET.NUM_JOINTS
        fake = FakeScaleModel(jm, seed, None if per_joint else 1)
        img = torch.zeros(2, 3, GLUE_CFG_SIZE, GLUE_CFG_SIZE)
        a, b = [t.numpy() for t in fake(img)], [t.numpy() for t in fake(img)]
        J = z["final_heatmaps"].shape[1]
        Hd, Wd = z["final_heatmaps"].shape[2:]
        det, tag = ge.glue(a[0], a[1], b[0], b[1], flip_index_for(cfg), J, Hd, Wd, Jm=jm, tag_shared=not per_joint)
        _check_golden(det, tag, z, "cfg_" + name, stats)
    assert len(stats) == 9 and max(max(v) for v in stats.values()) <= 4, stats
