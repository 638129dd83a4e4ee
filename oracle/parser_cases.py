"""ORACLE - TEST INFRASTRUCTURE ONLY.  Seeded, deterministic edge cases of the three parser stages (NMS + top-K, tag
matching, adjust + refine), shared by oracle/make_golden_parser_edges.py, tests/test_parser_edges_host.py and
tests/test_gpu_parser_edges.py.

* Matcher cases are top-K outputs built directly, inside the top-K contract (values descending, flat index ascending on
  ties, a zero tail with index 0, unique indices per plane), on tag lattices where round(dist) ties, exact .5 / 1.5 /
  2.5 distances, distances equal to TAG_THRESHOLD and tag[0] key collisions (-0.0 against +0.0 included) are common.
* Top-K cases are det / tag maps at the geometries where the strip kernel changes shape (strip height, vector or
  scalar path, bands, tall planes) with plateaus, ties on strip borders, NaN / inf / subnormal / -0.0 pixels.
* Refine cases are det / tag maps plus detected keypoints (``ans``) built directly: border keypoints, equal
  neighbours, equal refine scores in different 2048-pixel chunks, -0.0 against +0.0 scores, exact .5 distances,
  more than 32 persons missing a joint, T = 1..4, refine maxima whose value is <= 0 or NaN.
"""
import numpy as np

F = np.float32
ONE_TENTH = F(0.1)
BELOW_TENTH = np.nextafter(ONE_TENTH, F(0))             # one ulp below float32(0.1): dropped at threshold 0.1
VALS = [ONE_TENTH, BELOW_TENTH, F(0.25), F(0.3), F(0.5), F(0.75), F(1.0)]

_ORDER17 = [i - 1 for i in [1, 2, 3, 4, 5, 6, 7, 12, 13, 8, 9, 10, 11, 14, 15, 16, 17]]
_ORDER18 = [i - 1 for i in [18, 1, 2, 3, 4, 5, 6, 7, 12, 13, 8, 9, 10, 11, 14, 15, 16, 17]]
# joint count and joint order (lib/core/group.py Params): crowd_pose, COCO, WITH_CENTER kept, WITH_CENTER ignored
JOINTS = {"crowd_pose": (14, _ORDER17), "coco": (17, _ORDER17), "center_kept": (18, _ORDER18),
          "center_ignored": (17, _ORDER17)}


# ---------------------------------------------------------------------------------------------------- tag matching
def _plane(rs, cands, K, hw, T):
    """top-K slots of one joint plane from (val, tag) candidates: unique random indices, (val desc, index asc),
    the K best kept, zero tail with index 0 and tag 0."""
    val = np.zeros(K, F)
    ind = np.zeros(K, np.int32)
    tag = np.zeros((K, T), F)
    if not cands:
        return val, ind, tag
    v = np.array([c[0] for c in cands], F)
    t = np.array([c[1] for c in cands], F).reshape(len(cands), T)
    i = rs.choice(hw, size=len(cands), replace=False).astype(np.int32)
    order = np.lexsort((i, -v.astype(np.float64)))[:K]
    n = order.size
    val[:n], ind[:n], tag[:n] = v[order], i[order], t[order]
    return val, ind, tag


def matcher_case(seed, joints="crowd_pose", K=30, T=2, persons=4, step=0.5, spread=3, offsets=None, keys=None,
                 noise=0.0, clutter=1, presence=0.85, det_thr=0.1, tag_thr=1.0, use_det_val=True, ignore=False,
                 H=48, W=40):
    """One image's top-K arrays.  Person p has a base tag on the lattice ``step`` (``spread`` steps apart at most);
    each of its candidates sits at the base plus one of ``offsets`` (or a random lattice step), plus gaussian
    ``noise``; ``keys`` replaces tag[0] by a draw from a small set (key collisions); ``clutter`` candidates per joint
    carry random lattice tags."""
    rs = np.random.RandomState(seed)
    J, order = JOINTS[joints]
    base = rs.randint(-spread, spread + 1, size=(persons, T)) * step
    vals = np.zeros((J, K), F)
    inds = np.zeros((J, K), np.int32)
    tags = np.zeros((J, K, T), F)
    for j in range(J):
        cands = []
        for p in range(persons):
            if rs.rand() > presence:
                continue
            tg = base[p].astype(np.float64).copy()
            if offsets is not None:
                o = np.asarray(offsets[rs.randint(len(offsets))], np.float64)
                tg[:min(T, o.size)] += o[:T]
            else:
                tg += rs.randint(-1, 2, size=T) * step
            if noise:
                tg += rs.randn(T) * noise
            if keys is not None:
                tg[0] = keys[rs.randint(len(keys))]
            cands.append((VALS[rs.randint(len(VALS))], tg.astype(F)))
        for _ in range(clutter):
            tg = (rs.randint(-2 * spread, 2 * spread + 1, size=T) * step).astype(F)
            if keys is not None:
                tg[0] = keys[rs.randint(len(keys))]
            cands.append((VALS[rs.randint(len(VALS))], tg))
        vals[j], inds[j], tags[j] = _plane(rs, cands, K, H * W, T)
    return {"J": J, "order": list(order[:J]), "K": K, "T": T, "H": H, "W": W, "det_thr": det_thr,
            "tag_thr": tag_thr, "use_det_val": use_det_val, "ignore": ignore,
            "val_k": vals, "ind_k": inds, "tag_k": tags}


NEG0 = float(F(-0.0))
AXIS_HALF = [(0.5, 0.0), (0.0, -0.5), (1.5, 0.0), (0.0, 1.5), (-2.5, 0.0), (1.5, 2.0), (0.0, 0.0)]   # |d| = .5/1.5/2.5
AXIS_ONE = [(1.0, 0.0), (0.0, -1.0), (0.6, 0.0), (0.0, 0.0), (2.0, 0.0)]                            # |d| = TAG_THRESHOLD

# (name, seed, kwargs)
MATCHER_CASES = [
    ("lattice_k30", 1, dict()),
    ("lattice_quarter_k31", 2, dict(K=31, step=0.25, persons=8, clutter=3)),
    ("lattice_coco_k32", 3, dict(joints="coco", K=32, persons=10, clutter=4)),
    ("lattice_center_kept_k33", 4, dict(joints="center_kept", K=33, persons=12, clutter=4)),
    ("lattice_center_ignored_k48", 5, dict(joints="center_ignored", K=48, persons=14, clutter=6, step=0.25)),
    ("lattice_k64", 6, dict(K=64, persons=20, clutter=10, spread=6)),
    ("half_dist_t1", 7, dict(T=1, offsets=[(0.5,), (1.5,), (-2.5,), (0.0,)], persons=5, spread=4)),
    ("half_dist_t2", 8, dict(offsets=AXIS_HALF, persons=6, spread=4, step=1.0)),
    ("half_dist_t2_k2", 9, dict(K=2, offsets=AXIS_HALF, persons=3, spread=4, step=1.0, clutter=0)),
    ("half_dist_t3", 10, dict(T=3, offsets=AXIS_HALF, persons=6, spread=4, step=1.0)),
    ("at_threshold_1", 11, dict(offsets=AXIS_ONE, persons=5, spread=4, step=1.0)),
    ("at_threshold_05", 12, dict(offsets=[(0.5, 0.0), (0.0, 0.5), (0.25, 0.0)], tag_thr=0.5, persons=5, spread=4)),
    ("at_threshold_25", 13, dict(offsets=[(1.5, 2.0), (2.5, 0.0), (0.0, 1.0)], tag_thr=2.5, persons=4, spread=6,
                                 step=1.0)),
    ("keys_signed_zero", 14, dict(keys=[NEG0, 0.0, 1.0, 2.0], persons=5, clutter=2)),
    ("keys_dense_k33", 15, dict(K=33, keys=[NEG0, 0.0, 0.5], persons=12, clutter=6)),
    ("crowd_k1", 16, dict(K=1, persons=4, clutter=2)),
    ("crowd_k1_ignore", 16, dict(K=1, persons=4, clutter=2, ignore=True)),
    ("crowd_k2", 17, dict(K=2, persons=5, clutter=3)),
    ("crowd_k2_ignore", 17, dict(K=2, persons=5, clutter=3, ignore=True)),
    ("crowd_k31_ignore", 18, dict(K=31, persons=28, clutter=8, ignore=True, spread=8)),
    ("crowd_k33_ignore", 19, dict(K=33, persons=30, clutter=8, ignore=True, spread=8)),
    ("values_thr01", 20, dict(persons=6, clutter=6, presence=1.0)),
    ("values_thr0", 21, dict(persons=6, clutter=6, det_thr=0.0)),
    ("raw_costs", 22, dict(use_det_val=False, noise=0.2, persons=7, clutter=3)),
    ("raw_costs_k48", 23, dict(K=48, use_det_val=False, noise=0.3, persons=16, clutter=8, spread=6)),
    ("t1_mean_crowd_pose", 24, dict(T=1, noise=0.07, persons=2, spread=8, step=1.0, presence=1.0, clutter=0,
                                    offsets=[(0.0,)])),
    ("t1_mean_center_kept", 25, dict(joints="center_kept", T=1, noise=0.11, persons=3, spread=10, step=1.0,
                                     presence=1.0, clutter=0, offsets=[(0.0,)])),
    ("t4_lattice", 26, dict(T=4, persons=6, clutter=2)),
]


def t1_mean_edge_case(seed=90, n_prior=9, K=30):
    """T = 1, one person whose first ``n_prior`` joints (in joint order) carry noisy tags, then one candidate at exactly
    TAG_THRESHOLD (1.0) from numpy's mean of them (8-accumulator pairwise sum) and strictly closer to the
    sequentially summed mean: it starts a new person only if the mean is numpy's."""
    rs = np.random.RandomState(seed)
    J, order = JOINTS["crowd_pose"]
    while True:
        tags = (1.0 + rs.rand(n_prior) * 0.5).astype(F)
        pair = np.mean([np.array([t], F) for t in tags], axis=0)[0]
        seq = F(0)
        for t in tags:
            seq = F(seq + t)
        seq = F(seq / F(n_prior))
        cand = F(float(pair) + 1.0)
        if float(cand) - float(pair) == 1.0 and abs(float(cand) - float(seq)) < 1.0:
            break
    vals = np.zeros((J, K), F)
    inds = np.zeros((J, K), np.int32)
    tg = np.zeros((J, K, 1), F)
    for i, t in enumerate(list(tags) + [cand]):
        j = order[i]
        vals[j, 0], inds[j, 0], tg[j, 0, 0] = F(0.5), 7 * i + 3, t
    return {"J": J, "order": list(order[:J]), "K": K, "T": 1, "H": 48, "W": 40, "det_thr": 0.1, "tag_thr": 1.0,
            "use_det_val": True, "ignore": False, "val_k": vals, "ind_k": inds, "tag_k": tg}


MATCHER_NAMES = [c[0] for c in MATCHER_CASES] + ["t1_mean_at_threshold"]


def matcher_cases():
    return [(name, matcher_case(seed, **kw)) for name, seed, kw in MATCHER_CASES] + \
        [("t1_mean_at_threshold", t1_mean_edge_case())]


def loc_from_ind(ind, W):
    """[..., K] flat indices -> [..., K, 2] (x, y) as the reference's top_k returns them (int64)."""
    ind = ind.astype(np.int64)
    return np.stack((ind % W, ind // W), axis=-1)


def params_of(c):
    """An object with the fields of lib/core/group.py Params for a matcher / refine case."""
    class P(object):
        pass
    p = P()
    p.num_joints, p.max_num_people = c["J"], c.get("K", 30)
    p.detection_threshold, p.tag_threshold = c.get("det_thr", 0.1), c.get("tag_thr", 1.0)
    p.use_detection_val, p.ignore_too_much = c.get("use_det_val", True), c.get("ignore", False)
    p.joint_order = list(c.get("order", _ORDER17))
    return p


# ---------------------------------------------------------------------------------------------------- adjust + refine
def _refine_base(rs, J, H, W, T, persons, min_det=1, max_det=None, levels=None):
    det = (rs.rand(J, H, W) * 0.6 - 0.1).astype(F)
    if levels is not None:                           # few distinct values: equal neighbours everywhere
        det = np.asarray(levels, F)[rs.randint(len(levels), size=(J, H, W))]
    tag = (rs.randint(-4, 5, size=(J, H, W, T)) * 0.5).astype(F)
    ans = np.zeros((persons, J, 3 + T), F)
    max_det = J - 1 if max_det is None else max_det
    for p in range(persons):
        m = rs.randint(min_det, max_det + 1)
        for j in rs.choice(J, size=m, replace=False):
            y, x = rs.randint(H), rs.randint(W)
            v = F(0.2 + 0.8 * rs.rand())
            det[j, y, x] = v
            ans[p, j, :3] = (x, y, v)
            ans[p, j, 3:] = tag[j, y, x]
    return det, tag, ans


def refine_case(kind, seed, T=2, J=14, H=40, W=56):
    rs = np.random.RandomState(seed)
    if kind == "random":
        det, tag, ans = _refine_base(rs, J, H, W, T, persons=6)
    elif kind == "borders":
        # every keypoint on a border or a corner; det on two levels so that neighbours are often equal
        det, tag, ans = _refine_base(rs, J, H, W, T, persons=6, levels=[0.25, 0.5])
        edge = [(0, 0), (0, H - 1), (W - 1, 0), (W - 1, H - 1), (0, H // 2), (W - 1, H // 3), (W // 2, 0),
                (W // 3, H - 1)]
        for p in range(ans.shape[0]):
            for j in range(J):
                if ans[p, j, 2] > 0:
                    x, y = edge[(p * J + j) % len(edge)]
                    ans[p, j, 0:2] = (x, y)
                    ans[p, j, 3:] = tag[j, y, x]
    elif kind == "one_and_most":
        # persons with a single detected joint and persons missing a single joint
        det, tag, ans = _refine_base(rs, J, H, W, T, persons=8, min_det=1, max_det=1)
        _, _, many = _refine_base(rs, J, H, W, T, persons=4, min_det=J - 1, max_det=J - 1)
        for p in range(many.shape[0]):
            for j in range(J):
                if many[p, j, 2] > 0:
                    x, y = int(many[p, j, 0]), int(many[p, j, 1])
                    det[j, y, x] = many[p, j, 2]
                    many[p, j, 3:] = tag[j, y, x]
        ans = np.concatenate((ans, many))
    elif kind == "many_missing":
        # 40 persons, every one missing joint 3 (and some joint 7): more than one 32-person batch per plane
        det, tag, ans = _refine_base(rs, J, H, W, T, persons=40, min_det=J - 2, max_det=J - 1)
        ans[:, 3, :] = 0
        ans[::3, 7, :] = 0
        for p in range(ans.shape[0]):
            if not (ans[p, :, 2] > 0).any():
                ans[p, 0, :3] = (1, 1, det[0, 1, 1] if det[0, 1, 1] > 0 else 0.5)
    elif kind == "chunks":
        # maps of 3+ 2048-pixel chunks; per missing joint the refine maximum is tied across chunks (first index
        # wins), and -0.0 (det -0.0) ties +0.0 (det 1, distance 1) at a later index: the -0.0 pixel wins, so nothing
        # is filled.  Every detected tag is 1.0, so prev_tag == 1 and the distance is |tag - 1|.
        H, W = 48, 128
        det = np.full((J, H, W), F(-3.0))
        tag = np.full((J, H, W, T), F(1.0))
        ans = np.zeros((2, J, 3 + T), F)
        for p in range(2):
            for j in range(J // 2):
                x, y = 5 + 7 * j, 3 + 20 * p
                det[j, y, x] = F(0.9)
                ans[p, j, :3] = (x, y, 0.9)
                ans[p, j, 3:] = 1.0
        for j in range(J // 2, J):
            flat = det[j].reshape(-1)
            tg = tag[j].reshape(-1, T)
            if j % 2 == 0:
                for i in (300 + j, 2048 + 300 + j, 4096 + 1000):
                    flat[i] = F(0.7)
            else:
                flat[100 + j] = F(-0.0)
                flat[2048 + 77] = F(1.0)
                tg[2048 + 77, 0] = F(2.0)                   # distance 1 -> score 1 - 1 = +0.0
    elif kind == "rint_half":
        # refine distances exactly 0.5 and 2.5: rint sends them to 0 and 2, round-half-away to 1 and 3
        H, W = 24, 32
        det = np.full((J, H, W), F(-5.0))
        tag = np.zeros((J, H, W, T), F)
        ans = np.zeros((1, J, 3 + T), F)
        for j in range(0, J, 2):
            det[j, 2, 2 + j] = F(0.8)
            ans[0, j, :3] = (2 + j, 2, 0.8)
        for j in range(1, J, 2):
            det[j, 5, 9] = F(1.0)
            tag[j, 5, 9, 0] = F(0.5)                        # rint(0.5) = 0: score 1.0
            det[j, 9, 3] = F(0.6)                           # distance 0: score 0.6
            det[j, 12, 20] = F(3.0)
            tag[j, 12, 20, T - 1] = F(-2.5)                 # rint(2.5) = 2: score 1.0, later index
    elif kind == "nonpositive":
        # joints whose refine maximum is <= 0 or NaN: never filled
        det, tag, ans = _refine_base(rs, J, H, W, T, persons=3, min_det=4, max_det=6)
        for j in range(J):
            if (ans[:, j, 2] > 0).any():
                continue
            if j % 3 == 0:
                det[j] = -np.abs(det[j]) - F(0.01)
            elif j % 3 == 1:
                det[j] = -np.abs(det[j])
                det[j, H // 2, W // 3] = F(0.0)
            else:
                det[j, 7, 11] = F(np.nan)
    else:
        raise KeyError(kind)
    return {"J": J, "T": T, "det": det, "tag": tag, "ans": ans}


REFINE_CASES = [
    ("random_t1", "random", 31, 1), ("random_t2", "random", 32, 2), ("random_t3", "random", 33, 3),
    ("random_t4", "random", 34, 4), ("borders_t2", "borders", 35, 2), ("borders_t1", "borders", 36, 1),
    ("one_and_most_t2", "one_and_most", 37, 2), ("one_and_most_t4", "one_and_most", 38, 4),
    ("many_missing_t2", "many_missing", 39, 2), ("many_missing_t3", "many_missing", 40, 3),
    ("chunks_t1", "chunks", 41, 1), ("chunks_t2", "chunks", 42, 2), ("rint_half_t1", "rint_half", 43, 1),
    ("rint_half_t2", "rint_half", 44, 2), ("nonpositive_t2", "nonpositive", 45, 2),
]


def refine_cases():
    return [(name, refine_case(kind, seed, T=t)) for name, kind, seed, t in REFINE_CASES]


# ---------------------------------------------------------------------------------------------------- NMS + top-K
# peak heights, including the float32 neighbours of the thresholds 0.1 and 0.05 (both round up to float32)
PEAK_VALS = [F(0.05), np.nextafter(F(0.05), F(0)), ONE_TENTH, BELOW_TENTH] + [F(0.1 + k * 0.1) for k in range(1, 9)]


def _background(rs, shape):
    return (rs.rand(*shape) * 0.05).astype(F)


def topk_case(kind, seed, H, W, kernel=5, K=30, J=2, T=2, min_value=0.0):
    """det [1,J,H,W], tag [1,J,H,W,T] of one top-K edge case."""
    rs = np.random.RandomState(seed)
    det = _background(rs, (1, J, H, W))
    if kind == "peaks":
        for j in range(J):
            for _ in range(3 * K // 2):
                det[0, j, rs.randint(H), rs.randint(W)] = PEAK_VALS[rs.randint(len(PEAK_VALS))]
    elif kind == "plateau_borders":
        # equal values on the rows around every strip / band border: the K-th value is tied across CTAs and warps
        for j in range(J):
            for y in range(H):
                if y % 4 in (0, 3) or y in (H - 1, 1):
                    xs = rs.choice(W, size=min(W, 3), replace=False)
                    det[0, j, y, xs] = F(0.5)
            det[0, j, rs.randint(H), rs.randint(W)] = F(0.9)
    elif kind == "whole_plateau":
        det[0, 0] = F(0.3)
    elif kind == "sparse":
        # fewer survivors than K
        for j in range(J):
            for _ in range(K // 3):
                det[0, j, rs.randint(H), rs.randint(W)] = F(0.6)
    elif kind == "specials":
        # subnormals, -0.0, negatives, +inf and NaN pixels
        tiny = np.array([1e-45, 1e-42, 1e-40, 1.2e-38], F)
        for j in range(J):
            pl = det[0, j]
            n = H * W
            pl.reshape(-1)[rs.choice(n, size=n // 3, replace=False)] = -np.abs(pl.reshape(-1)[:n // 3]) - F(0.001)
            pl.reshape(-1)[rs.choice(n, size=max(1, n // 50), replace=False)] = F(-0.0)
            pl.reshape(-1)[rs.choice(n, size=max(1, n // 40), replace=False)] = tiny[rs.randint(4, size=max(1, n // 40))]
            pl.reshape(-1)[rs.choice(n, size=max(1, n // 60), replace=False)] = F(np.nan)
            pl[rs.randint(H), rs.randint(W)] = F(np.inf)
            for _ in range(K // 2):
                pl[rs.randint(H), rs.randint(W)] = F(0.2 + 0.1 * rs.randint(8))
    elif kind == "subnormal_only":
        det[0] = F(0.0)
        tiny = np.array([1e-45, 1e-42, 1e-40, 9.99995e-41, 1.2e-38], F)
        for j in range(J):
            for _ in range(K):
                det[0, j, rs.randint(H), rs.randint(W)] = tiny[rs.randint(len(tiny))]
    elif kind == "nan_window":
        # isolated peaks, each with one NaN at one offset of its window (every offset once), plus clean peaks
        R = kernel // 2
        offs = [(dy, dx) for dy in range(-R, R + 1) for dx in range(-R, R + 1) if (dy, dx) != (0, 0)]
        step = kernel + 2
        cells = [(y, x) for y in range(R + 1, H - R - 1, step) for x in range(R + 1, W - R - 1, step)]
        rs.shuffle(cells)
        per = len(offs) // J + 1
        c = 0
        for j in range(J):
            for dy, dx in offs[j * per:(j + 1) * per]:
                y, x = cells[c]
                c += 1
                det[0, j, y, x] = F(0.9)
                det[0, j, y + dy, x + dx] = F(np.nan)
            for _ in range(4):
                y, x = cells[c]
                c += 1
                det[0, j, y, x] = F(0.7)
    else:
        raise KeyError(kind)
    tag = rs.randn(1, J, H, W, T).astype(F)
    return det, tag


# (name, kind, seed, H, W, kernel, K, min_value).  strip heights: W <= 1024 -> 16 rows, <= 1536 -> 8, <= 2048 -> 4,
# wider -> 2; W % 4 != 0 takes the scalar path; H > 2048 at 16-row strips gives more than 4 strips per band.
TOPK_CASES = [
    ("k1", "peaks", 1, 40, 48, 1, 30, 0.0),
    ("k3", "peaks", 2, 40, 48, 3, 30, 0.0),
    ("k5", "peaks", 3, 40, 48, 5, 30, 0.0),
    ("k7", "peaks", 4, 40, 48, 7, 30, 0.0),
    ("k9", "peaks", 5, 40, 48, 9, 30, 0.0),
    ("k9_scalar", "peaks", 6, 45, 47, 9, 33, 0.0),
    ("h1", "peaks", 7, 1, 64, 5, 30, 0.0),
    ("h2_scalar", "peaks", 8, 2, 63, 3, 30, 0.0),
    ("sr16_h15", "plateau_borders", 9, 15, 1024, 5, 64, 0.0),
    ("sr16_h17_scalar", "plateau_borders", 10, 17, 1021, 5, 64, 0.0),
    ("sr16_bands", "plateau_borders", 11, 16 * 4 * 3 + 5, 96, 5, 64, 0.0),
    ("sr8_h7_scalar", "plateau_borders", 12, 7, 1025, 5, 48, 0.0),
    ("sr8_h9", "plateau_borders", 13, 9, 1536, 3, 48, 0.0),
    ("sr8_bands", "peaks", 14, 8 * 4 * 2 + 3, 1400, 5, 30, 0.0),
    ("sr4_h3", "plateau_borders", 15, 3, 2048, 5, 33, 0.0),
    ("sr4_h5_scalar", "plateau_borders", 16, 5, 1537, 7, 33, 0.0),
    ("sr4_bands", "peaks", 17, 4 * 4 * 2 + 1, 1800, 5, 30, 0.0),
    ("sr2_h1", "peaks", 18, 1, 2052, 5, 32, 0.0),
    ("sr2_h3_scalar", "plateau_borders", 19, 3, 2049, 5, 31, 0.0),
    ("sr2_bands", "plateau_borders", 20, 2 * 4 * 2 + 1, 2100, 3, 64, 0.0),
    ("tall_spb5", "peaks", 21, 2100, 64, 5, 64, 0.0),
    ("tall_spb5_scalar", "plateau_borders", 22, 2100, 30, 5, 64, 0.0),
    ("whole_plateau", "whole_plateau", 23, 64, 160, 5, 30, 0.0),
    ("sparse_k64", "sparse", 24, 48, 64, 5, 64, 0.0),
    ("sparse_k1", "sparse", 25, 48, 64, 5, 1, 0.0),
    ("specials", "specials", 26, 50, 72, 5, 30, 0.0),
    ("specials_k3_scalar", "specials", 27, 33, 41, 3, 64, 0.0),
    ("subnormal_thr0", "subnormal_only", 28, 30, 40, 3, 32, 0.0),
    ("subnormal_thr1e-40", "subnormal_only", 28, 30, 40, 3, 32, 1e-40),
    ("peaks_thr01", "peaks", 29, 40, 64, 5, 30, 0.1),
    ("peaks_thr005", "peaks", 30, 40, 64, 5, 30, 0.05),
    ("nan_window_k3", "nan_window", 31, 64, 64, 3, 64, 0.0),
    ("nan_window_k5", "nan_window", 32, 96, 96, 5, 64, 0.0),
    ("nan_window_k7", "nan_window", 33, 96, 100, 7, 64, 0.0),
    ("nan_window_k9", "nan_window", 34, 112, 112, 9, 64, 0.0),
]


def topk_cases():
    out = []
    for name, kind, seed, h, w, kernel, k, mv in TOPK_CASES:
        J = 4 if kind == "nan_window" and kernel >= 7 else 2
        det, tag = topk_case(kind, seed, h, w, kernel=kernel, K=k, J=J, min_value=mv)
        out.append((name, det, tag, kernel, k, mv))
    return out


def expected_topk(group_ref, det, tag, kernel, K, min_value):
    """group_ref.top_k with the survivors at or below ``min_value`` (compared in double, like the reference's
    threshold) turned into empty slots (value 0, index 0)."""
    class P(object):
        pass
    p = P()
    p.max_num_people, p.num_joints = K, det.shape[1]
    r = group_ref.top_k(det, tag, p, kernel, kernel // 2)
    val, ind = r["val_k"].copy(), (r["loc_k"][..., 1] * det.shape[3] + r["loc_k"][..., 0]).astype(np.int64)
    drop = ~(val.astype(np.float64) > min_value)
    val[drop] = 0
    ind[drop] = 0
    tg = tag.reshape(tag.shape[0], tag.shape[1], -1, tag.shape[-1])
    tag_k = np.stack([tg[a, b][ind[a, b]] for a in range(det.shape[0]) for b in range(det.shape[1])])
    return val, ind.astype(np.int32), tag_k.reshape(r["tag_k"].shape)
