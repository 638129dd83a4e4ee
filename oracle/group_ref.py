"""ORACLE (test infrastructure, not product code).

numpy restatement of the associative-embedding post-process of the reference:
``HeatmapParser`` / ``match_by_tag`` (reference lib/core/group.py:26-97,100-291).
Index / integer / assignment results are the bit-exact yardstick for the CUDA
parser (litepose_b200/csrc/parser_*.cu); coordinates and scores are exact too when
both sides see identical fp32 ``det``/``tag`` inputs.

Each function cites the reference lines it follows.  Two places need a canonical
choice because the reference delegates to implementation-defined behaviour:

  * ``top_k`` (group.py:141-176) uses ``torch.topk`` whose tie order is
    unspecified.  Canonical order here: value descending, flat index ascending,
    taken over NMS survivors with value > 0; if fewer than K such survivors exist
    the remaining slots are (val 0.0, flat index 0).  Slots with val <= 0 can never
    pass ``val > DETECTION_THRESHOLD`` (threshold >= 0 is asserted), so they do not
    influence grouping.  NaN never takes a slot (``torch.topk`` would rank it
    first): ``nms`` propagates NaN like the reference's max-pool, so a NaN pixel
    and every pixel with a NaN in its window drop out at ``> 0``.
  * ``py_max_match`` (group.py:19-23) calls the third-party ``munkres`` package;
    see oracle/munkres_ref.py ("parity unpinned" at that boundary).

Pinned against the real reference (run from /root/reference with the shims of
oracle/refshim.py) in tests/test_oracle_vs_reference.py and via tests/golden/.
"""
import numpy as np

from .munkres_ref import Munkres


class Params(object):
    """reference lib/core/group.py:100-120."""

    def __init__(self, cfg):
        self.num_joints = cfg.DATASET.NUM_JOINTS
        self.max_num_people = cfg.DATASET.MAX_NUM_PEOPLE
        self.detection_threshold = cfg.TEST.DETECTION_THRESHOLD
        self.tag_threshold = cfg.TEST.TAG_THRESHOLD
        self.use_detection_val = cfg.TEST.USE_DETECTION_VAL
        self.ignore_too_much = cfg.TEST.IGNORE_TOO_MUCH
        if cfg.DATASET.WITH_CENTER and cfg.TEST.IGNORE_CENTER:
            self.num_joints -= 1
        if cfg.DATASET.WITH_CENTER and not cfg.TEST.IGNORE_CENTER:
            self.joint_order = [i - 1 for i in
                                [18, 1, 2, 3, 4, 5, 6, 7, 12, 13, 8, 9, 10, 11, 14, 15, 16, 17]]
        else:
            self.joint_order = [i - 1 for i in
                                [1, 2, 3, 4, 5, 6, 7, 12, 13, 8, 9, 10, 11, 14, 15, 16, 17]]


def py_max_match(scores, solver=Munkres):
    """group.py:19-23."""
    return np.array(solver().compute(scores)).astype(np.int32)


def match_by_tag(inp, params, solver=Munkres, events=None):
    """group.py:26-97, statement by statement (float64 joints rows, float32 running
    tag means via np.mean, round-half-even cost, 1e10 column padding, dict keyed by
    the float32 tag[0] in insertion order).  ``solver`` and ``events`` (a
    collections.Counter) let the edge tests count which branches a case reaches;
    neither changes the result."""
    ev = events if events is not None else {}

    def hit(name, cond=True):
        if cond:
            ev[name] = ev.get(name, 0) + 1
    tag_k, loc_k, val_k = inp
    default_ = np.zeros((params.num_joints, 3 + tag_k.shape[2]))
    joint_dict = {}
    tag_dict = {}
    for i in range(params.num_joints):
        idx = params.joint_order[i]
        tags = tag_k[idx]
        joints = np.concatenate((loc_k[idx], val_k[idx, :, None], tags), 1)
        mask = joints[:, 2] > params.detection_threshold
        tags = tags[mask]
        joints = joints[mask]
        if joints.shape[0] == 0:
            continue
        if i == 0 or len(joint_dict) == 0:
            for tag, joint in zip(tags, joints):
                key = tag[0]
                hit("key_collision", key in joint_dict)
                joint_dict.setdefault(key, np.copy(default_))[idx] = joint
                tag_dict[key] = [tag]
        else:
            grouped_keys = list(joint_dict.keys())[:params.max_num_people]
            grouped_tags = [np.mean(tag_dict[k], axis=0) for k in grouped_keys]
            if params.ignore_too_much and len(grouped_keys) == params.max_num_people:
                hit("ignore_too_much_skip")
                continue
            diff = joints[:, None, 3:] - np.array(grouped_tags)[None, :, :]
            diff_normed = np.linalg.norm(diff, ord=2, axis=2)
            diff_saved = np.copy(diff_normed)
            hit("dist_eq_threshold", bool((diff_saved == params.tag_threshold).any()))
            if params.use_detection_val:
                hit("round_half_tie", bool((np.abs(diff_normed - np.floor(diff_normed) - 0.5) == 0).any()))
                diff_normed = np.round(diff_normed) * 100 - joints[:, 2:3]
            num_added = diff.shape[0]
            num_grouped = diff.shape[1]
            hit("pad_rows", num_added < num_grouped)
            hit("pad_cols", num_added > num_grouped)
            if num_added > num_grouped:
                diff_normed = np.concatenate(
                    (diff_normed, np.zeros((num_added, num_added - num_grouped)) + 1e10), axis=1)
            pairs = py_max_match(diff_normed, solver)
            for row, col in pairs:
                if row < num_added and col < num_grouped and diff_saved[row][col] < params.tag_threshold:
                    key = grouped_keys[col]
                    joint_dict[key][idx] = joints[row]
                    tag_dict[key].append(tags[row])
                else:
                    key = tags[row][0]
                    hit("key_collision", key in joint_dict)
                    joint_dict.setdefault(key, np.copy(default_))[idx] = joints[row]
                    tag_dict[key] = [tags[row]]
    return np.array([joint_dict[k] for k in joint_dict]).astype(np.float32)


def nms(det, kernel, padding):
    """group.py:131-135 with MaxPool2d(kernel, 1, padding) (-inf padding):
    ``det * (maxpool(det) == det)``.  det: [N,J,H,W] float32."""
    n, j, h, w = det.shape
    assert kernel == 2 * padding + 1, "NMS window must be centred (kernel == 2*padding+1)"
    pad = np.full((n, j, h + 2 * padding, w + 2 * padding), -np.inf, dtype=np.float32)
    pad[:, :, padding:padding + h, padding:padding + w] = det
    # separable running max
    m = pad[:, :, :, 0:w].copy()
    for d in range(1, kernel):
        np.maximum(m, pad[:, :, :, d:d + w], out=m)
    mm = m[:, :, 0:h, :].copy()
    for d in range(1, kernel):
        np.maximum(mm, m[:, :, d:d + h, :], out=mm)
    return det * (mm == det).astype(np.float32)


def top_k(det, tag, params, kernel, padding, tag_per_joint=True):
    """group.py:141-176 with the canonical tie/fill rule of the module docstring.
    det [N,J,H,W] f32, tag [N,J,H,W,T] f32 ->
    {'tag_k': [N,J,K,T] f32, 'loc_k': [N,J,K,2] i64 (x,y), 'val_k': [N,J,K] f32}."""
    det = np.ascontiguousarray(det, dtype=np.float32)
    tag = np.ascontiguousarray(tag, dtype=np.float32)
    n, j, h, w = det.shape
    k = params.max_num_people
    d = nms(det, kernel, padding).reshape(n, j, h * w)
    tg = tag.reshape(tag.shape[0], tag.shape[1], h * w, -1)
    if not tag_per_joint:
        tg = np.broadcast_to(tg, (n, params.num_joints, h * w, tg.shape[3]))
    t = tg.shape[3]
    val_k = np.zeros((n, j, k), np.float32)
    ind = np.zeros((n, j, k), np.int64)
    for a in range(n):
        for b in range(j):
            row = d[a, b]
            cand = np.nonzero(row > 0)[0]
            if cand.size > k:
                part = np.argpartition(-row[cand], k - 1)[:k]
                # keep every candidate tied with the k-th value so the index rule decides
                kth = row[cand[part]].min()
                cand = cand[row[cand] >= kth]
            order = np.lexsort((cand, -row[cand].astype(np.float64)))[:k]
            sel = cand[order]
            val_k[a, b, :sel.size] = row[sel]
            ind[a, b, :sel.size] = sel
    tag_k = np.zeros((n, j, k, t), np.float32)
    for a in range(n):
        for b in range(j):
            tag_k[a, b] = tg[a, b, ind[a, b], :]
    loc_k = np.stack((ind % w, ind // w), axis=3)
    return {"tag_k": tag_k, "loc_k": loc_k, "val_k": val_k}


def adjust(ans, det):
    """group.py:178-197 (quarter-pixel shift toward the larger neighbour, strict >,
    then +0.5).  ans: list over images of [P,J,3+T] float32; det [N,J,H,W]."""
    for batch_id, people in enumerate(ans):
        for people_id, person in enumerate(people):
            for joint_id, joint in enumerate(person):
                if joint[2] > 0:
                    x, y = joint[0:2]          # (column, row) coordinates
                    xi, yi = int(x), int(y)
                    tmp = det[batch_id][joint_id]
                    if tmp[yi, min(xi + 1, tmp.shape[1] - 1)] > tmp[yi, max(xi - 1, 0)]:
                        x += np.float32(0.25)
                    else:
                        x -= np.float32(0.25)
                    if tmp[min(yi + 1, tmp.shape[0] - 1), xi] > tmp[max(0, yi - 1), xi]:
                        y += np.float32(0.25)
                    else:
                        y -= np.float32(0.25)
                    ans[batch_id][people_id, joint_id, 0:2] = (x + np.float32(0.5), y + np.float32(0.5))
    return ans


def _row_sum_f32(col):
    """ATen CPU ``row_sum`` (aten/src/ATen/native/cpu/SumKernel.cpp): four interleaved
    partial sums over full groups of 4, tail added to partial 0, partials folded
    left to right; everything in float32 starting from 0."""
    f = np.float32
    n = len(col)
    g = n // 4
    p = [f(0), f(0), f(0), f(0)]
    for i in range(g):
        for k in range(4):
            p[k] = f(p[k] + col[4 * i + k])
    for i in range(4 * g, n):
        p[0] = f(p[0] + col[i])
    for k in range(1, 4):
        p[0] = f(p[0] + p[k])
    return p[0]


def _mean_f32_rows(rows):
    """``torch.mean(torch.cat(tags, 0), dim=0)`` of an [m,T] fp32 CPU tensor
    (group.py:220) restated: ATen sums columns in groups of 4 sequentially over the
    rows (``multi_row_sum``) and each left-over column with ``row_sum``; the mean
    divides the fp32 sum by m.  Verified bit-exact against torch 2.11 for T in 2..6
    and for T == 1 with m < 8 (tests/test_oracle_vs_reference.py).  For T == 1 and
    m >= SIMD width torch switches to a vectorised inner sum whose order depends on
    the host CPU (AVX2 vs AVX-512), i.e. the reference itself is not reproducible
    there; the scalar ``row_sum`` order is the canonical choice of this oracle."""
    a = np.stack(rows).astype(np.float32)
    m, t = a.shape
    out = np.zeros(t, np.float32)
    full = (t // 4) * 4
    for c in range(full):
        s = np.float32(0)
        for i in range(m):
            s = np.float32(s + a[i, c])
        out[c] = s
    for c in range(full, t):
        out[c] = _row_sum_f32(a[:, c])
    return (out / np.float32(m)).astype(np.float32)


def refine(det, tag, keypoints):
    """group.py:199-267 for one person.  det [J,H,W] f32, tag [J,H,W,T] f32,
    keypoints [J,3+T] f32 (modified in place and returned)."""
    if tag.ndim == 3:
        tag = tag[:, :, :, None]
    tags = []
    for i in range(keypoints.shape[0]):
        if keypoints[i, 2] > 0:
            x, y = keypoints[i][:2].astype(np.int32)
            tags.append(tag[i, y, x])
    prev_tag = _mean_f32_rows(tags)
    # dense pass with the same fp32 torch CPU ops the reference issues (group.py:221-224); torch is
    # multi-threaded, which keeps the CPU baseline representative of the reference's own cost
    import torch
    tt_ = torch.from_numpy(np.ascontiguousarray(tag))
    dt_ = torch.from_numpy(np.ascontiguousarray(det))
    tt = (((tt_ - torch.from_numpy(prev_tag)[None, None, None, :]) ** 2).sum(dim=3) ** 0.5)
    p, h, w = tt.shape
    pos = (dt_ - torch.round(tt)).view(p, -1).argmax(dim=1).numpy()
    ans = []
    for i in range(keypoints.shape[0]):
        tmp = det[i]
        y = int(pos[i] // w)
        x = int(pos[i] % w)
        xx, yy = x, y
        val = tmp[y, x]
        x += 0.5
        y += 0.5
        if tmp[yy, min(xx + 1, tmp.shape[1] - 1)] > tmp[yy, max(xx - 1, 0)]:
            x += 0.25
        else:
            x -= 0.25
        if tmp[min(yy + 1, tmp.shape[0] - 1), xx] > tmp[max(0, yy - 1), xx]:
            y += 0.25
        else:
            y -= 0.25
        ans.append((x, y, val))
    for i in range(det.shape[0]):
        if ans[i][2] > 0 and keypoints[i, 2] == 0:
            keypoints[i, :2] = ans[i][:2]
            keypoints[i, 2] = ans[i][2]
    return keypoints


class HeatmapParser(object):
    """group.py:123-291 on numpy inputs (``det`` [N,J,H,W], ``tag`` [N,J,H,W,T])."""

    def __init__(self, cfg):
        self.params = Params(cfg)
        self.tag_per_joint = cfg.MODEL.TAG_PER_JOINT
        self.kernel = cfg.TEST.NMS_KERNEL
        self.padding = cfg.TEST.NMS_PADDING
        assert self.params.detection_threshold >= 0

    def top_k(self, det, tag):
        return top_k(det, tag, self.params, self.kernel, self.padding, self.tag_per_joint)

    def match(self, tag_k, loc_k, val_k):
        return [match_by_tag(x, self.params) for x in zip(tag_k, loc_k, val_k)]

    def parse(self, det, tag, adjust_=True, refine_=True):
        """group.py:269-291: image 0 only for scores/refine, like the reference."""
        det = np.asarray(det, dtype=np.float32)
        tag = np.asarray(tag, dtype=np.float32)
        ans = self.match(**self.top_k(det, tag))
        if adjust_:
            ans = adjust(ans, det)
        scores = [i[:, 2].mean() for i in ans[0]]
        if refine_:
            ans = ans[0]
            tag0 = tag[0]
            if not self.tag_per_joint:
                # group.py:283-286 means to tile the shared tag map over the joints (the reference's own lines stop on
                # the unassigned name `tag_numpy` there; the tiling is the evident intent)
                tag0 = np.tile(tag0, (self.params.num_joints,) + (1,) * (tag0.ndim - 1))
            for i in range(len(ans)):
                ans[i] = refine(det[0], tag0, ans[i])
            ans = [ans]
        return ans, scores

    def parse_batch(self, det, tag, adjust_=True, refine_=True):
        """N independent ``parse`` calls (SURVEY H5)."""
        return [self.parse(det[i:i + 1], tag[i:i + 1], adjust_, refine_) for i in range(det.shape[0])]
