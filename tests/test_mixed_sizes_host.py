"""Host side of mixed batches (litepose_b200.mixed): size groups, arena layout, descriptors and workspace sizes - no GPU
needed."""
import numpy as np
import pytest
import torch

from litepose_b200 import _lib
from litepose_b200.lib.utils import transforms as tf
from litepose_b200.mixed import MAP_DESC, WARP_DESC, MixedPlan, image_shapes

SHAPES = [(480, 640), (640, 480), (481, 640), (300, 900), (512, 512), (479, 641), (640, 480)]


def _ref_multi_scale_size(h, w, input_size, s, smin):
    """reference lib/utils/transforms.py:155-180 restated independently of the module under test"""
    up = lambda v: int(np.ceil(v / 64.0) * 64)
    center = np.array([int(w / 2.0 + 0.5), int(h / 2.0 + 0.5)])
    short = up(smin * input_size)
    if w < h:
        w_r = int(short * s / smin)
        h_r = int(up(short / w * h) * s / smin)
        scale = np.array([w / 200.0, h_r / w_r * w / 200.0])
    else:
        h_r = int(short * s / smin)
        w_r = int(up(short / h * w) * s / smin)
        scale = np.array([w_r / h_r * h / 200.0, h / 200.0])
    return (h_r, w_r), center, scale


@pytest.mark.parametrize("scales,size,project", [([1.0], 512, True), ([2.0, 1.0, 0.5], 256, True),
                                                 ([2.0, 1.0, 0.5], 256, False)])
def test_groups_keys_centers_scales(scales, size, project):
    mp = MixedPlan(SHAPES, scales, size, project, 14, 2)
    for i, (h, w) in enumerate(SHAPES):
        ref = [_ref_multi_scale_size(h, w, size, s, min(scales)) for s in scales]
        assert mp.keys[i] == tuple(r[0] for r in ref)
        for (c, sc), r in zip(mp.center_scale[i], ref):
            assert np.array_equal(c, r[1]) and np.array_equal(sc, r[2])
        p = mp.pos[i]
        assert np.array_equal(mp.centers[p], ref[-1][1]) and np.array_equal(mp.scales_[p], ref[-1][2])
    # one group per distinct key, caller order inside a group, groups in first-appearance order
    keys = [mp.keys[i] for i in range(len(SHAPES))]
    assert [g.key for g in mp.groups] == list(dict.fromkeys(keys))
    for g in mp.groups:
        assert g.images == [i for i in range(len(SHAPES)) if keys[i] == g.key]
        h1, w1 = g.in_hw[1.0]
        hb, wb = g.in_hw[scales[0]]
        assert g.det_hw == ((h1, w1) if project else (hb // 2, wb // 2))
    assert len(mp.groups) >= 4


def test_order_is_restored():
    mp = MixedPlan(SHAPES, [1.0], 512, True, 14, 2)
    assert sorted(mp.order) == list(range(len(SHAPES)))
    assert [mp.order[p] for p in mp.pos] == list(range(len(SHAPES)))
    res = ["r%d" % i for i in mp.order]                  # results in arena order
    assert [res[p] for p in mp.pos] == ["r%d" % i for i in range(len(SHAPES))]


@pytest.mark.parametrize("J,T", [(14, 2), (17, 1)])
def test_descriptors_and_arena_offsets(J, T):
    scales = [2.0, 1.0, 0.5]
    mp = MixedPlan(SHAPES, scales, 256, True, J, T)
    md = mp.map_desc()
    assert md.dtype == MAP_DESC and md.dtype.itemsize == 24
    for p, i in enumerate(mp.order):
        g = next(g for g in mp.groups if i in g.images)
        hd, wd = g.det_hw
        assert (md[p]["h"], md[p]["w"]) == (hd, wd)
        assert md[p]["det_offset"] == mp.det_off[p] and mp.det_off[p + 1] - mp.det_off[p] == J * hd * wd
        assert md[p]["tag_offset"] == mp.tag_off[p] and mp.tag_off[p + 1] - mp.tag_off[p] == J * hd * wd * T
        h, w = SHAPES[i]
        assert mp.src_off[p + 1] - mp.src_off[p] == h * w * 3
    # a group's images are adjacent: its arena slice is an ordinary [n_g,J,Hd,Wd] tensor
    for g in mp.groups:
        assert [mp.pos[i] for i in g.images] == list(range(g.start, g.start + g.n))
    for s in scales:
        wd_ = mp.warp_desc(s)
        assert wd_.dtype == WARP_DESC and wd_.dtype.itemsize == 80
        for p, i in enumerate(mp.order):
            g = next(g for g in mp.groups if i in g.images)
            hs, ws = g.in_hw[s]
            assert (wd_[p]["out_h"], wd_[p]["out_w"]) == (hs, ws)
            assert wd_[p]["dst_offset"] == mp.in_off[s][p] and mp.in_off[s][p + 1] - mp.in_off[s][p] == 3 * hs * ws
            assert (wd_[p]["src_h"], wd_[p]["src_w"]) == SHAPES[i] and wd_[p]["src_offset"] == mp.src_off[p]
            c, sc = mp.center_scale[i][scales.index(s)]
            assert np.array_equal(wd_[p]["minv"], tf.invert_affine(tf.get_affine_transform(c, sc, 0, (ws, hs))))
        assert mp.max_in_hw(s) == (max(g.in_hw[s][0] for g in mp.groups), max(g.in_hw[s][1] for g in mp.groups))


def test_ragged_workspace_sizes():
    """The ragged top-K workspace is the sum of the uniform per-image workspaces (lists as prefix sums over images);
    a group of equal sizes needs exactly what the uniform call on that group needs."""
    lib = _lib.load()
    J, K = 14, 30
    mp = MixedPlan(SHAPES, [1.0], 512, True, J, 2)
    hw = np.ascontiguousarray(mp.det_hw, np.int32)
    n = hw.shape[0]
    got = lib.lp_nms_topk_ragged_workspace_bytes(n, hw.ctypes.data, J, K)
    assert got == sum(lib.lp_nms_topk_workspace_bytes(1, J, int(h), int(w), K) for h, w in hw)
    for g in mp.groups:
        sub = np.ascontiguousarray(hw[g.start:g.start + g.n])
        assert (lib.lp_nms_topk_ragged_workspace_bytes(g.n, sub.ctypes.data, J, K)
                == lib.lp_nms_topk_workspace_bytes(g.n, J, g.det_hw[0], g.det_hw[1], K))
    bad = np.array([[64, 0]], np.int32)
    assert lib.lp_nms_topk_ragged_workspace_bytes(1, bad.ctypes.data, J, K) == 0


def test_bad_image_lists_raise():
    with pytest.raises(ValueError, match="empty"):
        image_shapes([])
    with pytest.raises(TypeError, match="uint8"):
        image_shapes([np.zeros((8, 8, 3), np.uint8), np.zeros((8, 8, 3), np.float32)])
    with pytest.raises(TypeError, match=r"\[H,W,3\]"):
        image_shapes([np.zeros((8, 8, 4), np.uint8)])
    with pytest.raises(TypeError, match=r"\[H,W,3\]"):
        image_shapes([torch.zeros((8, 8), dtype=torch.uint8)])
    with pytest.raises(TypeError, match="uint8"):
        image_shapes([torch.zeros((8, 8, 3), dtype=torch.int32)])
    assert image_shapes([torch.zeros((8, 9, 3), dtype=torch.uint8), np.zeros((5, 7, 3), np.uint8)]) == [(8, 9), (5, 7)]
