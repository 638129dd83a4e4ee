"""Host planning of a mixed batch: differently sized images in one evaluation call (LitePosePipeline.infer_images with
a list).  Pure host logic, no device work, so that it can be checked without a GPU.

Every image gets, per scale of TEST.SCALE_FACTOR, its own network size, centre and scale from get_multi_scale_size
(reference lib/utils/transforms.py:155-180).  Images whose per-scale network sizes agree form one size group; a group
runs through the network and the glue as an ordinary equal-size batch.  Groups are laid out one after another (first
appearance order, caller order inside a group) in

  * the packed source buffer   (uint8 [h_i][w_i][3] per image),
  * one input arena per scale  (NCHW [3][h_s][w_s] per image: a group's slice is its [n_g,3,h_s,w_s] network input),
  * the det / tag arena        ([J][Hd][Wd] and [J][Hd][Wd][T] per image: a group's slice is the [n_g,J,Hd,Wd] /
                                [n_g,J,Hd,Wd,T] pair the glue writes),

and the ragged parser reads the whole det / tag arena in one chain through per-image descriptors (lp_map_desc_t).
"""
import numpy as np

from .lib.utils import transforms as tf

# include/litepose_b200.h: lp_warp_desc_t, lp_map_desc_t
WARP_DESC = np.dtype([("src_offset", "<i8"), ("src_h", "<i4"), ("src_w", "<i4"), ("minv", "<f8", (6,)),
                      ("dst_offset", "<i8"), ("out_h", "<i4"), ("out_w", "<i4")], align=True)
MAP_DESC = np.dtype([("h", "<i4"), ("w", "<i4"), ("det_offset", "<i8"), ("tag_offset", "<i8")], align=True)
assert WARP_DESC.itemsize == 80 and MAP_DESC.itemsize == 24


def image_shapes(images):
    """[(h, w)] of a list of uint8 [H,W,3] host arrays / tensors; raises on anything else."""
    import torch
    if not isinstance(images, (list, tuple)):
        raise TypeError("infer_images: a uint8 [N,H,W,3] tensor or a list of uint8 [H,W,3] images expected")
    if len(images) == 0:
        raise ValueError("infer_images: empty image list")
    shapes = []
    for i, im in enumerate(images):
        if torch.is_tensor(im):
            dt, shp = im.dtype, tuple(im.shape)
            ok_dtype = dt == torch.uint8
        else:
            im = np.asarray(im)
            dt, shp = im.dtype, im.shape
            ok_dtype = dt == np.uint8
        if not ok_dtype:
            raise TypeError("infer_images: image %d has dtype %s, uint8 expected" % (i, dt))
        if len(shp) != 3 or shp[2] != 3 or shp[0] <= 0 or shp[1] <= 0:
            raise TypeError("infer_images: image %d has shape %r, [H,W,3] expected" % (i, shp))
        shapes.append((int(shp[0]), int(shp[1])))
    return shapes


class Group(object):
    """One size group: ``images`` (caller indices, in arena order), per-scale input sizes ``in_hw[s]`` = (h, w), the
    common det / tag size ``det_hw`` and the group's first position in the arenas ``start``."""

    def __init__(self, key, scales):
        self.key = key
        self.images = []
        self.in_hw = {s: hw for s, hw in zip(scales, key)}
        self.det_hw = None
        self.start = 0

    @property
    def n(self):
        return len(self.images)


class MixedPlan(object):
    """Layout of one mixed batch.  Per arena position p (``order[p]`` = caller index of the image there):
    ``src_off[p]`` bytes, ``in_off[s][p]`` elements of the scale-s input arena, ``det_off[p]`` / ``tag_off[p]`` elements
    of the det / tag arena; ``centers[p]`` / ``scales_[p]`` are what valid.py hands to get_final_preds (the last
    scale's), ``minv[s][p]`` the inverted warp matrix of scale s."""

    def __init__(self, shapes, scales, input_size, project, J, T):
        scales = list(scales)                        # the pipeline's order: largest first
        smin = min(scales)
        self.scales = scales
        self.shapes = list(shapes)
        self.J, self.T = int(J), int(T)
        n = len(shapes)
        per = []
        groups = {}
        for i, (h, w) in enumerate(shapes):
            probe = np.empty((h, w, 3), np.uint8)
            sizes, cs = [], []
            for s in scales:
                (w_r, h_r), c, sc = tf.get_multi_scale_size(probe, input_size, s, smin)
                sizes.append((h_r, w_r))
                cs.append((c, sc))
            key = tuple(sizes)
            per.append((key, cs))
            g = groups.get(key)
            if g is None:
                g = groups[key] = Group(key, scales)
            g.images.append(i)
        self.groups = list(groups.values())
        self.order = [i for g in self.groups for i in g.images]
        self.pos = np.empty(n, np.int64)                # caller index -> arena position
        self.pos[self.order] = np.arange(n)
        self.keys = [per[i][0] for i in range(n)]
        self.center_scale = [per[i][1] for i in range(n)]     # caller order, per scale (center, scale)
        self.src_off = np.zeros(n + 1, np.int64)
        self.in_off = {s: np.zeros(n + 1, np.int64) for s in scales}
        self.det_off = np.zeros(n + 1, np.int64)
        self.tag_off = np.zeros(n + 1, np.int64)
        self.det_hw = np.zeros((n, 2), np.int32)
        self.centers = np.zeros((n, 2), np.float64)
        self.scales_ = np.zeros((n, 2), np.float64)
        self.minv = {s: np.zeros((n, 6), np.float64) for s in scales}
        p = 0
        for g in self.groups:
            g.start = p
            h1, w1 = g.in_hw[1.0]
            hb, wb = g.in_hw[scales[0]]
            g.det_hw = (h1, w1) if project else (hb // 2, wb // 2)
            for i in g.images:
                h, w = shapes[i]
                self.src_off[p + 1] = self.src_off[p] + h * w * 3
                for si, s in enumerate(scales):
                    hs, ws = g.in_hw[s]
                    self.in_off[s][p + 1] = self.in_off[s][p] + 3 * hs * ws
                    c, sc = per[i][1][si]
                    self.minv[s][p] = tf.invert_affine(tf.get_affine_transform(c, sc, 0, (ws, hs)))
                hd, wd = g.det_hw
                self.det_hw[p] = (hd, wd)
                self.det_off[p + 1] = self.det_off[p] + self.J * hd * wd
                self.tag_off[p + 1] = self.tag_off[p] + self.J * hd * wd * self.T
                c, sc = per[i][1][-1]                 # valid.py keeps the last scale's centre / scale
                self.centers[p], self.scales_[p] = c, sc
                p += 1

    @property
    def n(self):
        return len(self.order)

    def warp_desc(self, s):
        """lp_warp_desc_t [N] of scale s (arena order)."""
        d = np.zeros(self.n, WARP_DESC)
        for g in self.groups:
            hs, ws = g.in_hw[s]
            for k, i in enumerate(g.images):
                p = g.start + k
                d[p]["src_offset"] = self.src_off[p]
                d[p]["src_h"], d[p]["src_w"] = self.shapes[i]
                d[p]["minv"] = self.minv[s][p]
                d[p]["dst_offset"] = self.in_off[s][p]
                d[p]["out_h"], d[p]["out_w"] = hs, ws
        return d

    def map_desc(self):
        """lp_map_desc_t [N] of the det / tag arena (arena order)."""
        d = np.zeros(self.n, MAP_DESC)
        d["h"], d["w"] = self.det_hw[:, 0], self.det_hw[:, 1]
        d["det_offset"], d["tag_offset"] = self.det_off[:-1], self.tag_off[:-1]
        return d

    def final_trans(self):
        """[N,6] float64: get_affine_transform(center, scale, 0, [Wd, Hd], inv=1) per image (arena order)."""
        out = []
        for p in range(self.n):
            c, sc = self.center_scale[self.order[p]][-1]
            out.append(tf.get_affine_transform(np.asarray(c), np.asarray(sc), 0,
                                              [int(self.det_hw[p, 1]), int(self.det_hw[p, 0])], inv=1))
        return np.stack(out).reshape(self.n, 6)

    def max_in_hw(self, s):
        return (max(g.in_hw[s][0] for g in self.groups), max(g.in_hw[s][1] for g in self.groups))
