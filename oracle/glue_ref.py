"""ORACLE (test infrastructure, not product code).

CPU fp32 restatement of the test-time glue between model and parser:
``get_multi_stage_outputs`` (reference lib/core/inference.py:75-173) and
``aggregate_results`` (:176-208), single scale (``aggregate``) and the multi-scale loop of
valid.py:205-225 (``multi_scale``); floating point, so torch fp32 CPU ops.

The x2 bilinear resamples are written out explicitly (SURVEY Appendix A.4:
``align_corners=False``; out[2m] = .25*x[m-1] + .75*x[m], out[2m+1] = .75*x[m] +
.25*x[m+1], edge-clamped) rather than through F.interpolate, so the restatement is
independent of the op the reference calls; other ratios fall back to the general
rule.  Pinned against the real reference's outputs in tests/test_oracle_golden.py.
"""
import torch

from litepose_b200.config import flip_index_for


def _up_axis(x, out_size, dim):
    n_in = x.shape[dim]
    dst = torch.arange(out_size, dtype=torch.float32)
    # area_pixel_compute_source_index, align_corners=False, clamped at 0
    src = ((dst + 0.5) * (float(n_in) / float(out_size)) - 0.5).clamp_(min=0.0)
    i0 = src.floor().long().clamp_(max=n_in - 1)
    i1 = (i0 + 1).clamp_(max=n_in - 1)
    l1 = src - i0.float()
    l0 = 1.0 - l1
    shape = [1] * x.dim()
    shape[dim] = out_size
    return x.index_select(dim, i0) * l0.view(shape) + x.index_select(dim, i1) * l1.view(shape)


def bilinear(x, size):
    """F.interpolate(x, size=(H,W), mode='bilinear', align_corners=False): the
    torch CPU kernel interpolates with weights (h0,h1) x (w0,w1) on the four
    neighbours; separable form agrees within 1 ulp-level rounding."""
    h, w = int(size[0]), int(size[1])
    if x.shape[2] == h and x.shape[3] == w:
        return x
    return _up_axis(_up_axis(x, w, 3), h, 2)


def multi_stage_outputs(cfg, model, image, with_flip=False, project2image=False, size_projected=None):
    """inference.py:75-173.  ``model`` is any callable image -> [out0, out1]."""
    nj = cfg.DATASET.NUM_JOINTS
    heatmaps, tags = [], []
    fidx = flip_index_for(cfg) if with_flip else None

    def one_pass(outs, flipped):
        avg, cnt = 0, 0
        collected = []
        for i, o in enumerate(outs):
            if len(outs) > 1 and i != len(outs) - 1:
                o = bilinear(o, (outs[-1].shape[2], outs[-1].shape[3]))
            if flipped:
                o = torch.flip(o, [3])
            collected.append(o)
            off = nj if cfg.LOSS.WITH_HEATMAPS_LOSS[i] else 0
            if cfg.LOSS.WITH_HEATMAPS_LOSS[i] and cfg.TEST.WITH_HEATMAPS[i]:
                hm = o[:, :nj]
                if flipped:
                    hm = hm[:, fidx]
                avg = avg + hm
                cnt += 1
            if cfg.LOSS.WITH_AE_LOSS[i] and cfg.TEST.WITH_AE[i]:
                tg = o[:, off:]
                if flipped and cfg.MODEL.TAG_PER_JOINT:
                    tg = tg[:, fidx]
                tags.append(tg)
        if cnt > 0:
            heatmaps.append(avg / cnt)
        return collected

    outputs = one_pass(model(image), False)
    if with_flip:
        outputs = outputs + one_pass(model(torch.flip(image, [3])), True)
    if cfg.DATASET.WITH_CENTER and cfg.TEST.IGNORE_CENTER:
        heatmaps = [h[:, :-1] for h in heatmaps]
        tags = [t[:, :-1] for t in tags]
    if project2image and size_projected:
        sz = (size_projected[1], size_projected[0])
        heatmaps = [bilinear(h, sz) for h in heatmaps]
        tags = [bilinear(t, sz) for t in tags]
    return outputs, heatmaps, tags


def aggregate(cfg, heatmaps, tags):
    """inference.py:176-208 for one scale (final_heatmaps None on entry) followed by
    valid.py:224-225: returns (final_heatmaps [N,J,H,W], tags [N,J,H,W,T])."""
    tags_list = [t.unsqueeze(4) for t in tags]
    hm = (heatmaps[0] + heatmaps[1]) / 2.0 if cfg.TEST.FLIP_TEST else heatmaps[0]
    hm = hm / float(len(cfg.TEST.SCALE_FACTOR))
    return hm, torch.cat(tags_list, dim=4)


def aggregate_results(cfg, scale_factor, final_heatmaps, tags_list, heatmaps, tags):
    """inference.py:176-208, one scale of the multi-scale loop."""
    if scale_factor == 1 or len(cfg.TEST.SCALE_FACTOR) == 1:
        if final_heatmaps is not None and not cfg.TEST.PROJECT2IMAGE:
            tags = [bilinear(t, final_heatmaps.shape[2:4]) for t in tags]
        for t in tags:
            tags_list.append(t.unsqueeze(4))
    avg = (heatmaps[0] + heatmaps[1]) / 2.0 if cfg.TEST.FLIP_TEST else heatmaps[0]
    if final_heatmaps is None:
        final_heatmaps = avg
    elif cfg.TEST.PROJECT2IMAGE:
        final_heatmaps = final_heatmaps + avg
    else:
        final_heatmaps = final_heatmaps + bilinear(avg, final_heatmaps.shape[2:4])
    return final_heatmaps, tags_list


def multi_scale(cfg, model, images, base_size):
    """valid.py:205-225: ``images`` maps every scale of TEST.SCALE_FACTOR to its resized image batch; scales are
    visited largest first; returns (final_heatmaps [N,J,H,W], tags [N,J,H,W,T])."""
    final, tags_list = None, []
    scales = sorted(cfg.TEST.SCALE_FACTOR, reverse=True)
    for s in scales:
        _, hms, tgs = multi_stage_outputs(cfg, model, images[s], cfg.TEST.FLIP_TEST, cfg.TEST.PROJECT2IMAGE, base_size)
        final, tags_list = aggregate_results(cfg, s, final, tags_list, hms, tgs)
    final = final / float(len(scales))
    return final, torch.cat(tags_list, dim=4)
