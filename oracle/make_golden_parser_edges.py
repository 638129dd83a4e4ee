"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates tests/golden/parser_edges.npz: the UNMODIFIED reference's
match_by_tag, HeatmapParser.adjust and HeatmapParser.refine (lib/core/group.py, imported in place through
oracle/refshim.py) on the matcher and refine cases of oracle/parser_cases.py.  Every case stores the SHA-256 of its
seeded inputs, so a test notices when the generators drift from the fixture.  Needs a reference checkout:

    python -m oracle.make_golden_parser_edges
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import parser_cases as pc  # noqa: E402
from oracle import refshim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "parser_edges.npz")
ADJ_REF = ((1, 1), (1, 0), (0, 1), (0, 0))


def matcher_digest(c):
    h = hashlib.sha256(repr((c["J"], c["order"], c["K"], c["T"], c["W"], c["det_thr"], c["tag_thr"], c["use_det_val"],
                             c["ignore"])).encode())
    for k in ("val_k", "ind_k", "tag_k"):
        h.update(np.ascontiguousarray(c[k]).tobytes())
    return h.hexdigest()


def refine_digest(c):
    h = hashlib.sha256()
    for k in ("det", "tag", "ans"):
        h.update(np.ascontiguousarray(c[k]).tobytes())
    return h.hexdigest()


def run_adjust_refine(adjust, refine, c, do_adjust, do_refine):
    """parse()'s tail (group.py:273-291) on one image whose matched persons are c["ans"]: adjust, scores, refine.
    ``adjust(ans_list, det)`` and ``refine(det, tag, keypoints)`` are the reference's methods or the oracle's."""
    det, tag = c["det"], c["tag"]
    ans = [c["ans"].copy()]
    if do_adjust:
        ans = adjust(ans, det[None])
    scores = np.array([i[:, 2].mean() for i in ans[0]], np.float32)
    if do_refine:
        for i in range(len(ans[0])):
            ans[0][i] = refine(det, tag, ans[0][i])
    return np.asarray(ans[0], np.float32), scores


def main():
    ns = refshim.load()
    torch.set_num_threads(1)
    out = {}
    for name, c in pc.matcher_cases():
        params = ns.group.Params.__new__(ns.group.Params)
        for k, v in vars(pc.params_of(c)).items():
            setattr(params, k, v)
        loc = pc.loc_from_ind(c["ind_k"], c["W"])
        ans = ns.group.match_by_tag((c["tag_k"], loc, c["val_k"]), params)
        out["m_%s_in" % name] = np.array(matcher_digest(c))
        out["m_%s_ans" % name] = np.asarray(ans, np.float32).reshape(-1, c["J"], 3 + c["T"])
    cfg_parser = None
    for name, c in pc.refine_cases():
        if cfg_parser is None:
            from litepose_b200.config import get_cfg
            cfg_parser = ns.group.HeatmapParser(get_cfg(input_size=256))
        rp = cfg_parser
        dt, tt = torch.from_numpy(c["det"]), torch.from_numpy(c["tag"])
        tcase = dict(c, det=dt, tag=tt)
        out["r_%s_in" % name] = np.array(refine_digest(c))
        for a, r in ADJ_REF:
            ans, scores = run_adjust_refine(rp.adjust, rp.refine, tcase, a, r)
            out["r_%s_a%d_r%d" % (name, a, r)] = ans
            out["r_%s_scores_a%d" % (name, a)] = scores
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
