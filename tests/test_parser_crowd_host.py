"""CPU: the parser past 64 persons.  oracle/group_ref against the reference's goldens on planted crowds of 80 / 150 /
240 persons at K = 96 / 128 / 256; the Munkres restatement against scipy at sides up to 256; and the one bound
(LP_PARSER_MAX_PEOPLE = 256) that DeviceParser and LitePosePipeline refuse above."""
import os

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

from parity_util import assert_topk_equal
from litepose_b200 import _lib
from litepose_b200.config import get_cfg
from oracle import group_ref
from oracle.make_golden_parser_crowd import CROWD_CASES, crowd_inputs, digest
from oracle.munkres_ref import Munkres


@pytest.mark.parametrize("case", CROWD_CASES, ids=[c[0] for c in CROWD_CASES])
def test_oracle_equals_reference_crowd(golden_dir, case):
    z = np.load(os.path.join(golden_dir, "parser_crowd_%s.npz" % case[0]))
    cfg, (det, tag) = crowd_inputs(case)
    assert digest(det, tag) == str(z["in_digest"])
    op = group_ref.HeatmapParser(cfg)
    assert_topk_equal(op.top_k(det[None], tag[None]), {k: z[k] for k in ("val_k", "loc_k", "tag_k")}, case[0])
    ans, scores = op.parse(det[None].copy(), tag[None].copy(), True, True)
    a = np.asarray(ans[0], np.float32).reshape(-1, cfg.DATASET.NUM_JOINTS, 3 + case[3])
    assert a.shape == z["ans"].shape and a.shape[0] > 64, (a.shape, z["ans"].shape)
    assert np.array_equal(a.view(np.uint32), z["ans"].view(np.uint32))
    assert np.array_equal(np.asarray(scores, np.float32).view(np.uint32), z["scores"].view(np.uint32))


@pytest.mark.parametrize("n,kind,seed", [(65, "int", 1), (128, "int", 2), (200, "tag", 3), (256, "tag", 4),
                                         (256, "real", 5)])
def test_munkres_ref_large_vs_scipy(n, kind, seed):
    """total cost of the restated Munkres = scipy's optimum: integer costs with many ties, the matcher's own form
    round(d) * 100 - val, and real-valued costs (step 6 with non-integer minima)"""
    rs = np.random.RandomState(seed)
    if kind == "int":
        c = rs.randint(0, 5, size=(n, n)).astype(np.float64)
    elif kind == "tag":
        d = np.abs(rs.randn(n, 1) * 3 - rs.randn(1, n) * 3)
        c = np.rint(d) * 100 - rs.rand(n, 1)
    else:
        c = rs.rand(n, n)
    res = Munkres().compute(c.tolist())
    rows, cols = zip(*res)
    assert sorted(rows) == list(range(n)) and sorted(cols) == list(range(n))
    r, k = linear_sum_assignment(c)
    got = sum(c[i, j] for i, j in res)
    assert abs(got - c[r, k].sum()) <= 1e-9 * max(1.0, abs(c[r, k].sum()))


def _parser_args(k):
    return (14, k, 0.1, 1.0, True, False, list(range(14)), 5, 2)


def test_bound_is_the_kernels_bound():
    """the host's bound is the header's; the ragged entry points refuse K above it before touching the device (fake
    pointers, empty workspace: K = 256 gets as far as the workspace check), the uniform ones keep K <= 64"""
    from litepose_b200.parser import PARSER_MAX_PEOPLE
    assert PARSER_MAX_PEOPLE == 256
    lib = _lib.load()
    hw = np.array([[64, 64]], np.int32)
    for k, rc in ((257, 1), (256, 5), (65, 5)):
        assert lib.lp_nms_topk_ragged_f32(8, 8, 1, hw.ctypes.data, 8, 14, 2, 5, k, 0.1, 8, 8, 8, 8, 0, None) == rc
        if rc == 1:
            assert b"LP_PARSER_MAX_PEOPLE" in lib.lp_last_error()
        assert lib.lp_tag_match_ragged_f32(8, 8, 8, 1, 14, k, 2, 8, 8, 0.1, 1.0, 1, 0, k, 14 * k, 8, 8, 8, 0,
                                           None) == rc
        if rc == 1:
            assert b"LP_PARSER_MAX_PEOPLE=256" in lib.lp_last_error()
    assert lib.lp_nms_topk_f32(8, 8, 1, 14, 64, 64, 2, 5, 65, 0.1, 8, 8, 8, 8, 0, None) == 1
    assert b"lp_nms_topk_ragged_f32" in lib.lp_last_error()
    assert lib.lp_nms_topk_f32(8, 8, 1, 14, 64, 64, 2, 5, 64, 0.1, 8, 8, 8, 8, 0, None) == 5


def test_device_parser_bound():
    from litepose_b200.parser import DeviceParser
    assert DeviceParser(*_parser_args(256)).K == 256
    assert DeviceParser(*_parser_args(65)).pcap == 14 * 65
    with pytest.raises(ValueError, match=r"MAX_NUM_PEOPLE=257 exceeds LP_PARSER_MAX_PEOPLE=256"):
        DeviceParser(*_parser_args(257))


def test_pipeline_bound():
    from litepose_b200.pipeline import LitePosePipeline
    cfg = get_cfg(input_size=256)
    cfg.DATASET.MAX_NUM_PEOPLE = 256
    LitePosePipeline._validate_cfg(cfg)
    cfg.DATASET.MAX_NUM_PEOPLE = 257
    with pytest.raises(ValueError, match=r"LP_PARSER_MAX_PEOPLE=256"):
        LitePosePipeline._validate_cfg(cfg)
    with pytest.raises(ValueError, match=r"LP_PARSER_MAX_PEOPLE=256"):
        LitePosePipeline(None, cfg)


def test_dropin_parser_bound():
    from litepose_b200.lib.core.group import HeatmapParser
    cfg = get_cfg(input_size=256)
    cfg.DATASET.MAX_NUM_PEOPLE = 256
    assert HeatmapParser(cfg).device_parser.K == 256
    cfg.DATASET.MAX_NUM_PEOPLE = 257
    with pytest.raises(ValueError, match=r"LP_PARSER_MAX_PEOPLE=256"):
        HeatmapParser(cfg)


def test_fast_grouping_keeps_its_32():
    from litepose_b200.pipeline import LitePosePipeline
    cfg = get_cfg(input_size=256)
    cfg.DATASET.MAX_NUM_PEOPLE = 33
    cfg.TEST.ADJUST = cfg.TEST.REFINE = False
    with pytest.raises(ValueError, match="32 persons"):
        LitePosePipeline._validate_fast_cfg(cfg)
