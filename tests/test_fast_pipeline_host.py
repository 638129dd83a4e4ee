"""Host side of the pipeline's fast grouping mode (no GPU): the cfg rules of LitePosePipeline(grouping="fast") and the
unpacking of its per-image payload rows (M persons x J joints x (x, y, val, tag) | person count | KM status)."""
import numpy as np
import pytest
import torch

from litepose_b200 import _lib
from litepose_b200.config import get_cfg
from litepose_b200.pipeline import LitePosePipeline, unpack_fast_payload


def _demo_cfg():
    return get_cfg(input_size=128, flip_test=False, adjust=False, refine=False)


@pytest.mark.parametrize("mutate,reason", [
    (lambda c: setattr(c.DATASET, "MAX_NUM_PEOPLE", 33), "MAX_NUM_PEOPLE=33"),
    (lambda c: setattr(c.TEST, "ADJUST", True), "TEST.ADJUST"),
    (lambda c: setattr(c.TEST, "REFINE", True), "TEST.REFINE"),
])
def test_fast_cfg_refused_with_reason(mutate, reason):
    cfg = _demo_cfg()
    mutate(cfg)
    with pytest.raises(ValueError, match=reason.replace(".", r"\.")):
        LitePosePipeline(None, cfg, grouping="fast")         # refused before the model or the library is touched


def test_fast_cfg_lists_every_reason():
    cfg = get_cfg(input_size=128)                              # the evaluation cfg: adjust and refine on
    with pytest.raises(ValueError) as e:
        LitePosePipeline(None, cfg, grouping="fast")
    assert "ADJUST" in str(e.value) and "REFINE" in str(e.value)


def test_unknown_grouping_refused():
    with pytest.raises(ValueError, match="grouping"):
        LitePosePipeline(None, _demo_cfg(), grouping="greedy")


def _rows(counts, M, J, status=None, seed=0):
    rng = np.random.RandomState(seed)
    rows = np.zeros((len(counts), M * J * 4 + 2), np.float32)
    for i, p in enumerate(counts):
        rows[i, :p * J * 4] = rng.randn(p * J * 4)
        rows[i, -2] = p
        rows[i, -1] = 0 if status is None else status[i]
    return rows


@pytest.mark.parametrize("M,J", [(30, 14), (32, 17), (5, 18)])
def test_unpack_rows(M, J):
    counts = [0, 3, M]
    rows = _rows(counts, M, J)
    for host in (rows, torch.from_numpy(rows)):
        out = unpack_fast_payload(host, M, J)
        assert [p for _, p in out] == counts
        for i, (ans, p) in enumerate(out):
            assert ans.shape == (p, J, 4) and ans.dtype == np.float32
            assert np.array_equal(ans, rows[i, :M * J * 4].reshape(M, J, 4)[:p])
    # the results are copies: the pinned host rows may be reused by the next step
    out = unpack_fast_payload(torch.from_numpy(rows), M, J)
    rows[1, :] = 0
    assert np.any(out[1][0] != 0)


def test_status_one_row_raises():
    rows = _rows([2, 4, 1], 30, 14, status=[0, 1, 0])
    with pytest.raises(_lib.LitePoseError, match="image 1"):
        unpack_fast_payload(rows, 30, 14)
    assert len(unpack_fast_payload(rows[[0, 2]], 30, 14)) == 2


def test_row_width_checked():
    with pytest.raises(ValueError):
        unpack_fast_payload(np.zeros((1, 30 * 14 * 5 + 2), np.float32), 30, 14)
