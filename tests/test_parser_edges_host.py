"""CPU: the parser edge cases of oracle/parser_cases.py.  The oracle (oracle/group_ref.py) equals, bit for bit, the
unmodified reference's match_by_tag / adjust / refine on every case (tests/golden/parser_edges.npz); the case list
reaches every hard branch of the matcher and of the Munkres solver; and the oracle's top-K applies the NaN rule the
device kernel follows (NaN never takes a slot, a NaN in a pixel's window suppresses it)."""
import collections
import os

import numpy as np
import pytest

from oracle import group_ref
from oracle import parser_cases as pc
from oracle.make_golden_parser_edges import ADJ_REF, matcher_digest, refine_digest, run_adjust_refine
from oracle.munkres_ref import Munkres


@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "parser_edges.npz"))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", pc.MATCHER_NAMES)
def test_matcher_oracle_equals_reference(fixture, name):
    c = dict(pc.matcher_cases())[name]
    assert matcher_digest(c) == str(fixture["m_%s_in" % name]), "case generator drifted from the fixture"
    ans = group_ref.match_by_tag((c["tag_k"], pc.loc_from_ind(c["ind_k"], c["W"]), c["val_k"]), pc.params_of(c))
    got = np.asarray(ans, np.float32).reshape(-1, c["J"], 3 + c["T"])
    exp = fixture["m_%s_ans" % name]
    assert got.shape == exp.shape
    assert np.array_equal(_bits(got), _bits(exp))


@pytest.mark.parametrize("name", [c[0] for c in pc.REFINE_CASES])
def test_adjust_refine_oracle_equals_reference(fixture, name):
    c = dict(pc.refine_cases())[name]
    assert refine_digest(c) == str(fixture["r_%s_in" % name]), "case generator drifted from the fixture"
    for a, r in ADJ_REF:
        ans, scores = run_adjust_refine(group_ref.adjust, group_ref.refine, c, a, r)
        exp = fixture["r_%s_a%d_r%d" % (name, a, r)]
        assert np.array_equal(_bits(ans), _bits(exp)), (a, r)
        assert np.array_equal(_bits(scores), _bits(fixture["r_%s_scores_a%d" % (name, a)])), a


class CountingMunkres(Munkres):
    """munkres_ref.Munkres that records which of its hard paths a cost matrix takes."""
    events = collections.Counter()

    def _step5(self):
        self._primes = 1
        r = super()._step5()
        if self._primes >= 2:
            self.events["augment_2_primes"] += 1
        return r

    def _find_prime_in_row(self, row):
        self._primes += 1
        return super()._find_prime_in_row(row)

    def _step6(self):
        vals = [self.C[i][j] for i in range(self.n) for j in range(self.n)
                if not self.row_covered[i] and not self.col_covered[j]]
        if vals and min(vals) != int(min(vals)):
            self.events["step6_non_integer"] += 1
        return super()._step6()

    def _find_a_zero(self, i0, j0):
        row, col = super()._find_a_zero(i0, j0)
        if row >= 0:
            if col < j0 or row < i0:
                self.events["zero_after_wrap"] += 1
            zeros = [j for j in range(self.n)
                     if self.C[row][j] == 0 and not self.col_covered[j] and not self.row_covered[row]]
            if len(zeros) > 1:
                self.events["row_with_several_zeros"] += 1
        return row, col


def test_cases_reach_every_hard_branch():
    CountingMunkres.events = collections.Counter()
    ev = collections.Counter()
    for name, c in pc.matcher_cases():
        group_ref.match_by_tag((c["tag_k"], pc.loc_from_ind(c["ind_k"], c["W"]), c["val_k"]), pc.params_of(c),
                               solver=CountingMunkres, events=ev)
    ev.update(CountingMunkres.events)
    need = ["step6_non_integer", "augment_2_primes", "zero_after_wrap", "row_with_several_zeros", "key_collision",
            "ignore_too_much_skip", "pad_rows", "pad_cols", "round_half_tie", "dist_eq_threshold"]
    missing = [k for k in need if ev[k] == 0]
    assert not missing, (missing, dict(ev))


def test_refine_cases_reach_their_edges():
    """the refine cases hold what they are named for: > 32 persons missing one joint, T = 1..4, persons with 1 and
    J-1 detected joints, keypoints on every border"""
    cs = dict(pc.refine_cases())
    miss = (cs["many_missing_t2"]["ans"][:, 3, 2] == 0).sum()
    assert miss > 32
    assert {c["T"] for c in cs.values()} == {1, 2, 3, 4}
    det_counts = (cs["one_and_most_t2"]["ans"][:, :, 2] > 0).sum(axis=1)
    assert 1 in det_counts and cs["one_and_most_t2"]["J"] - 1 in det_counts
    b = cs["borders_t2"]
    xy = b["ans"][b["ans"][:, :, 2] > 0][:, :2]
    H, W = b["det"].shape[1:]
    assert {(0, 0), (W - 1, H - 1), (0, H - 1), (W - 1, 0)} <= {(int(x), int(y)) for x, y in xy}


def _nan_rule_topk(det, kernel, K):
    """The canonical top-K written out plainly: a pixel survives iff it is > 0, its k x k window (-inf outside the
    map) holds no NaN and it equals the window maximum; survivors ordered by value desc, flat index asc."""
    n, j, h, w = det.shape
    R = kernel // 2
    pad = np.full((n, j, h + 2 * R, w + 2 * R), -np.inf, np.float32)
    pad[:, :, R:R + h, R:R + w] = det
    win = np.stack([pad[:, :, dy:dy + h, dx:dx + w] for dy in range(kernel) for dx in range(kernel)])
    has_nan = np.isnan(win).any(axis=0)
    wmax = np.where(np.isnan(win), -np.inf, win).max(axis=0)
    keep = (det > 0) & ~has_nan & (det == wmax)
    val = np.zeros((n, j, K), np.float32)
    ind = np.zeros((n, j, K), np.int64)
    for a in range(n):
        for b in range(j):
            flat = np.nonzero(keep[a, b].reshape(-1))[0]
            v = det[a, b].reshape(-1)[flat]
            o = np.lexsort((flat, -v.astype(np.float64)))[:K]
            val[a, b, :o.size], ind[a, b, :o.size] = v[o], flat[o]
    return val, ind


@pytest.mark.parametrize("name", ["nan_window_k3", "nan_window_k5", "nan_window_k7", "nan_window_k9", "specials",
                                  "specials_k3_scalar", "k9_scalar", "subnormal_thr0"])
def test_oracle_topk_nan_rule(name):
    (_, det, tag, kernel, K, mv), = [c for c in pc.topk_cases() if c[0] == name]
    val, ind, _ = pc.expected_topk(group_ref, det, tag, kernel, K, mv)
    ev, ei = _nan_rule_topk(det, kernel, K)
    assert np.array_equal(_bits(val), _bits(ev)) and np.array_equal(ind, ei)
    assert not np.isnan(val).any()
    if name.startswith("nan_window"):
        # every peak with a NaN in its window is gone, the clean ones are all there
        assert (val == np.float32(0.9)).sum() == 0 and ((val == np.float32(0.7)).sum(axis=2) == 4).all()
