"""Host logic of the asynchronous list API across GPUs: the cost-balanced shard plan of a mixed-size list
(litepose_b200.dist.plan_shards), the merge back into the caller's order, and a world_size-2 gloo run of the padded
row gather with unequal shard lengths."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from litepose_b200.config import get_cfg
from litepose_b200.dist import gather_rows, merge_shards, plan_shards, split_rows
from litepose_b200.mixed import MixedPlan, group_order

POOL = [(480, 640), (640, 480), (427, 640), (640, 427), (333, 500), (612, 612), (375, 500), (500, 375), (120, 900),
        (64, 64)]


def _cfg(scales=(1,), flip=True, size=512):
    cfg = get_cfg(input_size=size)
    cfg.TEST.SCALE_FACTOR = list(scales)
    cfg.TEST.FLIP_TEST = flip
    return cfg


def _shapes(n, seed):
    rng = np.random.RandomState(seed)
    return [POOL[k] for k in rng.randint(0, len(POOL), n)]


@pytest.mark.parametrize("scales,flip", [((1,), True), ((0.5, 1, 2), False)])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_plan_shards_cover_balance_determinism(scales, flip, world):
    cfg = _cfg(scales, flip)
    order = sorted((float(s) for s in scales), reverse=True)
    for seed, n in [(0, 1), (1, 5), (2, 32), (3, 67)]:
        shapes = _shapes(n, seed)
        plan = plan_shards(shapes, cfg, world)
        again = plan_shards(list(shapes), cfg, world)
        assert plan.indices == again.indices and plan.rows == again.rows
        assert plan.world == world and len(plan.indices) == world
        assert sorted(i for ix in plan.indices for i in ix) == list(range(n))
        assert plan.counts == [len(ix) for ix in plan.indices] and plan.rows == max(plan.counts)
        # cost: network input pixels over TEST.SCALE_FACTOR (the sizes MixedPlan lays out), doubled under flip
        mp_all = MixedPlan(shapes, order, 512, True, 14, 2)
        exp = [(2 if flip else 1) * sum(h * w for h, w in mp_all.keys[i]) for i in range(n)]
        assert plan.costs == exp
        assert max(plan.load) - min(plan.load) <= max(exp)
        for ix in plan.indices:
            if ix:
                # each shard is listed in the arena order its pipeline lays it out in
                sub = MixedPlan([shapes[i] for i in ix], order, 512, True, 14, 2)
                assert sub.order == list(range(len(ix)))


def test_plan_shards_refuses_bad_input():
    with pytest.raises(ValueError):
        plan_shards([], _cfg(), 2)
    with pytest.raises(ValueError):
        plan_shards([(10, 10)], _cfg(), 0)


def test_group_order_is_mixed_plan_order():
    shapes = _shapes(40, 9)
    mp_ = MixedPlan(shapes, [2.0, 1.0, 0.5], 256, False, 14, 2)
    assert group_order(mp_.keys) == mp_.order
    grouped = [mp_.keys[i] for i in mp_.order]
    assert group_order(grouped) == list(range(len(grouped)))


def test_merge_shards_restores_caller_order():
    shapes = _shapes(23, 4)
    plan = plan_shards(shapes, _cfg(), 3)
    per_rank = [[("img", i) for i in ix] for ix in plan.indices]
    assert merge_shards(per_rank, plan) == [("img", i) for i in range(23)]
    with pytest.raises(ValueError):
        merge_shards(per_rank[:2], plan)
    with pytest.raises(ValueError):
        merge_shards([per_rank[0][:-1]] + per_rank[1:], plan)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


# one large image against many small ones: the cost balance gives the two ranks shards of different lengths
GATHER_SHAPES = [(900, 900)] + [(100, 100)] * 5 + [(480, 640)]
WIDTH = 9


def _rows_of(plan, rank):
    """Rank ``rank``'s padded [rows, WIDTH] payload: row k carries caller index plan.indices[rank][k]; padding -7."""
    rows = torch.full((plan.rows, WIDTH), -7.0)
    for k, i in enumerate(plan.indices[rank]):
        rows[k] = torch.arange(WIDTH, dtype=torch.float32) + 100.0 * i
    return rows


def _gather_worker(rank, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    try:
        plan = plan_shards(GATHER_SHAPES, _cfg(), 2)
        out = torch.empty((2, plan.rows, WIDTH)) if rank == 0 else None
        got = gather_rows(_rows_of(plan, rank), out, dst=0)
        q.put((rank, None if got is None else [r.numpy().copy() for r in split_rows(got, plan)]))
    finally:
        dist.destroy_process_group()


def test_padded_row_gather_world2_gloo():
    plan = plan_shards(GATHER_SHAPES, _cfg(), 2)
    assert plan.counts[0] != plan.counts[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gather_worker, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=120) for _ in range(2))
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    assert res[1] is None
    got = res[0]
    assert [g.shape[0] for g in got] == plan.counts
    for r in range(2):
        assert np.array_equal(got[r], _rows_of(plan, r)[:plan.counts[r]].numpy())
    merged = merge_shards([list(g) for g in got], plan)
    for i, row in enumerate(merged):
        assert np.array_equal(row, np.arange(WIDTH, dtype=np.float32) + 100.0 * i)
