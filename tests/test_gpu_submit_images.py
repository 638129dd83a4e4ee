"""-m gpu: the asynchronous list API (LitePosePipeline.submit_images / collect_images).  Per list the collected result
equals infer_images on the same list, element for element: two lists of different compositions in flight, interleaved
with the equal-size entry points, crowds past ``keep``, the per-slot memory bound, the refusals, and the two-rank
gather of a sharded list."""
import numpy as np
import pytest
import torch

from litepose_b200 import synth
from litepose_b200.config import get_arch, get_cfg
from litepose_b200.lib.models.pose_mobilenet import get_pose_net
from litepose_b200.mixed import MixedPlan
from litepose_b200.pipeline import ImagesTicket, LitePosePipeline, PlantedCrowd

pytestmark = pytest.mark.gpu

SIZE = 128
# at INPUT_SIZE 128: 128x192, 192x128, 128x384, 128x128, 384x128 and 128x320 network inputs (six size groups)
POOL = [(150, 200), (200, 150), (100, 300), (120, 120), (300, 100), (90, 200), (201, 149)]
LIST_A = [(150, 200), (200, 150), (150, 200), (100, 300), (120, 120), (300, 100), (90, 200), (201, 149)]
LIST_B = [(300, 100), (90, 200), (120, 120), (200, 150), (100, 300), (150, 200), (90, 200)]


def _images(shapes, seed):
    rng = np.random.RandomState(seed)
    return [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]


def _cfg_case(name):
    from oracle.make_golden import glue_cfg
    if name in ("shipped", "crowd"):
        return get_cfg(input_size=SIZE)
    if name == "nano":
        cfg = get_cfg(input_size=SIZE)
        cfg.TEST.FLIP_TEST = cfg.TEST.ADJUST = cfg.TEST.REFINE = False
        return cfg
    if name == "multiscale":
        cfg = get_cfg(input_size=SIZE)
        cfg.TEST.SCALE_FACTOR = [0.5, 1, 2]
        return cfg
    if name == "coco":
        return glue_cfg(False, False, True, True, size=SIZE, dataset="coco")
    if name == "shared_tag":
        return glue_cfg(False, True, False, True, size=SIZE)
    if name.startswith("fast"):
        coco = name == "fast_coco"
        cfg = glue_cfg(False, True, not coco, True, size=SIZE, dataset="coco" if coco else "crowd_pose")
        cfg.TEST.FLIP_TEST = not coco
        cfg.TEST.ADJUST = cfg.TEST.REFINE = False
        cfg.TEST.SCALE_FACTOR = [0.5, 1, 2] if coco else [1]
        return cfg
    raise KeyError(name)


def _pipe(cfg, keep=64, grouping="ae"):
    torch.manual_seed(0)
    model = synth.scale_heads_(synth.randomize_bn_(get_pose_net(cfg, False, get_arch("XS")), 1)).eval()
    return LitePosePipeline(model.cuda(), cfg, use_graphs=True, keep=keep, grouping=grouping)


def _plants(pipe, shapes, people=3, seed=40):
    """One batch-1 PlantedCrowd per image (the fifth without one), sized to the image's det / tag maps."""
    J, t = pipe.params.num_joints, pipe.T
    mp = MixedPlan(shapes, pipe.scales, SIZE, pipe.project, J, t)
    out = []
    for i in range(len(shapes)):
        if i == 4:
            out.append(None)
            continue
        hd, wd = mp.det_hw[mp.pos[i]]
        pl = PlantedCrowd(1, J, int(hd), int(wd), t, num_people=people, seed=seed + i, device="cuda")
        if pipe.tag_shared:
            pl.tidx, pl.tval = pl.tidx[:0], pl.tval[:0]          # the tag patches index J maps: heat peaks only
        out.append(pl)
    return out


def _same(got, exp, what=""):
    assert len(got) == len(exp), what
    for i, (g, e) in enumerate(zip(got, exp)):
        assert len(g) == len(e) and g[-1] == e[-1], (what, i)
        assert g[0].dtype == e[0].dtype and np.array_equal(g[0], e[0]), (what, i)
        if len(e) == 3:
            assert np.array_equal(np.asarray(g[1], np.float32), np.asarray(e[1], np.float32)), (what, i)


CASES = ["shipped", "nano", "multiscale", "coco", "shared_tag", "fast", "fast_coco"]


@pytest.mark.parametrize("case", CASES)
def test_two_lists_in_flight_equal_infer_images(case):
    """Two lists of different compositions in flight at once; each collect equals infer_images on its list (ae: keep 2,
    so planted crowds overflow the payload and are read in full from the slot's own parser buffers)."""
    cfg = _cfg_case(case)
    fast = case.startswith("fast")
    pipe = _pipe(cfg, keep=2, grouping="fast" if fast else "ae")
    assert len(MixedPlan(LIST_A, pipe.scales, SIZE, pipe.project, pipe.params.num_joints, pipe.T).groups) >= 5
    a, b = _images(LIST_A, 1), [torch.from_numpy(im).cuda() for im in _images(LIST_B, 2)]
    pa, pb = _plants(pipe, LIST_A, seed=40), _plants(pipe, LIST_B, seed=60)
    exp_a, exp_b = pipe.infer_images(a, plant=pa), pipe.infer_images(b, plant=pb)
    assert sum(r[-1] for r in exp_a) > 0 and sum(r[-1] for r in exp_b) > 0
    for _ in range(2):
        ta = pipe.submit_images(a, plant=pa)
        tb = pipe.submit_images(b, plant=pb)
        _same(pipe.collect_images(ta), exp_a, case)
        _same(pipe.collect_images(tb), exp_b, case)


def test_crowd_past_keep_returned_in_full():
    """A planted crowd of 12 persons per image against keep=4: without a group every person comes back, from the
    parser buffers of the slot that ran the list, also while a second list is in flight."""
    cfg = _cfg_case("crowd")
    pipe = _pipe(cfg, keep=4)
    imgs = _images(LIST_A, 5)
    plants = _plants(pipe, LIST_A, people=12, seed=80)
    exp = pipe.infer_images(imgs, plant=plants)
    assert max(r[2] for r in exp) > pipe.keep
    other = _images(LIST_B, 6)
    t0 = pipe.submit_images(imgs, plant=plants)
    t1 = pipe.submit_images(other)
    _same(pipe.collect_images(t0), exp)
    _same(pipe.collect_images(t1), pipe.infer_images(other))


def test_interleaved_with_equal_size_entry_points():
    """Outstanding list tickets interleaved with step, submit / collect and infer_images (batch and list): every result
    equals the one each call gives alone."""
    cfg = _cfg_case("shipped")
    pipe = _pipe(cfg)                            # keep 64: submit() / collect() refuse an overflowing payload
    J, n = pipe.params.num_joints, 2
    hd = SIZE if pipe.project else SIZE // 2
    plant = PlantedCrowd(n, J, hd, hd, pipe.T, num_people=3, seed=9, device="cuda")
    fr = synth.make_frames(n, SIZE, seed=4).half().pin_memory()
    batch = torch.from_numpy(np.stack(_images([(SIZE, SIZE)] * n, 3))).pin_memory()
    a, b, c = _images(LIST_A, 1), _images(LIST_B, 2), _images(POOL, 3)
    pa = _plants(pipe, LIST_A)
    ref_step = pipe.step(fr, plant)
    ref_batch = pipe.infer_images(batch)
    ref_a, ref_b, ref_c = pipe.infer_images(a, plant=pa), pipe.infer_images(b), pipe.infer_images(c)
    t0 = pipe.submit(fr, plant)
    ref_sub = pipe.collect(t0)[0]
    _same(ref_sub, ref_step)

    ta = pipe.submit_images(a, plant=pa)
    got_step = pipe.step(fr, plant)
    t1 = pipe.submit(fr, plant)
    tb = pipe.submit_images(b)
    got_batch = pipe.infer_images(batch)
    got_c = pipe.infer_images(c)                 # the blocking list form while two lists are outstanding
    got_sub = pipe.collect(t1)[0]
    got_a = pipe.collect_images(ta)
    tc = pipe.submit_images(c)
    got_step2 = pipe.step(fr, plant)
    got_b = pipe.collect_images(tb)
    got_c2 = pipe.collect_images(tc)
    for got, exp, what in [(got_step, ref_step, "step"), (got_sub, ref_step, "submit"), (got_batch, ref_batch, "batch"),
                           (got_c, ref_c, "list"), (got_a, ref_a, "ticket a"), (got_step2, ref_step, "step 2"),
                           (got_b, ref_b, "ticket b"), (got_c2, ref_c, "ticket c")]:
        _same(got, exp, what)


def test_refusals():
    cfg = _cfg_case("shipped")
    pipe = _pipe(cfg)
    a = _images(LIST_A[:3], 1)
    t0 = pipe.submit_images(a)
    t1 = pipe.submit_images(a)
    with pytest.raises(RuntimeError):
        pipe.submit_images(a)                   # a third list while two are outstanding
    exp = pipe.infer_images(a)
    _same(pipe.collect_images(t0), exp)
    with pytest.raises(RuntimeError):
        pipe.collect_images(t0)                 # already collected
    with pytest.raises(RuntimeError):
        pipe.collect_images(ImagesTicket(pipe, 0, 12345))       # never submitted
    with pytest.raises(RuntimeError):
        pipe.collect_images(ImagesTicket(_pipe(cfg), 1, t1.serial))    # another pipeline's ticket
    with pytest.raises(TypeError):
        pipe.collect_images(1)                  # a ticket of submit()
    _same(pipe.collect_images(t1), exp)
    t2 = pipe.submit_images(a)                  # a slot is free again
    _same(pipe.collect_images(t2), exp)
    with pytest.raises(ValueError):
        pipe.submit_images(a, group=object())   # a group needs the shard plan
    with pytest.raises(ValueError):
        pipe.submit_images(a, plant=[None])


def test_per_slot_memory_bound():
    """After each slot has served a list that holds the largest group and the most images, 24 lists of other
    compositions, two in flight at a time, grow neither the device memory nor the number of plans."""
    from litepose_b200.engine import ARENA_PLANS
    cfg = _cfg_case("shipped")
    pipe = _pipe(cfg)
    rng = np.random.RandomState(5)
    first = POOL * 8                               # every group at least as large as in any list below
    t0 = pipe.submit_images(_images(first, 1))
    t1 = pipe.submit_images(_images(first, 2))
    pipe.collect_images(t0)
    pipe.collect_images(t1)
    torch.cuda.synchronize()
    mem0 = torch.cuda.memory_allocated()
    plans0 = len(pipe.engine.plans)
    pending = []
    for b in range(24):
        k = rng.randint(3, 9)
        shapes = [POOL[j] for j in rng.randint(0, len(POOL), k)]
        pending.append((pipe.submit_images(_images(shapes, 10 + b)), k))
        if len(pending) == 2:
            tk, kk = pending.pop(0)
            assert len(pipe.collect_images(tk)) == kk
            torch.cuda.synchronize()
            assert torch.cuda.memory_allocated() <= mem0, b
            assert len(pipe.engine.plans) == plans0 and len(pipe.engine.arena_plans) <= ARENA_PLANS
    for tk, kk in pending:
        assert len(pipe.collect_images(tk)) == kk
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= mem0


# -- two ranks: a sharded list, one gather, merged on dst ------------------------------------------------------------
TWO_RANK_SHAPES = LIST_A + LIST_B


def _two_rank_worker(rank, port, q):
    import os
    import torch.distributed as dist
    from litepose_b200.dist import merge_shards, plan_shards
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=2)
    try:
        cfg = _cfg_case("shipped")
        pipe = _pipe(cfg)
        imgs = _images(TWO_RANK_SHAPES, 11)
        plants = _plants(pipe, TWO_RANK_SHAPES, seed=90)
        plan = plan_shards(TWO_RANK_SHAPES, cfg, 2)
        mine = plan.indices[rank]
        tk = pipe.submit_images([imgs[i] for i in mine], plant=[plants[i] for i in mine], group=dist.group.WORLD,
                                dst=0, plan=plan)
        res = pipe.collect_images(tk)
        if rank == 0:
            merged = merge_shards(res, plan)
            full = pipe.infer_images(imgs, plant=plants)
            pack = lambda rs: [(r[0].tolist(), np.asarray(r[1], np.float32).tolist(), r[2]) for r in rs]
            q.put((rank, plan.counts, pack(merged), pack(full)))
        else:
            q.put((rank, plan.counts, res, None))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (one rank per GPU, NCCL gather)")
def test_two_rank_sharded_list_equals_one_process():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_two_rank_worker, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        out = {}
        for _ in range(2):
            rank, counts, merged, full = q.get(timeout=600)
            out[rank] = (counts, merged, full)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    assert out[1][1] is None
    counts, merged, full = out[0]
    assert sum(counts) == len(TWO_RANK_SHAPES) and min(counts) > 0
    assert len(merged) == len(full)
    for i, (g, e) in enumerate(zip(merged, full)):
        assert g == e, i
