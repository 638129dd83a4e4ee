"""Multi-GPU plumbing: frames are independent, so ranks shard the batch with no data-path
collective; one gather of the packed fixed-capacity keypoint payload per batch follows
(SURVEY.md §8e).  Mixed-size lists are sharded by network cost (plan_shards) and gathered as
padded rows of a length every rank knows (gather_rows).  Backend: NCCL over NVLink on the GPU
box, gloo in the CPU tests."""
import torch
import torch.distributed as dist


def shard_range(n_total, rank, world):
    """Contiguous batch split: rank r owns frames [lo, hi).  Remainder frames go to the first ranks."""
    base, rem = divmod(n_total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_packed(packed, dst=0, group=None):
    """Gather every rank's packed result [n_r, width] on ``dst``.  Shards may differ by one frame, so
    payloads are padded to the largest shard; returns the list of per-rank tensors (trimmed) on dst,
    None elsewhere."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    n = torch.tensor([packed.shape[0]], dtype=torch.int64, device=packed.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    nmax = int(max(int(s.item()) for s in sizes))
    if packed.shape[0] < nmax:
        pad = torch.zeros((nmax - packed.shape[0],) + tuple(packed.shape[1:]), dtype=packed.dtype, device=packed.device)
        packed = torch.cat([packed, pad], 0)
    out = [torch.empty_like(packed) for _ in range(world)] if rank == dst else None
    dist.gather(packed.contiguous(), out, dst=dst, group=group)
    if rank != dst:
        return None
    return [o[: int(s.item())] for o, s in zip(out, sizes)]


# -- mixed-size lists: shard by network cost, gather fixed-size padded rows ---------------------------------------------
class ShardPlan(object):
    """Rank r's share of a mixed-size list: ``indices[r]`` are caller indices, listed in the arena order the rank's
    pipeline lays its shard out in (litepose_b200.mixed.group_order), so the rows it gathers come back in that order.
    ``rows`` is the common padded shard length of the gather; ``costs[i]`` the network cost of image i, ``load[r]`` the
    sum of rank r's costs."""

    def __init__(self, shapes, indices, costs):
        self.shapes = [tuple(s) for s in shapes]
        self.indices = indices
        self.costs = costs
        self.world = len(indices)
        self.counts = [len(ix) for ix in indices]
        self.rows = max(self.counts)
        self.load = [sum(costs[i] for i in ix) for ix in indices]


def plan_shards(shapes, cfg, world):
    """Deterministic split of a list of images of sizes ``shapes`` [(h, w)] over ``world`` ranks, balanced by the
    network cost of each image: the network input pixels get_multi_scale_size gives over TEST.SCALE_FACTOR, doubled under
    the flip test.  Greedy longest-first onto the least-loaded rank (ties: lower index, lower rank), so the loads of two
    ranks differ by at most one image's cost.  Every rank computes the same plan from the shapes alone: the gather's
    size is known without a collective."""
    from .mixed import group_order, multi_scale_sizes
    shapes = [(int(h), int(w)) for h, w in shapes]
    if not shapes:
        raise ValueError("plan_shards: empty image list")
    if int(world) < 1:
        raise ValueError("plan_shards: world=%r" % (world,))
    scales = sorted((float(v) for v in cfg.TEST.SCALE_FACTOR), reverse=True)
    size = int(cfg.DATASET.INPUT_SIZE)
    keys = [multi_scale_sizes(s, scales, size)[0] for s in shapes]
    flip = 2 if cfg.TEST.FLIP_TEST else 1
    costs = [flip * sum(h * w for h, w in k) for k in keys]
    load = [0] * int(world)
    own = [[] for _ in range(int(world))]
    for i in sorted(range(len(shapes)), key=lambda i: (-costs[i], i)):
        r = min(range(int(world)), key=lambda r: (load[r], r))
        own[r].append(i)
        load[r] += costs[i]
    indices = []
    for ix in own:
        ix.sort()
        indices.append([ix[k] for k in group_order([keys[i] for i in ix])])
    return ShardPlan(shapes, indices, costs)


def gather_rows(rows, out=None, dst=0, group=None):
    """ONE gather of every rank's [L, width] rows into ``out`` [world, L, width] on ``dst`` (None elsewhere).  L, the
    padded shard length of a ShardPlan, is the same on every rank, so no size is exchanged and nothing synchronises the
    host: on an NCCL group it runs on the current stream."""
    glist = list(out.unbind(0)) if dist.get_rank(group) == dst else None
    dist.gather(rows, glist, dst=dst, group=group)
    return out


def split_rows(gathered, plan):
    """[world, L, width] gathered rows -> per rank its [counts[r], width] rows (the padding dropped)."""
    return [gathered[r, :plan.counts[r]] for r in range(plan.world)]


def merge_shards(per_rank, plan):
    """Per-rank result lists (rank r's in the order of plan.indices[r]) -> one list in the caller's order."""
    if len(per_rank) != plan.world:
        raise ValueError("merge_shards: %d rank lists for a plan over %d ranks" % (len(per_rank), plan.world))
    out = [None] * len(plan.shapes)
    for r, (res, ix) in enumerate(zip(per_rank, plan.indices)):
        if len(res) != len(ix):
            raise ValueError("merge_shards: rank %d returned %d results for %d images" % (r, len(res), len(ix)))
        for i, v in zip(ix, res):
            out[i] = v
    return out
