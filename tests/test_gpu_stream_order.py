"""-m gpu: the ordering between the pipeline's streams.  Every asynchronous form spreads one result over several streams
that hand buffers to each other through events; on an idle device the producer of a buffer nearly always finishes long
before its consumer runs, so a missing wait never shows.  Here one stream at a time is held back by a bounded spin
(``late``) at a chosen point, and every result is compared, element for element, with the blocking call on the same
input: step() for frames, infer_images for lists.  Right after the call under test returns, each case notes whether the
spin is still running, and asserts it once the results are in: the call's work really was queued behind the spin.

Every path is warmed up without stalls first (graph capture synchronises the device), every step or list has its own
input (stale data from another step changes the answer), and a control drops the waits on one stream's events to show
that the comparisons catch a missing wait."""
import time

import numpy as np
import pytest
import torch

from litepose_b200 import synth
from litepose_b200.pipeline import PlantedCrowd
from test_gpu_submit_images import LIST_A, LIST_B, POOL, SIZE, _cfg_case, _images, _pipe, _plants, _same

pytestmark = pytest.mark.gpu

STALL_MS = 40
# the list form stages each list and launches its eager network passes on the host, tens of milliseconds per list: the
# list cases hold a stream back for longer, so that the window still spans the calls under test
LIST_STALL_MS = 150
N = 2
# a list whose largest size group (4 images at 128x320) is larger than any group of LIST_A, LIST_B or POOL, while its
# image count and bytes are smaller: it grows the engine's arenas (and drops the arena plans built on them) and nothing
# else
BIG_GROUP = [(90, 200), (90, 200), (90, 200), (120, 120), (90, 200)]

_CYCLES_PER_MS = {}


def _cycles_per_ms():
    """torch.cuda._sleep cycles per millisecond on the current device, timed once per process with CUDA events.  Only
    used to size the stalls: no assertion rests on it."""
    dev = torch.cuda.current_device()
    if dev not in _CYCLES_PER_MS:
        torch.cuda._sleep(1000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        cycles = 20_000_000
        e0.record()
        torch.cuda._sleep(cycles)
        e1.record()
        e1.synchronize()
        _CYCLES_PER_MS[dev] = cycles / max(e0.elapsed_time(e1), 1e-3)
    return _CYCLES_PER_MS[dev]


def late(stream, ms=STALL_MS):
    """Queue one bounded spin of about ``ms`` milliseconds on ``stream``; returns an event recorded after it."""
    cycles = int(ms * _cycles_per_ms())
    with torch.cuda.stream(stream):
        torch.cuda._sleep(cycles)
        ev = torch.cuda.Event()
        ev.record(stream)
    return ev


def pipeline_streams(pipe):
    """Every stream the pipeline owns, by name: the current stream, per uniform-size state its side stream and the
    parser stream of its overlapped form, the copy and result streams of submit() and of submit_images(), and the side
    stream of the list form.  Only the streams made so far are listed."""
    out = {"current": torch.cuda.current_stream(pipe.device)}
    for key, st in pipe._state.items():
        out["side %r" % (key,)] = st["side"]
        if st.get("ov") is not None:
            out["pstream %r" % (key,)] = st["ov"]["pstream"]
    if pipe._async is not None:
        out["copy"], out["res"] = pipe._async["copy"], pipe._async["res"]
    if hasattr(pipe, "_lists"):
        out["lists copy"], out["lists res"] = pipe._lists["copy"], pipe._lists["res"]
        out["mixed side"] = pipe._mixed_side
    return out


def _streams_held_by(root):
    """Every torch.cuda.Stream reachable from ``root`` through containers, closures and the attributes of the package's
    own objects."""
    import types
    found, seen, todo = [], set(), [root]
    while todo:
        o = todo.pop()
        if id(o) in seen:
            continue
        seen.add(id(o))
        if isinstance(o, torch.cuda.Stream):
            found.append(o)
        elif isinstance(o, dict):
            todo.extend(o.keys())
            todo.extend(o.values())
        elif isinstance(o, (list, tuple, set, frozenset)):
            todo.extend(o)
        elif isinstance(o, types.FunctionType):
            for c in o.__closure__ or ():
                try:
                    todo.append(c.cell_contents)
                except ValueError:
                    pass
        elif isinstance(o, types.MethodType):
            todo.append(o.__self__)
        elif type(o).__module__.startswith("litepose_b200"):
            todo.extend(getattr(o, "__dict__", {}).values())
            todo.extend(getattr(o, s) for s in getattr(type(o), "__slots__", ()) if hasattr(o, s))
    return found


# -- frames: submit / collect, step_device_overlapped, step_device --------------------------------------------------
class _Frames(object):
    """One warmed-up pipeline and its inputs: frames A, B, C (pinned and on the device), one plant hook shared by every
    step (a plant change recaptures the graphs), the blocking step() of each frame, and a batch of uint8 images whose
    network input has the frames' shape."""

    def __init__(self, grouping):
        cfg = _cfg_case("shipped" if grouping == "ae" else "fast")
        self.pipe = pipe = _pipe(cfg, grouping=grouping)
        J, t = pipe.params.num_joints, pipe.T
        hd = SIZE if pipe.project else SIZE // 2
        # heat peaks only: the keypoints' tags are the network's own, so every frame has its own answer
        self.plant = PlantedCrowd(N, J, hd, hd, t, num_people=3, seed=9, device="cuda")
        self.plant.tidx, self.plant.tval = self.plant.tidx[:0], self.plant.tval[:0]
        self.frames = {k: synth.make_frames(N, SIZE, seed=s).half().pin_memory() for k, s in zip("ABC", (4, 5, 6))}
        self.dev = {k: f.cuda() for k, f in self.frames.items()}
        self.ref = {k: pipe.step(f, self.plant) for k, f in self.frames.items()}
        for k in "ABC":
            assert sum(r[-1] for r in self.ref[k]) > 0, k
        for x, y in (("A", "B"), ("B", "C"), ("A", "C")):
            assert not _equal(self.ref[x], self.ref[y]), "frames %s and %s give the same keypoints" % (x, y)
        self.batch = torch.from_numpy(np.stack(_images([(SIZE, SIZE)] * N, 3))).pin_memory()
        self.ref_batch = pipe.infer_images(self.batch)
        assert pipe._last_state["x"].shape == self.dev["A"].shape and pipe._last_state["x"].dtype == torch.float16
        # warm-up: both buffer sets of the overlapped form captured, both submit() slots made
        for ticket in [pipe.submit(self.frames[k], self.plant) for k in "AB"]:
            pipe.collect(ticket)
        torch.cuda.synchronize()
        self.state = pipe._get_state(N, SIZE, SIZE, torch.float16, self.plant)
        assert all(g is not None for g in self.state["ov"]["gF"])

    def streams(self):
        a, st = self.pipe._async, self.state
        return {"current": torch.cuda.current_stream(), "copy": a["copy"], "res": a["res"],
                "pstream": st["ov"]["pstream"], "side": st["side"]}

    def next_set(self, b):
        """Make the next overlapped step run in buffer set ``b`` (one unstalled overlapped step if needed)."""
        if self.state["ov"]["idx"] != b:
            self.pipe.step_device_overlapped(self.dev["C"], self.plant)
            torch.cuda.synchronize()
        assert self.state["ov"]["idx"] == b


def _equal(got, exp):
    try:
        _same(got, exp)
        return True
    except AssertionError:
        return False


@pytest.fixture(scope="module", params=["ae", "fast"])
def frames_rig(request):
    return _Frames(request.param)


SEQ = "ABCABC"


def _submit_run(rig, stall, newest_first=False):
    """Six submits over SEQ, two in flight; ``stall`` (a name of rig.streams(), or None) is held back right before the
    third submit.  Oldest first: each submit is followed by the collect of the one before it.  Newest first: submits in
    pairs, the second of each pair collected first.  Returns the collected results in submission order; asserts, once
    they have been collected, that the stall was still running when the third submit returned."""
    pipe = rig.pipe
    got = [None] * len(SEQ)
    opened = []

    def submit(i):
        ev = late(rig.streams()[stall]) if stall is not None and i == 2 else None
        t = pipe.submit(rig.frames[SEQ[i]], rig.plant)
        if ev is not None:
            opened.append(not ev.query())
        return t

    if newest_first:
        for i in range(0, len(SEQ), 2):
            ta, tb = submit(i), submit(i + 1)
            got[i + 1] = pipe.collect(tb)[0]
            got[i] = pipe.collect(ta)[0]
    else:
        prev = None
        for i in range(len(SEQ)):
            t = submit(i)
            if prev is not None:
                got[i - 1] = pipe.collect(prev)[0]
            prev = t
        got[-1] = pipe.collect(prev)[0]
    torch.cuda.synchronize()
    assert opened == ([] if stall is None else [True]), "the stall on %s ended before submit() returned" % stall
    return got


@pytest.mark.parametrize("stall", ["current", "copy", "res", "pstream", "side"])
def test_submit_collect_with_a_late_stream(frames_rig, stall):
    got = _submit_run(frames_rig, stall)
    for i, k in enumerate(SEQ):
        _same(got[i], frames_rig.ref[k], "step %d (%s), %s stalled" % (i, k, stall))


def test_submit_collect_newest_first(frames_rig):
    got = _submit_run(frames_rig, "res", newest_first=True)
    for i, k in enumerate(SEQ):
        _same(got[i], frames_rig.ref[k], "step %d (%s)" % (i, k))


@pytest.mark.parametrize("stall", ["pstream", "current"])
def test_step_device_overlapped_with_a_late_stream(frames_rig, stall):
    """Four overlapped steps alternating the buffer sets; each payload is read on the current stream after its event,
    before the second next call (the documented lifetime), while the following step's network is already queued."""
    rig, pipe = frames_rig, frames_rig.pipe
    main = torch.cuda.current_stream()
    seq, outs, pending = "BCAB", [], []
    ev = late(rig.streams()[stall])
    for i, k in enumerate(seq):
        packed, done = pipe.step_device_overlapped(rig.dev[k], rig.plant)
        if i == 0:
            opened = not ev.query()
        pending.append((k, packed, done))
        if len(pending) == 2:
            kk, p, d = pending.pop(0)
            main.wait_event(d)
            outs.append((kk, p.clone()))
    for kk, p, d in pending:
        main.wait_event(d)
        outs.append((kk, p.clone()))
    torch.cuda.synchronize()
    assert opened, "the stall on %s ended before step_device_overlapped returned" % stall
    assert [k for k, _ in outs] == list(seq)
    for i, (k, p) in enumerate(outs):
        _same(pipe._decode(p.cpu()), rig.ref[k], "overlapped step %d (%s), %s stalled" % (i, k, stall))


def test_step_device_after_an_overlapped_step_still_parsing(frames_rig):
    """step_device while an overlapped step of buffer set 0 - whose det, tag and packed it shares - is still queued on
    the parser stream: its payload must be its own frames' answer."""
    rig, pipe = frames_rig, frames_rig.pipe
    rig.next_set(0)
    ev = late(rig.streams()["pstream"])
    pipe.step_device_overlapped(rig.dev["A"], rig.plant)
    packed = pipe.step_device(rig.dev["B"], rig.plant)
    opened = not ev.query()
    got = pipe._decode(packed.cpu())
    torch.cuda.synchronize()
    assert opened, "the stall on the parser stream ended before step_device returned"
    _same(got, rig.ref["B"], "step_device")


def test_step_between_submit_and_collect(frames_rig):
    """submit() into buffer set 0, then a blocking step() of the same shape on other frames, then collect().  The
    submitted payload leaves set 0's packed through a copy on the result stream; that stream is held back from before
    the submit (a spin queued after the submit would not delay a copy already queued ahead of it), so the step runs
    while the copy is still pending and must not overwrite the payload under it."""
    rig, pipe = frames_rig, frames_rig.pipe
    rig.next_set(0)
    ev = late(rig.streams()["res"])
    t = pipe.submit(rig.frames["A"], rig.plant)
    opened = not ev.query()
    in_set = rig.state["ov_last"]
    got_step = pipe.step(rig.frames["B"], rig.plant)
    got_sub = pipe.collect(t)[0]
    torch.cuda.synchronize()
    assert opened, "the stall on the result stream ended before submit() returned"
    assert in_set == 0
    _same(got_step, rig.ref["B"], "step")
    _same(got_sub, rig.ref["A"], "collected")


def test_infer_images_between_submit_and_collect(frames_rig):
    """submit() into buffer set 0 with the parser stream held back, then infer_images on a batch whose network input
    has the frames' shape, then collect().  The batch runs in a state of its own, but on the same engine buffer set 0
    (the network outputs the submitted step's glue has yet to read) and the same parser buffers."""
    rig, pipe = frames_rig, frames_rig.pipe
    rig.next_set(0)
    ev = late(rig.streams()["pstream"])
    t = pipe.submit(rig.frames["C"], rig.plant)
    opened = not ev.query()
    in_set = rig.state["ov_last"]
    got_batch = pipe.infer_images(rig.batch)
    got_sub = pipe.collect(t)[0]
    torch.cuda.synchronize()
    assert opened, "the stall on the parser stream ended before submit() returned"
    assert in_set == 0
    _same(got_batch, rig.ref_batch, "infer_images")
    _same(got_sub, rig.ref["C"], "collected")


@pytest.mark.parametrize("frames_rig", ["ae"], indirect=True)
def test_control_dropped_copy_wait_is_caught(frames_rig):
    """The harness has teeth: with every wait on an event recorded on submit()'s copy stream dropped, the network reads
    an input slot before its frames have arrived, and the six-step run with the copy stream held back no longer equals
    step().  With the waits restored the same run does."""
    rig = frames_rig
    copy = rig.pipe._async["copy"]
    record, wait_event = torch.cuda.Event.record, torch.cuda.Stream.wait_event

    def tagged_record(self, stream=None):
        s = torch.cuda.current_stream() if stream is None else stream
        self._recorded_on = s.cuda_stream
        return record(self, stream)

    def dropping_wait(self, event):
        if getattr(event, "_recorded_on", None) == copy.cuda_stream:
            return None
        return wait_event(self, event)

    try:
        torch.cuda.Event.record = tagged_record
        torch.cuda.Stream.wait_event = dropping_wait
        got = _submit_run(rig, "copy")
    finally:
        torch.cuda.Event.record, torch.cuda.Stream.wait_event = record, wait_event
        torch.cuda.synchronize()
    assert not all(_equal(g, rig.ref[k]) for g, k in zip(got, SEQ)), "a dropped wait went unnoticed"
    got = _submit_run(rig, "copy")
    for i, k in enumerate(SEQ):
        _same(got[i], rig.ref[k], "step %d (%s), waits restored" % (i, k))


# -- lists: submit_images / collect_images ---------------------------------------------------------------------------
class _Lists(object):
    """One warmed-up pipeline and its lists: A (host images) and B (device images) with planted persons, D (POOL) and
    a uniform batch for the blocking calls, each with the blocking infer_images result."""

    def __init__(self, case):
        cfg = _cfg_case(case)
        self.pipe = pipe = _pipe(cfg, grouping="fast" if case.startswith("fast") else "ae")
        self.images = {"A": _images(LIST_A, 1), "B": [torch.from_numpy(im).cuda() for im in _images(LIST_B, 2)],
                       "D": _images(POOL, 3)}
        self.plants = {"A": _plants(pipe, LIST_A, seed=40), "B": _plants(pipe, LIST_B, seed=60), "D": None}
        self.ref = {k: pipe.infer_images(v, plant=self.plants[k]) for k, v in self.images.items()}
        self.batch = torch.from_numpy(np.stack(_images([(SIZE, SIZE)] * N, 3))).pin_memory()
        self.ref_batch = pipe.infer_images(self.batch)
        assert sum(r[-1] for r in self.ref["A"]) > 0 and sum(r[-1] for r in self.ref["B"]) > 0
        # warm-up: both slots served a list at least as large as any submitted below (BIG_GROUP aside)
        ta, tb = self.submit("A"), self.submit("B")
        self.pipe.collect_images(ta)
        self.pipe.collect_images(tb)
        tb, ta = self.submit("B"), self.submit("A")
        self.pipe.collect_images(tb)
        self.pipe.collect_images(ta)
        # first-time device allocations on the current stream are served from this cached block
        del_me = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        del del_me
        torch.cuda.synchronize()

    def submit(self, k):
        return self.pipe.submit_images(self.images[k], plant=self.plants[k])

    def streams(self):
        p = self.pipe
        return {"current": torch.cuda.current_stream(), "copy": p._lists["copy"], "res": p._lists["res"],
                "mixed_side": p._mixed_side}


@pytest.fixture(scope="module", params=["shipped", "fast"])
def lists_rig(request):
    return _Lists(request.param)


def _window(ev, t0):
    """(whether the stall behind ``ev`` was still running, host milliseconds since ``t0``)"""
    return not ev.query(), (time.perf_counter() - t0) * 1e3


@pytest.mark.parametrize("stall", ["current", "copy", "res", "mixed_side"])
def test_two_lists_with_a_late_stream(lists_rig, stall):
    """Two lists of different compositions in flight, the first one's work held back on one stream while the second
    is queued."""
    rig, pipe = lists_rig, lists_rig.pipe
    ev, t0 = late(rig.streams()[stall], LIST_STALL_MS), time.perf_counter()
    ta = rig.submit("A")
    tb = rig.submit("B")
    opened, ms = _window(ev, t0)
    got_a, got_b = pipe.collect_images(ta), pipe.collect_images(tb)
    torch.cuda.synchronize()
    assert opened, "the stall on %s ended before submit_images returned (%.1f ms on the host)" % (stall, ms)
    _same(got_a, rig.ref["A"], "list A, %s stalled" % stall)
    _same(got_b, rig.ref["B"], "list B, %s stalled" % stall)


def test_larger_list_while_a_list_is_outstanding(lists_rig):
    """A list with a larger size group than any before it is submitted after one collect, while the other list's
    mirrored passes are still held back on the list form's side stream: it grows the engine's arenas (dropping the
    arena plans the outstanding list ran on) under work that still reads the old ones."""
    rig, pipe = lists_rig, lists_rig.pipe
    big = _images(BIG_GROUP, 7)
    big_plants = _plants(pipe, BIG_GROUP, seed=70)
    ta = rig.submit("A")
    ev, t0 = late(rig.streams()["mixed_side"], LIST_STALL_MS), time.perf_counter()
    tb = rig.submit("B")
    got_a = pipe.collect_images(ta)
    arenas = {k: v.numel() for k, v in pipe.engine.arenas.items()}
    tc = pipe.submit_images(big, plant=big_plants)
    opened, ms = _window(ev, t0)
    grown = [k for k, n in arenas.items() if pipe.engine.arenas[k].numel() > n]
    got_b, got_c = pipe.collect_images(tb), pipe.collect_images(tc)
    torch.cuda.synchronize()
    assert opened, "the stall on the list side stream ended before submit_images returned (%.1f ms on the host)" % ms
    assert grown, "the engine's arenas did not grow"
    _same(got_a, rig.ref["A"], "list A")
    _same(got_b, rig.ref["B"], "list B")
    # the blocking reference only now: run first, it would have grown the arenas before the case
    _same(got_c, pipe.infer_images(big, plant=big_plants), "larger list")


def test_blocking_calls_while_a_list_is_outstanding(lists_rig):
    """infer_images on a list and on a uniform batch while a list's payload copy is held back on the result stream."""
    rig, pipe = lists_rig, lists_rig.pipe
    ev, t0 = late(rig.streams()["res"], LIST_STALL_MS), time.perf_counter()
    ta = rig.submit("A")
    got_d = pipe.infer_images(rig.images["D"])
    got_batch = pipe.infer_images(rig.batch)
    opened, ms = _window(ev, t0)
    got_a = pipe.collect_images(ta)
    torch.cuda.synchronize()
    assert opened, "the stall on the result stream ended before the blocking calls returned (%.1f ms on the host)" % ms
    _same(got_a, rig.ref["A"], "list A")
    _same(got_d, rig.ref["D"], "blocking list")
    _same(got_batch, rig.ref_batch, "blocking batch")


def test_caller_may_reuse_its_images_after_submit_images(lists_rig):
    """Once submit_images has returned, the caller may overwrite its host images and (on the current stream) its
    device images: the list's device work is held back on the current stream, and the result is unchanged."""
    rig, pipe = lists_rig, lists_rig.pipe
    src = _images(LIST_A, 8)
    imgs = [im.copy() if i % 2 == 0 else torch.from_numpy(im).cuda() for i, im in enumerate(src)]
    exp = pipe.infer_images([im.copy() for im in src], plant=rig.plants["A"])
    ev, t0 = late(torch.cuda.current_stream(), LIST_STALL_MS), time.perf_counter()
    t = pipe.submit_images(imgs, plant=rig.plants["A"])
    opened, ms = _window(ev, t0)
    for im in imgs:
        if torch.is_tensor(im):
            im.fill_(255)
        else:
            im[...] = 0
    got = pipe.collect_images(t)
    torch.cuda.synchronize()
    assert opened, "the stall on the current stream ended before submit_images returned (%.1f ms on the host)" % ms
    _same(got, exp, "caller's images overwritten")


# -- the stream inventory ----------------------------------------------------------------------------------------------
def test_every_stream_is_in_the_inventory():
    """After every entry point has run, no stream reachable from the pipeline lies outside pipeline_streams(): a stream
    added later cannot escape this file's stalls unnoticed."""
    cfg = _cfg_case("shipped")
    pipe = _pipe(cfg)
    fr = synth.make_frames(N, SIZE, seed=4).half().pin_memory()
    pipe.step(fr)
    pipe.collect(pipe.submit(fr))
    pipe.step_device_overlapped(fr.cuda())
    pipe.infer_images(torch.from_numpy(np.stack(_images([(SIZE, SIZE)] * N, 3))))
    pipe.infer_images(_images(LIST_B, 2))
    pipe.collect_images(pipe.submit_images(_images(LIST_A, 1)))
    torch.cuda.synchronize()
    inventory = pipeline_streams(pipe)
    assert {"copy", "res", "lists copy", "lists res", "mixed side"} <= set(inventory)
    assert sum(k.startswith("pstream") for k in inventory) == 1 and sum(k.startswith("side") for k in inventory) == 2
    known = {s.cuda_stream for s in inventory.values()}
    held = _streams_held_by(pipe)
    stray = [s for s in held if s.cuda_stream not in known]
    assert not stray, "streams outside the inventory: %r" % (stray,)
    # and every named stream but the current one is one the pipeline holds
    assert {s.cuda_stream for s in held} == known - {inventory["current"].cuda_stream}


# -- two ranks: the sharded list, gathered on the result stream --------------------------------------------------------
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
        plants = _plants(pipe, TWO_RANK_SHAPES, seed=90)
        plan = plan_shards(TWO_RANK_SHAPES, cfg, 2)
        mine = plan.indices[rank]

        def submit(imgs):
            return pipe.submit_images([imgs[i] for i in mine], plant=[plants[i] for i in mine],
                                      group=dist.group.WORLD, dst=0, plan=plan)

        pipe.collect_images(submit(_images(TWO_RANK_SHAPES, 12)))       # warm-up: communicator, slot, arena plans
        torch.cuda.synchronize()
        imgs = _images(TWO_RANK_SHAPES, 11)
        ev = late(pipe._lists["res"], LIST_STALL_MS) if rank == 1 else None
        tk = submit(imgs)
        opened = ev is None or not ev.query()
        res = pipe.collect_images(tk)
        if rank == 0:
            merged = merge_shards(res, plan)
            full = pipe.infer_images(imgs, plant=plants)
            pack = lambda rs: [(r[0].tolist(), np.asarray(r[1], np.float32).tolist(), r[2]) for r in rs]
            q.put((rank, opened, pack(merged), pack(full)))
        else:
            q.put((rank, opened, res, None))
        torch.cuda.synchronize()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (one rank per GPU, NCCL gather)")
def test_two_rank_gather_with_a_late_result_stream():
    """The sharded submit_images with rank 1's result stream (which runs the NCCL gather) held back before its submit:
    the merged list on rank 0 equals infer_images on the whole list."""
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
            rank, opened, merged, full = q.get(timeout=600)
            out[rank] = (opened, merged, full)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    assert out[1][0], "the stall on rank 1's result stream ended before submit_images returned"
    assert out[1][1] is None
    _, merged, full = out[0]
    assert len(merged) == len(full) == len(TWO_RANK_SHAPES)
    for i, (g, e) in enumerate(zip(merged, full)):
        assert g == e, i
