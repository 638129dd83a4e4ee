"""Guarded device buffers for the footprint tests: where a kernel reads and writes, not only what it computes.

Every tensor of a call lives in a device allocation of its own, laid out [front guard | payload | back guard].  The guards
are GUARD bytes each (more than the largest output tile of any kernel, so a plausible overrun lands inside the
allocation), and the payload starts SKEW bytes past the front guard: 16-byte aligned but not 128-byte aligned, unless a
case asks for another skew (the smallest alignment an entry point documents, or an odd element offset).
  - inputs, weights and descriptors: payload flush against guards of a poison that propagates (fp16 / fp32 / fp64 NaN,
    0xA5 for uint8 images, 0x7F7F... for integers and raw descriptor bytes), so a read past the payload turns the result
    into NaN or garbage instead of the zeros a fresh allocation usually holds;
  - outputs: payload and guards prefilled with a sentinel NaN of distinctive payload (fp16 0x7D5A, fp32 0x7FA5A5A5;
    0x5A... for integers), which no kernel computes: "never written" is told apart from "computed NaN" (uint8 outputs
    are filled with 0x5A too, but that is a pixel value: they are held to their reference alone);
  - workspaces: exactly the bytes their *_workspace_bytes function reports, guards of 0xA5.
Guarded.verify then checks that every guard byte is unchanged, every input payload byte is unchanged, and every output
equals its reference, naming the buffer and the byte offset where a check fails.

Plain is the same interface on ordinary torch tensors (outputs sentinel-filled too): a case run with it is "the same
call on plain tensors", the reference of the entry points the suite already holds to their oracles that way."""
import numpy as np
import torch

GUARD = 1 << 20
SKEW = 16

_UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
_TORCH = {np.float16: torch.float16, np.float32: torch.float32, np.float64: torch.float64, np.uint8: torch.uint8,
          np.int32: torch.int32, np.int64: torch.int64}
POISON = {np.float16: 0x7E00, np.float32: 0x7FC00000, np.float64: 0x7FF8000000000000, np.uint8: 0xA5,
          np.int32: 0x7F7F7F7F, np.int64: 0x7F7F7F7F7F7F7F7F}
SENTINEL = {np.float16: 0x7D5A, np.float32: 0x7FA5A5A5, np.uint8: 0x5A, np.int32: 0x5AA55AA5}
WS_POISON = 0xA5
DESC_POISON = 0x7F


def _pattern(nbytes, dtype, bits):
    """nbytes bytes of the element bit pattern ``bits`` repeated (phase 0 at byte 0)"""
    es = np.dtype(dtype).itemsize
    return np.full(-(-nbytes // es), bits, _UINT[es]).view(np.uint8)[:nbytes].copy()


def sentinel_array(shape, dtype):
    """an array of ``shape`` holding the output sentinel of ``dtype``"""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape))
    return _pattern(n * dtype.itemsize, dtype, SENTINEL[dtype.type]).view(dtype).reshape(shape)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(_UINT[a.dtype.itemsize])


def _at(mask):
    """index of the first True of mask, as a tuple of ints"""
    return tuple(int(v) for v in np.argwhere(mask)[0])


def compare(name, got, want, may_keep_sentinel=False):
    """got (device result) against want (reference): equal as values (+0 == -0) or as bits; positions where want holds
    the sentinel must hold it in got too (entries the header leaves untouched), and - unless may_keep_sentinel - the
    reference must hold no sentinel at all.  -> list of error strings"""
    want = np.asarray(want)
    got = np.asarray(got).astype(want.dtype, copy=False) if got.dtype != want.dtype else np.asarray(got)
    got = got.reshape(want.shape)
    dt = want.dtype.type
    # a uint8 sentinel is a legitimate pixel value: bytes are held to the reference alone
    s = None if want.dtype.itemsize == 1 else SENTINEL.get(dt)
    errs = []
    gb, wb = _bits(got), _bits(want)
    if s is not None:
        ws_, gs = wb == s, gb == s
        if ws_.any() and not may_keep_sentinel:
            errs.append("%s: the reference leaves %d elements unwritten (first at %s)"
                        % (name, ws_.sum(), _at(ws_)))
        left = gs & ~ws_
        if left.any():
            errs.append("%s: %d of %d elements never written (sentinel left; first at %s)"
                        % (name, left.sum(), left.size, _at(left)))
        over = ws_ & ~gs
        if over.any():
            errs.append("%s: %d elements written that must stay untouched (first at %s: %r)"
                        % (name, over.sum(), _at(over), got[_at(over)]))
    with np.errstate(invalid="ignore"):
        same = (gb == wb) | (got == want)
        if np.issubdtype(want.dtype, np.floating):
            same |= np.isnan(got) & np.isnan(want)
    if s is not None:
        same |= (gb == s) | (wb == s)          # reported above
    if not same.all():
        i = _at(~same)
        errs.append("%s: %d of %d elements differ from the reference (first at %s: %r vs %r)"
                    % (name, (~same).sum(), same.size, i, got[i], want[i]))
    return errs


class _Buf(object):
    __slots__ = ("name", "role", "raw", "before", "off", "nbytes", "dtype", "shape", "t")


class Guarded(object):
    """one guarded allocation per tensor; see the module docstring"""

    def __init__(self):
        self.bufs = {}

    def _add(self, name, role, data, shape, dtype, skew, fill):
        assert name not in self.bufs, name
        dtype = np.dtype(dtype)
        es = dtype.itemsize
        skew = SKEW if skew is None else skew
        assert skew % es == 0, (name, skew, es)
        n = int(np.prod(shape))
        b = _Buf()
        b.name, b.role, b.dtype, b.shape = name, role, dtype, tuple(shape)
        b.off, b.nbytes = GUARD + skew, n * es
        host = _pattern(b.off + b.nbytes + GUARD, dtype, fill)
        if data is not None:
            host[b.off:b.off + b.nbytes] = np.ascontiguousarray(data, dtype).reshape(-1).view(np.uint8)
        b.before = host
        b.raw = torch.from_numpy(host.copy()).cuda()
        b.t = b.raw[b.off:b.off + b.nbytes].view(_TORCH[dtype.type]).view(b.shape)
        self.bufs[name] = b
        return b.t

    def inp(self, name, arr, skew=None):
        """an input (activation, weight, index list): payload unchanged by the call"""
        arr = np.asarray(arr)
        return self._add(name, "in", arr, arr.shape, arr.dtype, skew, POISON[arr.dtype.type])

    def desc(self, name, arr, skew=None):
        """a descriptor array of a structured dtype, held as raw bytes"""
        raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
        return self._add(name, "in", raw, raw.shape, np.uint8, skew, DESC_POISON)

    def out(self, name, shape, dtype, skew=None, init=None):
        """an output, sentinel-filled; ``init`` gives the payload of an in-place (read-modify-write) output"""
        dtype = np.dtype(dtype)
        return self._add(name, "out", init, shape, dtype, skew, SENTINEL[dtype.type])

    def ws(self, name, nbytes, skew=256):
        """a workspace of exactly nbytes (256-byte aligned by default: the parser's workspaces require it)"""
        return self._add(name, "ws", None, (max(int(nbytes), 1),), np.uint8, skew, WS_POISON)

    def scratch(self, name, shape, dtype, skew=None):
        """a buffer written and read by a chain of calls, sentinel-filled; only its guards are checked"""
        dtype = np.dtype(dtype)
        return self._add(name, "scratch", None, shape, dtype, skew, SENTINEL[dtype.type])

    def outputs(self):
        torch.cuda.synchronize()
        return {n: b.t.cpu().numpy() for n, b in self.bufs.items() if b.role == "out"}

    def verify(self, expect, untouched=()):
        """guards of every buffer, input payloads, outputs against ``expect`` (name -> array); ``untouched`` names the
        outputs whose reference may keep the sentinel.  -> list of error strings (empty: clean)"""
        torch.cuda.synchronize()
        errs = []
        for name, b in self.bufs.items():
            after = b.raw.cpu().numpy()
            o, e = b.off, b.off + b.nbytes
            d = np.nonzero(after[:o] != b.before[:o])[0]
            if d.size:
                errs.append("%s: front guard modified: %d bytes at payload offsets %d .. %d"
                            % (name, d.size, d[0] - o, d[-1] - o))
            d = np.nonzero(after[e:] != b.before[e:])[0]
            if d.size:
                errs.append("%s: back guard modified: %d bytes at end + %d .. end + %d" % (name, d.size, d[0], d[-1]))
            if b.role == "in":
                d = np.nonzero(after[o:e] != b.before[o:e])[0]
                if d.size:
                    errs.append("%s: input payload modified: %d bytes, first at byte %d" % (name, d.size, d[0]))
            elif b.role == "out":
                assert name in expect, "no reference for output %s" % name
                got = after[o:e].view(b.dtype).reshape(b.shape)
                errs += compare(name, got, expect[name], name in untouched)
        return errs


class Plain(object):
    """the Guarded interface on ordinary torch tensors (no guards, no skew); outputs sentinel-filled"""

    def __init__(self):
        self.bufs = {}

    def inp(self, name, arr, skew=None):
        self.bufs[name] = ("in", torch.from_numpy(np.ascontiguousarray(arr)).cuda())
        return self.bufs[name][1]

    def desc(self, name, arr, skew=None):
        return self.inp(name, np.ascontiguousarray(arr).view(np.uint8).reshape(-1))

    def out(self, name, shape, dtype, skew=None, init=None):
        a = sentinel_array(shape, dtype) if init is None else np.asarray(init, dtype).reshape(shape)
        self.bufs[name] = ("out", torch.from_numpy(np.ascontiguousarray(a)).cuda())
        return self.bufs[name][1]

    def ws(self, name, nbytes, skew=None):
        self.bufs[name] = ("ws", torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device="cuda"))
        return self.bufs[name][1]

    def outputs(self):
        torch.cuda.synchronize()
        return {n: t.cpu().numpy() for n, (role, t) in self.bufs.items() if role == "out"}


def host_guarded(elems, dtype, fill_bits, tail=4096):
    """a host array of elems + tail elements filled with fill_bits; -> (whole, payload view)"""
    whole = _pattern((elems + tail) * np.dtype(dtype).itemsize, dtype, fill_bits).view(dtype)
    return whole, whole[:elems]
