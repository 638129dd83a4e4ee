"""CPU: the host weight packers write exactly their *_elems elements and all of them, and every launching entry point
of the C ABI has a case in the footprint table (tests/footprint_cases.py, run on the GPU by test_gpu_footprint.py).

Each packer runs twice into a destination of exactly *_elems elements followed by a guard tail: once prefilled with
0xFFFF (fp16 NaN; 0xFFFFFFFF for fp32 biases), once with zeros.  Both results must be identical - a packer that leaves
its padding to the caller's zero-fill fails - and the tail must be untouched."""
import numpy as np
import pytest

import footprint_cases as fc
from footprint_util import host_guarded
from litepose_b200 import _lib

TAIL_BITS = 0x5AA5


def _lib_or_skip():
    try:
        return _lib.load()
    except _lib.LitePoseLibraryError as e:       # pragma: no cover - the library is built before the suite runs
        pytest.skip(str(e))


def _pack_twice(fill_call, sizes):
    """fill_call(*dst) packs into the destinations; sizes = [(elems, dtype)].  -> the packed arrays (after checking
    that 0xFF.. and zero prefills give the same result and the guard tails survive)"""
    results = []
    for fill in (0xFF, 0x00):
        wholes, dsts = [], []
        for elems, dt in sizes:
            es = np.dtype(dt).itemsize
            whole, dst = host_guarded(elems, dt, TAIL_BITS if es == 2 else 0x5AA55AA5)
            dst.view(np.uint8)[:] = fill
            wholes.append(whole)
            dsts.append(dst)
        _lib.check(fill_call(*[d.ctypes.data for d in dsts]), "pack")
        for (elems, dt), whole in zip(sizes, wholes):
            tail = whole[elems:].view(np.uint16 if np.dtype(dt).itemsize == 2 else np.uint32)
            assert (tail == (TAIL_BITS if np.dtype(dt).itemsize == 2 else 0x5AA55AA5)).all(), (
                "written past *_elems: first at +%d" % np.nonzero(tail != tail[-1])[0][0])
        results.append([d.copy() for d in dsts])
    for a, b in zip(*results):
        bad = a.view(np.uint8) != b.view(np.uint8)
        assert not bad.any(), "%d bytes depend on the destination's prior contents (first at byte %d)" % (
            bad.sum(), np.nonzero(bad)[0][0])
    return results[1]


def _w(shape, seed):
    return np.ascontiguousarray((np.random.default_rng(seed).standard_normal(shape) * 0.3).astype(np.float16)).view(
        np.uint16)


def _b(n, seed):
    return np.random.default_rng(seed).standard_normal(n).astype(np.float32)


@pytest.mark.parametrize("k,n,bias", [(8, 8, True), (72, 24, True), (96, 160, False), (72, 168, True), (960, 160, True),
                                      (32, 1024, True)])
def test_pw1x1_pack_footprint(k, n, bias):
    lib = _lib_or_skip()
    w, b = _w((n, k), k + n), _b(n, k * n) if bias else None
    _pack_twice(lambda wp, bp: lib.lp_pw1x1_pack(w.ctypes.data, None if b is None else b.ctypes.data, k, n, wp, bp),
                [(lib.lp_pw1x1_packed_elems(k, n), np.float16), (lib.lp_pw1x1_packed_bias_elems(n), np.float32)])


# (Cr, Cw, Co): the row kernel's layout, the tiled layout (Cr + Cw > 64, Co > 32, a second K block), one branch each
@pytest.mark.parametrize("cr_,cw,co", [(16, 16, 16), (24, 16, 8), (40, 24, 32), (72, 40, 64), (80, 48, 16),
                                       (32, 0, 16), (96, 0, 24), (40, 24, 40)])
def test_deconv_pack_footprint(cr_, cw, co):
    lib = _lib_or_skip()
    wr, ww, b = _w((cr_, co, 4, 4), cr_ + co), _w((cw, co, 4, 4), cw + co + 1) if cw else None, _b(co, co)
    _pack_twice(lambda wp, bp: lib.lp_deconv_pack(wr.ctypes.data, None if ww is None else ww.ctypes.data, b.ctypes.data,
                                                  cr_, cw, co, wp, bp),
                [(lib.lp_deconv_packed_elems(cr_, cw, co), np.float16), (lib.lp_deconv_packed_bias_elems(co), np.float32)])


@pytest.mark.parametrize("c1,c2,co", [(16, 16, 17), (32, 32, 34), (8, 16, 30), (24, 0, 17), (72, 96, 17)])
def test_head_pack_footprint(c1, c2, co):
    lib = _lib_or_skip()
    w1, w2 = _w((co, c1), c1 + co), _w((co, c2), c2 + co + 1) if c2 else None
    _pack_twice(lambda wp: lib.lp_head_pack(w1.ctypes.data, None if w2 is None else w2.ctypes.data, c1, c2, co, wp),
                [(lib.lp_head_packed_elems(c1, c2, co), np.float16)])


@pytest.mark.parametrize("c1,c2,co", [(24, 16, 28), (72, 40, 34), (40, 0, 17), (24, 0, 14)])
def test_head_fused_pack_footprint(c1, c2, co):
    lib = _lib_or_skip()
    d1, b1, w1 = _w((25, c1), c1), _b(c1, c1), _w((co, c1), c1 + co)
    d2, b2, w2 = (_w((25, c2), c2 + 1), _b(c2, c2 + 1), _w((co, c2), c2 + co + 1)) if c2 else (None, None, None)

    def addr(a):
        return None if a is None else a.ctypes.data
    dw = lib.lp_head_fused_dw_elems(c1, c2)
    _pack_twice(lambda dc, bc, pc: lib.lp_head_fused_pack(d1.ctypes.data, b1.ctypes.data, addr(d2), addr(b2),
                                                          w1.ctypes.data, addr(w2), c1, c2, co, dc, bc, pc),
                [(dw, np.float16), (dw // 25, np.float32), (lib.lp_head_fused_pw_elems(c1, c2, co), np.float16)])


# (Cin, Ce): Ce a multiple of the 32-channel slab and not (40, 48, 200)
@pytest.mark.parametrize("cin,ce", [(16, 96), (24, 40), (8, 48), (48, 288), (16, 200)])
def test_block_s1_pack_wexp_footprint(cin, ce):
    lib = _lib_or_skip()
    w = _w((ce, cin), cin + ce)
    _pack_twice(lambda out: lib.lp_block_s1_pack_wexp(w.ctypes.data, cin, ce, out),
                [(lib.lp_block_s1_wexp_elems(cin, ce), np.float16)])


def test_every_launching_entry_point_has_a_footprint_case():
    """every symbol of _lib.SIGNATURES but the packers, *_elems, *_supported, *_workspace_bytes and library state"""
    missing = fc.launching_symbols() - fc.covered_symbols()
    assert not missing, "entry points without a footprint case: %s" % sorted(missing)
    unknown = fc.covered_symbols() - fc.launching_symbols()
    assert not unknown, "footprint cases name symbols that launch nothing: %s" % sorted(unknown)
    assert len(fc.launching_symbols()) >= 31


def test_footprint_case_ids_are_unique():
    ids = [c.id for c in fc.CASES]
    assert len(ids) == len(set(ids))
