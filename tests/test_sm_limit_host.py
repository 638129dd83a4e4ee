"""CPU: lp_set_sm_limit / lp_get_sm_limit, the SM count the persistent kernels size their grids from.

With no device, the library counts 132 SMs (an H100 SXM), so the clamp to the device's count is checked against 132
here; test_gpu_sm_limit.py checks it against the device's own count and checks that the grids follow it."""
import os
import re
import threading

import pytest

import footprint_cases as fc
from litepose_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = {"lp_set_sm_limit", "lp_get_sm_limit"}


@pytest.fixture
def lib():
    try:
        lib = _lib.load()
    except _lib.LitePoseLibraryError as e:       # pragma: no cover - the library is built before the suite runs
        pytest.skip(str(e))
    lib.lp_set_sm_limit(0)
    device = lib.lp_get_sm_limit()
    try:
        yield lib
    finally:
        lib.lp_set_sm_limit(0)
    assert lib.lp_get_sm_limit() == device


def _device_sms():
    try:
        import torch
        if torch.cuda.is_available():
            return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    except Exception:                              # pragma: no cover
        pass
    return 132


def test_sm_limit_setter_and_getter(lib):
    device = _device_sms()
    assert lib.lp_get_sm_limit() == device
    for n in (1, 2, 3, 7, 16, 66, device - 1, device):
        lib.lp_set_sm_limit(n)
        assert lib.lp_get_sm_limit() == n, n
    for n in (device + 1, 4 * device, 2 ** 31 - 1):      # a cap above the device's count has no effect
        lib.lp_set_sm_limit(n)
        assert lib.lp_get_sm_limit() == device, n
    lib.lp_set_sm_limit(5)
    lib.lp_set_sm_limit(0)                                # 0 restores the device's count ...
    assert lib.lp_get_sm_limit() == device
    for n in (-1, -132, -2 ** 31):                        # ... and so does any negative value
        lib.lp_set_sm_limit(5)
        lib.lp_set_sm_limit(n)
        assert lib.lp_get_sm_limit() == device, n


def test_sm_limit_is_process_wide(lib):
    """a thread started after the call sees the limit, and a limit set in a thread holds for the caller too"""
    lib.lp_set_sm_limit(3)
    seen = []
    t = threading.Thread(target=lambda: (seen.append(lib.lp_get_sm_limit()), lib.lp_set_sm_limit(11)))
    t.start()
    t.join()
    assert seen == [3]
    assert lib.lp_get_sm_limit() == 11


def test_debug_header_matches_binding():
    """every symbol include/litepose_b200_debug.h declares is exported and bound (_lib.DEBUG_SIGNATURES) with the
    declared types, and none is in another table: the inference table (and so its footprint coverage) is unchanged"""
    hdr = open(os.path.join(ROOT, "include", "litepose_b200_debug.h")).read()
    code = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    assert set(re.findall(r"\b(lp_[a-z0-9_]+)\s*\(", code)) == set(_lib.DEBUG_SIGNATURES) == NAMES
    assert re.search(r"\bvoid\s+lp_set_sm_limit\s*\(\s*int\s+n\s*\)\s*;", code)
    assert re.search(r"\bint\s+lp_get_sm_limit\s*\(\s*void\s*\)\s*;", code)
    assert _lib.DEBUG_SIGNATURES["lp_set_sm_limit"] == (None, [_lib._i])
    assert _lib.DEBUG_SIGNATURES["lp_get_sm_limit"] == (_lib._i, [])
    for table in (_lib.SIGNATURES, _lib.TRAIN_SIGNATURES, _lib.TRAIN_BN_SIGNATURES):
        assert not NAMES & set(table)
    assert not NAMES & fc.launching_symbols() and not NAMES & fc.covered_symbols()
    try:
        lib = _lib.load()
    except _lib.LitePoseLibraryError as e:       # pragma: no cover - the library is built before the suite runs
        pytest.skip(str(e))
    assert all(hasattr(lib, s) for s in NAMES)
