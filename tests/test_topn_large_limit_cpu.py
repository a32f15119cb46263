"""TopN LIMIT up to 4096 on the device path, without a GPU: what plan lowering accepts and refuses, and that the limit
stays a launch parameter, so a large-limit plan reuses the plan-specialised kernel of the same ORDER BY."""
import ctypes as C
import os
import sys

import pytest

import emu
import scenarios as sc
from tikv_b200 import ffi
from tikv_b200.plan import Plan, col

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _topn(limit, order=None):
    order = order or [(col(sc.C2), True), (col(sc.C6), False)]
    return Plan().table_scan(sc.TABLE, sc.COLUMNS).topn(order, limit).build()


@pytest.mark.parametrize("limit", [1, 2048, 2049, 4000, 4095, 4096])
def test_limits_up_to_4096_are_accepted(limit):
    L = ffi.lib()
    plan = _topn(limit)
    assert L.b2_check_supported(C.byref(plan.c)) == ffi.B2_OK, L.b2_last_error_message()
    assert emu.check_supported(plan) == (ffi.B2_OK, "")


@pytest.mark.parametrize("limit", [4097, 5000, 1 << 20, (1 << 64) - 1])
def test_limits_above_4096_are_refused_with_a_message(limit):
    L = ffi.lib()
    plan = _topn(limit)
    assert L.b2_check_supported(C.byref(plan.c)) == ffi.B2_ERR_UNSUPPORTED
    assert b"4096" in L.b2_last_error_message()
    rc, msg = emu.check_supported(plan)
    assert rc == ffi.B2_ERR_UNSUPPORTED and "4096" in msg


def test_large_limit_plan_reuses_the_cached_kernel():
    """LIMIT 4096 and LIMIT 10 of one ORDER BY are one plan shape: the second precompile is served by the on-disk cache
    and runs no NVRTC compilation."""
    pytest.importorskip("cuda.bindings.nvrtc")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import jit_compile_check as J
    assert J.literal_of(_topn(10)) == J.literal_of(_topn(4096)) == J.literal_of(_topn(2049))
    L = ffi.lib()
    n = C.c_int32(-1)
    assert L.b2_plan_precompile(C.byref(_topn(10).c), C.byref(n)) == 0, L.b2_last_error_message()
    compiles, hits = C.c_uint64(0), C.c_uint64(0)
    L.b2_jit_counters(C.byref(compiles), C.byref(hits))
    before = compiles.value
    for limit in (4096, 3000):
        assert L.b2_plan_precompile(C.byref(_topn(limit).c), C.byref(n)) == 0, L.b2_last_error_message()
        assert n.value == 0, limit  # nothing compiled: the LIMIT 10 kernel is the one
    L.b2_jit_counters(C.byref(compiles), C.byref(hits))
    assert compiles.value == before
