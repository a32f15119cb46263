"""`-m "not gpu"`: the device's FIRST / BIT_* state code (tikv_b200/csrc/b2_device.h: first_agg_key, bit_agg_word,
first_bit_update, agg_word_op, first_bit_result, on the state layout plan_compile.h lays out) run on the CPU through
tests/first_bit_emul.cpp, over the oracle's scan rows, against the reference semantics: the scenario plans over dirty
regions (forward and backward, 1 and 3 blocks, whole and split ranges, rows spread over several partial states that
merge in reverse order) and the reference's own test_select.rs FIRST / bit-op cases."""
import ctypes as C
import os
import subprocess

import pytest

import scenarios as sc
from first_bit_ref import NEW_KINDS, WIDTH, _group_key, bits, scenario_specs, select_cases, select_region
from tikv_b200 import ffi

import orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "first_bit_emul.cpp")
SO = os.path.join(ROOT, "tests", "_build", "libfbe.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        deps = [SRC] + [os.path.join(ROOT, "tikv_b200", "csrc", f) for f in ("b2_device.h", "plan_compile.h")] + [os.path.join(ROOT, "include", "b2_copr.h")]
        if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
            os.makedirs(os.path.dirname(SO), exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", SO, SRC])
        L = C.CDLL(SO)
        L.fbe_run.argtypes = [C.POINTER(ffi.DagPlan), C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64),
                              C.POINTER(C.c_uint8), C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint8), C.c_char_p, C.c_size_t]
        L.fbe_run.restype = C.c_int
        _lib = L
    return _lib


def _raw(v):
    b = bits(v)
    return (0, 0) if b is None else (b[1], 1)


def emulate(spec, ranges, region, part_rows=7, n_parts=5):
    """{group key: [cells of the FIRST / BIT_* aggregates, in plan order]} as the device state code computes them."""
    scan = orc.dag_handle(spec._scan().build(), ranges, region)
    assert scan.status == 0, scan.message
    rows = scan.rows()
    fast_hash = len(spec.group_by) == 1
    keys, gid = {}, []
    for r in rows:
        gid.append(keys.setdefault(_group_key([r[c] for c, _ in spec.group_by], fast_hash), len(keys)))
    if not spec.group_by and not keys:
        keys[()] = 0
    na, n, ng = len(spec.aggs), len(rows), len(keys)
    vals = [_raw(r[c]) for r in rows for _, c, _ in spec.aggs]
    out, nn = (C.c_uint64 * max(1, ng * na))(), (C.c_uint8 * max(1, ng * na))()
    msg = C.create_string_buffer(256)
    rc = lib().fbe_run(C.byref(spec.plan().c), int(spec.desc), n, part_rows, n_parts, (C.c_uint32 * max(1, n))(*gid),
                       (C.c_uint64 * max(1, n * na))(*[v for v, _ in vals]), (C.c_uint8 * max(1, n * na))(*[h for _, h in vals]),
                       ng, out, nn, msg, 256)
    assert rc == 0, (rc, msg.value)
    kind_of = [k for k, _, _ in spec.aggs]
    real = [kw.get("tp") == ffi.TP_DOUBLE for _, _, kw in spec.aggs]
    res = {}
    for key, g in keys.items():
        cells = []
        for a in range(na):
            if kind_of[a] not in NEW_KINDS:
                continue
            v = out[g * na + a]
            cells.append(None if not nn[g * na + a] else (("f" if real[a] and kind_of[a] == "first" else "i"), v))
        res[key] = cells
    return res


def _new_cells(spec, exp):
    idx, pos = [], 0
    for kind, _, _ in spec.aggs:
        if kind in NEW_KINDS:
            idx.append(pos)
        pos += WIDTH[kind]
    return {k: [v[i] for i in idx] for k, v in exp.items()}


@pytest.mark.parametrize("desc", [False, True], ids=["fwd", "bwd"])
@pytest.mark.parametrize("blocks", [1, 3])
def test_scenarios_state_code_matches_reference(blocks, desc):
    host = sc.dirty_region(21, n_keys=1500).build(read_ts=sc.READ_TS, n_write_blocks=blocks)
    for name, spec in scenario_specs(desc):
        for ranges in (sc.WHOLE, sc.split_ranges()):
            exp = _new_cells(spec, spec.expected(ranges, host))
            for part_rows, n_parts in ((1, 1), (7, 5), (256, 3)):
                got = emulate(spec, ranges, host, part_rows, n_parts)
                assert got == exp, (name, blocks, desc, part_rows)


@pytest.mark.parametrize("desc", [False, True], ids=["fwd", "bwd"])
def test_reference_select_cases(desc):
    """test_select.rs test_aggr_first / test_aggr_bit_ops: the reference's expected rows, from the reference semantics
    over the oracle's scan and from the device state code."""
    for name, rows, spec, want in select_cases(desc):
        region = select_region(rows)
        assert spec.expected(sc.WHOLE, region) == want, name
        assert emulate(spec, sc.WHOLE, region) == want, name
