"""`-m gpu`: opening and finishing a request over device-resident blocks.

A device-resident source is read once while the request opens: one probe launch returns every block's heap sizes, the
range bounds in every CF_WRITE block, the unit prefixes and the first value of the first unit (the row-format sample),
and writes the CF_DEFAULT views.  An aggregation compacts its group table behind the last unit and reads its counters
once.  Every case is checked against the oracle and against the same request over the host-resident source, whose
blocks are read on the host."""
import ctypes as C

import pytest

import kvfmt
import orc
import scenarios as sc
from compare import assert_same_rows
from tikv_b200 import ffi
from tikv_b200.executor import BatchExecutor, DagHandler, DeviceRegion, checksum
from tikv_b200.plan import ColumnDef, Plan, col, const_int, le

pytestmark = pytest.mark.gpu

AGG_PLANS = [(n, p) for n, p in sc.plans() if n in ("group_by_small", "count_star", "agg_after_filter")]
SCAN_PLANS = [(n, p) for n, p in sc.plans() if n in ("sel_lt_const", "scan_all")]


def many_ranges():
    """Several ranges per block, ranges of one key, ranges between keys (no unit) and ranges past the table."""
    r = lambda lo, hi: kvfmt.table_range(sc.TABLE, lo, hi)  # noqa: E731
    return [r(-1000, -95), r(-94, 50), r(50, 51), r(51, 52), r(60, 200), r(200, 203), r(203, 900), r(901, 902), r(905, 1700),
            r(1700, 2600), r(2600, 2800), r(5000, 6000)]


def check_request(plan, name, ranges, host):
    exp = orc.dag_handle(plan, ranges, host)
    assert exp.status == 0
    for region in (DeviceRegion(host), host):
        got = DagHandler(plan, ranges, region).handle_request()
        assert_same_rows(got, exp, ordered=not sc.is_agg(name), ctx=f"{name}/{'host' if region is host else 'device'}")
        assert got.stats.write_processed_keys == exp.stats["processed_keys"], name
        assert got.stats.processed_size == exp.stats["processed_size"], name
        assert got.stats.default_lookups == exp.stats["data_processed_keys"], name
        assert got.stats.met_newer_ts_data == exp.stats["met_newer"], name


@pytest.mark.parametrize("fmt", [None, 1, 2])
@pytest.mark.parametrize("n_blocks", [1, 4, 7])
def test_many_blocks_and_ranges(n_blocks, fmt):
    """Every MVCC shape (CF_DEFAULT values included) over 1 .. 7 blocks and 12 ranges; rows of format v1, v2 or both, so
    the row-format sample of the first unit decides both ways."""
    host = sc.dirty_region(5, n_keys=900, only_fmt=fmt).build(read_ts=sc.READ_TS, n_write_blocks=n_blocks)
    assert host.dblock is not None
    for ranges in (many_ranges(), sc.WHOLE):
        for name, plan in AGG_PLANS + SCAN_PLANS:
            check_request(plan, name, ranges, host)
        st, exp, _ = orc.checksum(ranges, host)
        for region in (DeviceRegion(host), host):
            rc, got, msg = checksum(ranges, region)
            assert st == 0 == rc and got == exp, msg


def test_no_units():
    """Ranges that hold no key of any block: no unit, an empty result, the statistics of an empty scan."""
    host = sc.dirty_region(6, n_keys=300).build(read_ts=sc.READ_TS, n_write_blocks=3)
    ranges = [kvfmt.table_range(sc.TABLE, 51, 52), kvfmt.table_range(sc.TABLE, 5000, 6000)]
    for name, plan in AGG_PLANS + SCAN_PLANS:
        check_request(plan, name, ranges, host)
    assert checksum(ranges, DeviceRegion(host))[:2] == orc.checksum(ranges, host)[:2]


def test_blocks_of_different_entry_sizes():
    """One request over blocks whose average entry sizes differ tenfold (short rows, then rows near the 255-byte limit of
    a short value), each block's heap sizes coming from the open probe."""
    r = kvfmt.Region()
    for h in range(1500):
        pad = 180 if 500 <= h < 1000 else 0
        cols = [(1, h * 7 - 300, "int"), (2, h % 5, "int"), (3, h, "uint"), (4, 0.5 * h, "f64"), (6, h % 9, "int")]
        if pad:
            cols.append((7, bytes(pad), "bytes"))
        r.put(kvfmt.row_key(sc.TABLE, h), kvfmt.row_v2(cols), 10, 20)
    host = r.build(read_ts=sc.READ_TS, n_write_blocks=3)
    for ranges in (sc.WHOLE, [kvfmt.table_range(sc.TABLE, 400, 1100)]):
        for name, plan in AGG_PLANS + SCAN_PLANS:
            check_request(plan, name, ranges, host)


def test_rows_per_range_and_scanned_range():
    """Per-range rows, processed keys and take_scanned_range of a device-resident scan over many ranges equal the host
    source's and the oracle's."""
    host = sc.dirty_region(7, n_keys=900).build(read_ts=sc.READ_TS, n_write_blocks=4)
    ranges = many_ranges()
    plan = dict(SCAN_PLANS)["sel_lt_const"]
    per_range = [len(orc.mvcc_scan(host, kvfmt.enc_bytes_memcmp(lo), kvfmt.enc_bytes_memcmp(hi))[1]) for lo, hi in ranges]
    seen = []
    for region in (DeviceRegion(host), host):
        with BatchExecutor(plan, ranges, region) as ex:
            got, takes = [0] * len(ranges), []
            while True:
                res = ex.next_batch(200)
                assert res.error is None
                takes.append(ex.take_scanned_range())
                for i, n in enumerate(ex.collect_scanned_rows_per_range()):
                    got[i] += n
                if res.is_drained:
                    break
            st = ex.collect_exec_stats()
        assert got == per_range and takes[0][0] == ranges[0][0] and takes[-1][1] == ranges[-1][1]
        assert all(takes[i][1] == takes[i + 1][0] for i in range(len(takes) - 1))
        seen.append((takes, st.write_processed_keys, st.met_newer_ts_data))
    assert seen[0] == seen[1]


def _gen_block(n_rows, first_handle, seed=11):
    L = ffi.lib()
    spec = ffi.GenSpec()
    spec.table_id, spec.first_handle, spec.n_rows, spec.n_cols, spec.row_format, spec.seed = sc.TABLE, first_handle, n_rows, 4, 2, seed
    lo, rng = (C.c_int64 * 4)(0, 0, 0, 0), (C.c_uint64 * 4)(0, 37, 0, 0)
    spec.col_lo, spec.col_range = lo, rng
    spec.commit_ts, spec.newer_ts = 100, 5000
    g, blk = C.c_void_p(), ffi.GenBlock()
    assert L.b2_gen_create(0, C.byref(spec), C.byref(g), C.byref(blk)) == 0, L.b2_last_error_message()
    return g, blk


def test_table_growth_and_redo_over_several_units():
    """4.5 M groups over three blocks (three units): the first HBM table (2^22 slots) overflows, the compacted group list
    of that pass is discarded, the table grows and all units run again."""
    n_rows, first, parts = 4_500_000, 1000, 3
    gens = [_gen_block(n_rows // parts, first + i * (n_rows // parts)) for i in range(parts)]
    try:
        arr = (ffi.CfBlock * parts)(*[b.block for _, b in gens])
        s = ffi.RegionSource()
        s.location, s.device, s.write, s.n_write, s.read_ts, s.isolation_level, s.check_has_newer_ts_data = ffi.LOC_DEVICE, 0, arr, parts, 1000, ffi.ISO_SI, 1

        class Src:
            c = s
        columns = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(4)]
        r = DagHandler(Plan().table_scan(sc.TABLE, columns).aggregation([("count", const_int(1)), ("max", col(0))], group_by=[col(0)]).build(),
                       sc.WHOLE, Src).handle_request()
        assert r.status == 0, r.message
        assert r.n_rows == n_rows and all(x == 1 for x in r.columns[0])
        want_sum = n_rows * first + n_rows * (n_rows - 1) // 2
        assert sum(r.columns[1]) == want_sum and sum(r.columns[2]) == want_sum
        assert r.stats.write_processed_keys == n_rows
    finally:
        for g, _ in gens:
            ffi.lib().b2_gen_destroy(g)


def test_division_by_zero_warnings_over_many_units():
    """Warnings of a projection that divides by zero, over 4 blocks and many ranges: the device-resident and the
    host-resident source count what the oracle counts."""
    from tikv_b200.executor import _read_batch
    from tikv_b200.plan import const_real, divide, multiply
    host = sc.dirty_region(8, n_keys=900).build(read_ts=sc.READ_TS, n_write_blocks=4)
    c4 = col(sc.C4, tp=ffi.TP_DOUBLE)
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).projection(col(sc.C_H), divide(c4, multiply(c4, const_real(0.0)))).build()
    ranges = many_ranges()
    exp = orc.dag_handle(plan, ranges, host)
    assert exp.status == 0 and exp.warning_count > 100
    for region in (DeviceRegion(host), host):
        with BatchExecutor(plan, ranges, region) as ex:
            rows, per_batch = [], 0
            while True:
                rc, b = ex.next_batch_raw(300)
                assert rc == 0
                per_batch += b.n_warnings
                cols, _, _ = _read_batch(b, ffi.LOC_HOST)
                rows += list(zip(*cols)) if cols else []
                if b.is_drained != ffi.DRAIN_REMAIN:
                    break
            total, details = ex.warnings()
        assert rows == exp.rows()
        assert total == exp.warning_count == per_batch and details[0] == (1365, "Division by 0")


def _jit_events():
    a, b = C.c_uint64(), C.c_uint64()
    ffi.lib().b2_jit_counters(C.byref(a), C.byref(b))
    return a.value + b.value  # kernels compiled + kernels loaded from the disk cache (an in-process hit counts neither)


def test_row_format_sample_picks_the_first_unit():
    """The row-format sample (the first value of the first unit) decides whether the plan-specialised kernel carries the
    row-format-v1 twin; that kernel variant is a separate compilation.  Rows are v2 below handle 600 and v1 from it on, in 3
    blocks.  For each set of ranges the device-resident request (sample read by the open probe) and the host-resident one
    (sample read on the host) must pick the same variant: the second request then finds the first one's kernel in the
    process and compiles or loads nothing.  Only speed depends on the pick, so results alone could not show a wrong one."""
    r = kvfmt.Region()
    for h in range(1200):
        vals = [(1, h * 7 - 300), (2, h % 5), (3, h % 11)]
        row = kvfmt.row_v2([(cid, v, "int") for cid, v in vals]) if h < 600 else kvfmt.row_v1([(cid, kvfmt.datum_int(v)) for cid, v in vals])
        r.put(kvfmt.row_key(sc.TABLE, h), row, 10, 20)
    host = r.build(read_ts=sc.READ_TS, n_write_blocks=3)
    columns = [ColumnDef(100, pk_handle=True), ColumnDef(1), ColumnDef(2), ColumnDef(3)]
    # a plan shape of its own, so that no other test has put its kernels in the process
    plan = (Plan().table_scan(sc.TABLE, columns).selection(le(col(2), const_int(3)))
            .aggregation([("max", col(1)), ("count", col(3)), ("min", col(2))], group_by=[col(3, tp=ffi.TP_LONG)]).build())
    dev = DeviceRegion(host)
    v1_only = [kvfmt.table_range(sc.TABLE, 900, 1100), kvfmt.table_range(sc.TABLE, 1150, 1160)]  # first unit in the last block
    v2_first = [kvfmt.table_range(sc.TABLE, 0, 50), kvfmt.table_range(sc.TABLE, 700, 1000)]       # first unit: v2 rows
    events = []
    for ranges in (v1_only, v2_first):
        exp = orc.dag_handle(plan, ranges, host)
        for region in (dev, host):
            before = _jit_events()
            got = DagHandler(plan, ranges, region, jit=ffi.JIT_SYNC).handle_request()
            assert_same_rows(got, exp, ordered=False, ctx="sample")
            events.append(_jit_events() - before)
    if events[0] == 0:
        pytest.skip("plan-specialised kernels are not available in this process")
    # device v1 variant (new), host same (none); device v2 variant (new), host same (none)
    assert events == [1, 0, 1, 0], events
