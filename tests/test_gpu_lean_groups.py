"""`-m gpu`: aggregation and checksum requests run the units that take the lean kernel as one launch group (all of them
over device-resident blocks, the units of one staged block over host-resident ones): the CTAs claim tiles from one
counter across units, attribute rows per unit, and hand runs over into per-unit segments that scan_body then reads in
list mode.  Checked against the oracle and against the same request over the host-resident source."""
import pytest

import kvfmt
import orc
import scenarios as sc
from test_gpu_request_units import _gen_block, check_request, many_ranges
from tikv_b200 import ffi
from tikv_b200.executor import BatchExecutor, DagHandler, DeviceRegion, checksum
from tikv_b200.plan import ColumnDef, Plan, col, const_int, lt

pytestmark = pytest.mark.gpu

AGG_PLANS = [(n, p) for n, p in sc.plans() if n in ("group_by_small", "count_star", "agg_after_filter")]


def odd_ranges():
    """Units whose entry counts are not multiples of 256, and units of a single entry."""
    r = lambda lo, hi: kvfmt.table_range(sc.TABLE, lo, hi)  # noqa: E731
    return [r(-1000, 7), r(7, 8), r(8, 9), r(9, 300), r(300, 301), r(301, 1777), r(1777, 1778), r(1778, 4000)]


@pytest.mark.parametrize("desc", [False, True])
def test_forty_blocks_many_ranges(desc):
    """~40 blocks, 12 ranges or units of one entry: Lock / Rollback records in every block, so every unit hands runs over
    to its own segment."""
    host = sc.dirty_region(21, n_keys=4000).build(read_ts=sc.READ_TS, n_write_blocks=40)
    for ranges in (many_ranges(), odd_ranges(), sc.WHOLE):
        for name, plan in AGG_PLANS:
            check_request(plan, name, ranges, host)
        st, exp, _ = orc.checksum(ranges, host)
        for region in (DeviceRegion(host), host):
            rc, got, msg = checksum(ranges, region)
            assert st == 0 == rc and got == exp, msg
    # FIRST and BIT_* with and without a key, forward and backward: the device-resident request (one group) and the
    # host-resident one (a group per block) agree
    for group_by in ([], [col(sc.C2)]):
        plan = Plan().table_scan(sc.TABLE, sc.COLUMNS, desc=desc).aggregation([("first", col(sc.C1)), ("bit_xor", col(sc.C1)), ("bit_or", col(sc.C3)), ("count", col(sc.C1))],
                                                                        group_by=group_by).build()
        res = [DagHandler(plan, many_ranges(), region).handle_request() for region in (DeviceRegion(host), host)]
        assert res[0].status == 0 == res[1].status, res[0].message
        key = lambda r: sorted(zip(*[tuple(c) for c in r.columns]), key=repr)  # noqa: E731
        assert key(res[0]) == key(res[1])
        assert res[0].stats.write_processed_keys == res[1].stats.write_processed_keys


def test_unit_without_the_lean_kernel_inside_a_group():
    """A unit whose keys do not all share their first 12 bytes (negative and positive handles) has fast_ok = 0: that unit
    runs the general kernel while the other units of the request form the group."""
    r = kvfmt.Region()
    for h in range(-600, 2400):
        r.put(kvfmt.row_key(sc.TABLE, h), kvfmt.row_v2([(1, h * 3 - 500, "int"), (2, h % 7, "int")]), 10, 20)
    host = r.build(read_ts=sc.READ_TS, n_write_blocks=6)
    for ranges in (sc.WHOLE, odd_ranges()):
        for name, plan in AGG_PLANS:
            check_request(plan, name, ranges, host)


def test_rows_per_range_over_a_group():
    """Per-range rows of an aggregation over many ranges and blocks: each unit's rows go to its own range's slot."""
    host = sc.dirty_region(23, n_keys=2000).build(read_ts=sc.READ_TS, n_write_blocks=9)
    ranges = many_ranges()
    per_range = [len(orc.mvcc_scan(host, kvfmt.enc_bytes_memcmp(lo), kvfmt.enc_bytes_memcmp(hi))[1]) for lo, hi in ranges]
    plan = dict(AGG_PLANS)["group_by_small"]
    for region in (DeviceRegion(host), host):
        with BatchExecutor(plan, ranges, region) as ex:
            got = [0] * len(ranges)
            while True:
                res = ex.next_batch(1 << 20)
                assert res.error is None
                for i, n in enumerate(ex.collect_scanned_rows_per_range()):
                    got[i] += n
                if res.is_drained:
                    break
        assert got == per_range


def test_sixteen_device_blocks_make_one_lean_launch():
    """A clean C3-shaped request over 16 device-resident blocks: one lean launch and 16 list-mode launches, not a lean and
    a list-mode launch per unit (32)."""
    n_blocks, per = 16, 40_000
    gens = [_gen_block(per, 1000 + i * per, seed=5 + i) for i in range(n_blocks)]
    try:
        arr = (ffi.CfBlock * n_blocks)(*[b.block for _, b in gens])
        s = ffi.RegionSource()
        s.location, s.device, s.write, s.n_write, s.read_ts, s.isolation_level, s.check_has_newer_ts_data = ffi.LOC_DEVICE, 0, arr, n_blocks, 1000, ffi.ISO_SI, 1

        class Src:
            c = s
        columns = [ColumnDef(100, pk_handle=True), ColumnDef(1, tp=ffi.TP_LONG), ColumnDef(2)]
        plan = Plan().table_scan(sc.TABLE, columns).selection(lt(col(2), const_int(0))).aggregation([("sum", col(2))], group_by=[col(1, tp=ffi.TP_LONG)]).build()
        r = DagHandler(plan, sc.WHOLE, Src).handle_request()
        assert r.status == 0, r.message
        assert r.stats.kernel_launches == 1 + n_blocks
        assert r.stats.write_processed_keys == n_blocks * per
    finally:
        for g, _ in gens:
            ffi.lib().b2_gen_destroy(g)
