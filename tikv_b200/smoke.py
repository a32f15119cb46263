"""One small pass of the hot path on cuda:0 through the C ABI, checked against the oracle (used by smoke())."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def plans():
    """The two DAGs smoke() runs (also precompiled by __graft_entry__.build())."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import scenarios as sc
    from tikv_b200.plan import Plan, col, const_int, lt
    scan_filter = Plan().table_scan(sc.TABLE, sc.COLUMNS).selection(lt(col(sc.C1), const_int(0))).build()
    hash_agg = (Plan().table_scan(sc.TABLE, sc.COLUMNS).selection(lt(col(sc.C1), const_int(1 << 62)))
                .aggregation([("sum", col(sc.C1)), ("count", const_int(1))], group_by=[col(sc.C6)]).build())
    return [scan_filter, hash_agg]


def run():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import kvfmt
    import orc
    import scenarios as sc
    from compare import assert_same_rows
    import sstfmt
    import sstlz4
    from tikv_b200.executor import DagHandler, DeviceRegion, SstRegion, checksum

    host = sc.dirty_region(3, n_keys=2000).build(read_ts=sc.READ_TS, n_write_blocks=2)  # (three blocks: 3034 + 3034 + 1 entries)
    dev = DeviceRegion(host)
    scan_filter, hash_agg = plans()
    for name, plan, ordered in (("scan+filter", scan_filter, True), ("scan+filter+hash-agg", hash_agg, False)):
        for region in (host, dev):
            assert_same_rows(DagHandler(plan, sc.WHOLE, region).handle_request(), orc.dag_handle(plan, sc.WHOLE, host), ordered=ordered, ctx=name)
    # the same region arriving as RocksDB data blocks (built by the checker): expanded on the device, then scanned,
    # and as the same blocks stored LZ4-compressed (inflated on the device first)
    for what, build in (("data blocks", sstfmt.build), ("LZ4 data blocks", sstlz4.build)):
        sst = SstRegion(host, [build(b, block_size=4096) for b in host.wblocks])
        try:
            assert_same_rows(DagHandler(hash_agg, sc.WHOLE, sst).handle_request(), orc.dag_handle(hash_agg, sc.WHOLE, host), ordered=False, ctx=what + " -> scan+filter+hash-agg")
            assert (sum(st.n_lz4_blocks for st in sst.stats) > 0) == (build is sstlz4.build), what
        finally:
            sst.close()
    st, exp, _ = orc.checksum(sc.WHOLE, host)
    rc, got, msg = checksum(sc.WHOLE, dev)
    assert st == 0 == rc and got == exp, msg
