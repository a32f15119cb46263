"""`-m gpu`: parity of the CUDA path (through the C ABI) against the oracle on seeded inputs.
Bit-exact for ints / counts / decimals / CRC; f64 SUM within 1e-12 relative (atomic summation order)."""
import ctypes as C

import numpy as np
import pytest

import kvfmt
import orc
import scenarios as sc
from compare import assert_same_rows
from tikv_b200 import ffi
from tikv_b200.executor import BatchExecutor, DagHandler, DeviceRegion, checksum
from tikv_b200.plan import ColumnDef, Plan, col, const_int, lt, multiply

pytestmark = pytest.mark.gpu

PLANS = sc.plans()


@pytest.fixture(scope="module")
def regions():
    return {seed: sc.dirty_region(seed, n_keys=900) for seed in (1, 2)}


@pytest.mark.parametrize("name,plan", PLANS, ids=[n for n, _ in PLANS])
def test_host_source_matches_oracle(name, plan, regions):
    """HOST-resident blocks: the engine stages them to HBM itself (H2D inside the call)."""
    for seed, n_blocks, ranges in ((1, 1, sc.WHOLE), (2, 3, sc.split_ranges())):
        region = regions[seed].build(read_ts=sc.READ_TS, n_write_blocks=n_blocks)
        exp = orc.dag_handle(plan, ranges, region)
        got = DagHandler(plan, ranges, region).handle_request()
        assert_same_rows(got, exp, ordered=not sc.is_agg(name), ctx=f"{name}/seed{seed}")
        assert got.stats.write_processed_keys == exp.stats["processed_keys"]
        assert got.stats.processed_size == exp.stats["processed_size"]
        assert got.stats.default_lookups == exp.stats["data_processed_keys"]
        assert got.stats.met_newer_ts_data == exp.stats["met_newer"]


@pytest.mark.parametrize("name,plan", PLANS[:6] + PLANS[-8:], ids=[n for n, _ in PLANS[:6] + PLANS[-8:]])
def test_device_source_matches_oracle(name, plan, regions):
    host = regions[1].build(read_ts=sc.READ_TS, n_write_blocks=2)
    dev = DeviceRegion(host)
    exp = orc.dag_handle(plan, sc.split_ranges(), host)
    got = DagHandler(plan, sc.split_ranges(), dev).handle_request()
    assert_same_rows(got, exp, ordered=not sc.is_agg(name), ctx=name)


@pytest.mark.parametrize("scan_rows", [1, 7, 100, 256, 257, 1000])
def test_small_batches_keep_order(scan_rows, regions):
    """next_batch(scan_rows) with tiny batches: many launches, look-back across tiles, rows stay in key order."""
    host = regions[2].build(read_ts=sc.READ_TS, n_write_blocks=2)
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).selection(lt(col(sc.C1), const_int(1 << 62))).build()
    exp = orc.dag_handle(plan, sc.WHOLE, host)
    got = DagHandler(plan, sc.WHOLE, host, batch_rows=scan_rows).handle_request()
    assert_same_rows(got, exp, ordered=True, ctx=f"scan_rows={scan_rows}")


def test_batch_executor_interface(regions):
    host = regions[1].build(read_ts=sc.READ_TS)
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).build(output_offsets=[sc.C_H, sc.C4])
    with BatchExecutor(plan, sc.WHOLE, host) as ex:
        assert ex.schema() == [(ffi.TP_LONGLONG, 0), (ffi.TP_DOUBLE, 0)]
        r = ex.next_batch(500)
        assert not r.is_drained and r.kinds == [ffi.COL_I64, ffi.COL_F64]
        n = r.n_rows
        while not r.is_drained:
            r = ex.next_batch(500)
            n += r.n_rows
        st = ex.collect_exec_stats()
        assert st.num_produced_rows == n == orc.dag_handle(plan, sc.WHOLE, host).n_rows
        assert st.write_entries_scanned == host.n_entries and st.time_processed_ns > 0
        assert not ex.can_be_cached()  # the region holds versions newer than read_ts
    clean = kvfmt.Region()
    for h in range(10):
        clean.put(kvfmt.row_key(sc.TABLE, h), kvfmt.row_v2([(1, h, "int")]), 10, 20)
    with BatchExecutor(plan, sc.WHOLE, clean.build(read_ts=100)) as ex:
        assert ex.next_batch(1 << 20).n_rows == 10 and ex.can_be_cached()


@pytest.mark.parametrize("name,plan", sc.real_sum_plans())
def test_real_sum(name, plan, regions):
    host = regions[1].build(read_ts=sc.READ_TS)
    assert_same_rows(DagHandler(plan, sc.WHOLE, host).handle_request(), orc.dag_handle(plan, sc.WHOLE, host), ordered=False,
                     float_rel_tol=1e-12, ctx=name)


def test_real_sums_are_exactly_rounded(regions):
    """north_star: float SUM / AVG within 1 ULP.  The device sum is exact (fixed-point accumulator), so it is the correctly
    rounded true sum: 0 ULP, on host- and device-resident sources, generic and plan-specialised kernels alike."""
    host = regions[1].build(read_ts=sc.READ_TS)
    for region in (host, DeviceRegion(host)):
        for jit in (ffi.JIT_OFF, ffi.JIT_SYNC):
            sc.check_exact_real_sums(lambda plan: DagHandler(plan, sc.WHOLE, region, jit=jit).handle_request(), host)


def test_isolation_levels_and_read_ts(regions):
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).build()
    for ts in (1, 25, 150, sc.READ_TS + 100, (1 << 64) - 1):
        region = regions[2].build(read_ts=ts, isolation=ffi.ISO_RC)
        assert_same_rows(DagHandler(plan, sc.WHOLE, region).handle_request(), orc.dag_handle(plan, sc.WHOLE, region), ctx=f"ts{ts}")
    region = regions[2].build(read_ts=sc.READ_TS, isolation=ffi.ISO_RC_CHECK_TS)
    exp, got = orc.dag_handle(plan, sc.WHOLE, region), DagHandler(plan, sc.WHOLE, region).handle_request()
    assert exp.status == ffi.B2_ERR_WRITE_CONFLICT == got.status and got.rows() == exp.rows()


def test_locks(regions):
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).build(output_offsets=[sc.C_H])
    r = kvfmt.Region()
    for h in range(50):
        r.put(kvfmt.row_key(sc.TABLE, h), kvfmt.row_v2([(1, h, "int")]), 10, 20)
    r.add_lock(kvfmt.row_key(sc.TABLE, 30), kvfmt.lock_record(b"P", kvfmt.row_key(sc.TABLE, 30), 50))
    r.add_lock(kvfmt.row_key(sc.TABLE, 10), kvfmt.lock_record(b"L", kvfmt.row_key(sc.TABLE, 10), 50))  # Lock-type locks never block
    for kw in (dict(read_ts=100), dict(read_ts=100, bypass=[50]), dict(read_ts=40), dict(read_ts=100, isolation=ffi.ISO_RC)):
        region = r.build(**kw)
        exp, got = orc.dag_handle(plan, sc.WHOLE, region), DagHandler(plan, sc.WHOLE, region).handle_request()
        assert exp.status == got.status and got.rows() == exp.rows(), kw
    region = r.build(read_ts=100)
    got = DagHandler(plan, sc.WHOLE, region).handle_request()
    assert got.status == ffi.B2_ERR_KEY_IS_LOCKED and got.n_rows == 30 and not got.can_be_cached
    agg = Plan().table_scan(sc.TABLE, sc.COLUMNS).aggregation([("count", const_int(1))]).build()
    assert DagHandler(agg, sc.WHOLE, region).handle_request().status == ffi.B2_ERR_KEY_IS_LOCKED


def test_errors_match_oracle():
    T, cols = sc.TABLE, sc.COLUMNS
    base = kvfmt.Region()
    for h in range(600):
        base.put(kvfmt.row_key(T, h), kvfmt.row_v2([(1, h, "int"), (2, h % 5, "int"), (3, 7, "uint"), (4, 1.0, "f64"), (6, 1, "int")]), 10, 20)

    def with_extra(fn):
        r = kvfmt.Region()
        r.write, r.dflt = list(base.write), list(base.dflt)
        fn(r)
        return r.build(read_ts=100)

    plan = Plan().table_scan(T, cols).build()
    cases = [
        (plan, with_extra(lambda r: r.put(kvfmt.row_key(T, 333), kvfmt.row_v1([(1, kvfmt.datum_int(5))]) + bytes([kvfmt.VAR_INT, 0x80]), 30, 40)), ffi.B2_ERR_CORRUPTED),
        (plan, with_extra(lambda r: r.raw_write(kvfmt.row_key(T, 5), 50, b"Xjunk")), ffi.B2_ERR_STORAGE),
        (plan, with_extra(lambda r: r.write.append((kvfmt.write_key(kvfmt.row_key(T, 3), 60), kvfmt.write_record(b"P", 55)))), ffi.B2_ERR_STORAGE),
        (Plan().table_scan(T, cols).selection(lt(multiply(col(sc.C1), const_int(4)), const_int(100))).build(),
         with_extra(lambda r: r.put(kvfmt.row_key(T, 1000), kvfmt.row_v2([(1, 1 << 62, "int"), (6, 1, "int")]), 10, 20)), ffi.B2_ERR_EVALUATE),
    ]
    for p, region, status in cases:
        exp, got = orc.dag_handle(p, sc.WHOLE, region), DagHandler(p, sc.WHOLE, region).handle_request()
        assert exp.status == status == got.status, (got.message, exp.message)
        assert got.rows() == exp.rows()
        if status == ffi.B2_ERR_EVALUATE:
            assert got.mysql_code == exp.mysql_code == 1690


def test_checksum_matches_oracle(regions):
    for seed in (1, 2):
        host = regions[seed].build(read_ts=sc.READ_TS, n_write_blocks=2)
        for region in (host, DeviceRegion(host)):
            for ranges in (sc.WHOLE, sc.split_ranges()):
                st, exp, _ = orc.checksum(ranges, host)
                rc, got, msg = checksum(ranges, region)
                assert st == 0 == rc and got == exp and exp[1] > 0, msg
    old, new = b"t" + kvfmt.enc_i64_cmp(42), b"t" + kvfmt.enc_i64_cmp(sc.TABLE)
    host = regions[1].build(read_ts=sc.READ_TS)
    st, exp, _ = orc.checksum(sc.WHOLE, host, old, new)
    rc, got, _ = checksum(sc.WHOLE, host, old, new)
    assert rc == 0 == st and got == exp
    assert checksum(sc.WHOLE, host, b"", b"x")[0] != 0


def _gen_block(n_rows, n_cols, fmt, seed, lo=None, rng=None, nulls=None, extra=0, delete=0, lockrec=0, first_handle=0):
    L = ffi.lib()
    spec = ffi.GenSpec()
    spec.table_id, spec.first_handle, spec.n_rows, spec.n_cols, spec.row_format, spec.seed = sc.TABLE, first_handle, n_rows, n_cols, fmt, seed
    keep = []
    if lo is not None:
        a = (C.c_int64 * n_cols)(*lo); b = (C.c_uint64 * n_cols)(*rng); keep += [a, b]
        spec.col_lo, spec.col_range = a, b
    if nulls is not None:
        c = (C.c_uint32 * n_cols)(*nulls); keep.append(c)
        spec.null_per_million = c
    spec.extra_versions_per_million, spec.delete_per_million, spec.lock_rec_per_million = extra, delete, lockrec
    spec.commit_ts, spec.newer_ts = 100, 5000
    g, blk = C.c_void_p(), ffi.GenBlock()
    rc = L.b2_gen_create(0, C.byref(spec), C.byref(g), C.byref(blk))
    assert rc == 0, L.b2_last_error_message()
    return g, blk


def _block_to_host(blk):
    L = ffi.lib()
    n = blk.block.n
    keys = np.zeros(((blk.key_bytes + 31) // 16) * 16, dtype=np.uint8); vals = np.zeros(((blk.val_bytes + 31) // 16) * 16, dtype=np.uint8)
    koff = np.zeros(n + 1, dtype=np.uint32); voff = np.zeros(n + 1, dtype=np.uint32)
    assert L.b2_copy_to_host(0, keys.ctypes.data, blk.block.keys, blk.key_bytes) == 0
    assert L.b2_copy_to_host(0, vals.ctypes.data, blk.block.vals, blk.val_bytes) == 0
    assert L.b2_copy_to_host(0, koff.ctypes.data, blk.block.key_offs, 4 * (n + 1)) == 0
    assert L.b2_copy_to_host(0, voff.ctypes.data, blk.block.val_offs, 4 * (n + 1)) == 0
    hb = ffi.CfBlock()
    hb.keys, hb.key_offs, hb.vals, hb.val_offs, hb.n = keys.ctypes.data, koff.ctypes.data, vals.ctypes.data, voff.ctypes.data, n
    return hb, (keys, vals, koff, voff)


def _source(blocks, location, read_ts=1000):
    arr = (ffi.CfBlock * len(blocks))(*blocks)
    s = ffi.RegionSource()
    s.location, s.device, s.write, s.n_write, s.read_ts, s.isolation_level, s.check_has_newer_ts_data = location, 0, arr, len(blocks), read_ts, ffi.ISO_SI, 1

    class R:
        pass
    r = R()
    r.c, r._arr = s, arr
    return r


MIX_MASK = (1 << 64) - 1


def _mix64(x):
    x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & MIX_MASK; x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & MIX_MASK; x ^= x >> 33
    return x


def _gen_mix(seed, handle, salt):
    return _mix64(seed ^ ((handle * 0x9E3779B97F4A7C15) & MIX_MASK) ^ (((salt + 1) * 0xBF58476D1CE4E5B9) & MIX_MASK))


@pytest.mark.parametrize("fmt", [2, 1])
def test_generated_region_parity(fmt):
    """Device generator -> (a) closed-form check of decoded values, (b) oracle on the D2H copy == CUDA path on HBM."""
    n_cols, n_rows, seed = 8, 20000, 0x525C682A2F7CE3DB
    lo = [0, 0, -(1 << 40), 0, 0, 0, 0, 0]
    rng = [0, 1024, 1 << 41, 0, 0, 0, 3, 0]
    nulls = [0, 0, 0, 10000, 0, 0, 0, 0]
    g, blk = _gen_block(n_rows, n_cols, fmt, seed, lo, rng, nulls, extra=20000, delete=20000, lockrec=20000)
    try:
        hb, keep = _block_to_host(blk)
        host, dev = _source([hb], ffi.LOC_HOST), _source([blk.block], ffi.LOC_DEVICE)
        columns = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(n_cols)]
        scan = Plan().table_scan(sc.TABLE, columns).build()
        exp = orc.dag_handle(scan, sc.WHOLE, host)
        assert exp.status == 0 and 0.97 * n_rows < exp.n_rows < n_rows
        for row in exp.rows()[:2000]:
            h = row[0]
            for c in range(n_cols):
                want = None
                if not (nulls[c] and _gen_mix(seed, h, 500 + c) % 1000000 < nulls[c]):
                    x = _gen_mix(seed, h, c)
                    want = (lo[c] + x % rng[c]) if rng[c] else (x - (1 << 64) if x >= (1 << 63) else x)
                assert row[1 + c] == want, (h, c)
        for name, plan in (("scan", scan),
                           ("filter", Plan().table_scan(sc.TABLE, columns).selection(lt(col(1), const_int(0))).build()),
                           ("group", Plan().table_scan(sc.TABLE, columns).aggregation([("sum", col(3)), ("count", const_int(1)), ("avg", col(4))], group_by=[col(2)]).build()),
                           ("group3", Plan().table_scan(sc.TABLE, columns).aggregation([("sum", col(1))], group_by=[col(7)]).build()),
                           ("count", Plan().table_scan(sc.TABLE, columns).aggregation([("count", const_int(1)), ("sum", col(1))]).build())):
            e = orc.dag_handle(plan, sc.WHOLE, host)
            gres = DagHandler(plan, sc.WHOLE, dev).handle_request()
            assert_same_rows(gres, e, ordered=name in ("scan", "filter"), ctx=f"gen/{name}/v{fmt}")
        st, echk, _ = orc.checksum(sc.WHOLE, host)
        rc, gchk, _ = checksum(sc.WHOLE, dev)
        assert st == 0 == rc and echk == gchk
    finally:
        ffi.lib().b2_gen_destroy(g)


def test_large_scale_properties():
    """At a size the oracle does not run: size-independent properties of the CUDA path on generated data."""
    n_rows, n_cols, seed = 4_000_000, 8, 77
    blocks, gens = [], []
    for i in range(2):
        g, blk = _gen_block(n_rows // 2, n_cols, 2, seed, [0] * 8, [0, 1000, 0, 0, 0, 0, 0, 0], None, first_handle=i * (n_rows // 2))
        gens.append(g); blocks.append(blk.block)
    try:
        dev = _source(blocks, ffi.LOC_DEVICE)
        columns = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(n_cols)]
        cnt = DagHandler(Plan().table_scan(sc.TABLE, columns).aggregation([("count", const_int(1)), ("sum", col(0))]).build(), sc.WHOLE, dev).handle_request()
        assert cnt.rows() == [(n_rows, n_rows * (n_rows - 1) // 2)]
        # partition property: filter(x < 0) + filter(x >= 0) row counts add up; group counts add up to the total
        from tikv_b200.plan import ge
        neg = DagHandler(Plan().table_scan(sc.TABLE, columns).selection(lt(col(1), const_int(0))).aggregation([("count", const_int(1))]).build(), sc.WHOLE, dev).handle_request()
        pos = DagHandler(Plan().table_scan(sc.TABLE, columns).selection(ge(col(1), const_int(0))).aggregation([("count", const_int(1))]).build(), sc.WHOLE, dev).handle_request()
        assert neg.rows()[0][0] + pos.rows()[0][0] == n_rows and abs(neg.rows()[0][0] - n_rows // 2) < n_rows // 100
        grp = DagHandler(Plan().table_scan(sc.TABLE, columns).aggregation([("count", const_int(1)), ("sum", col(0))], group_by=[col(2)]).build(), sc.WHOLE, dev).handle_request()
        assert grp.n_rows == 1000 and sum(r[0] for r in grp.rows()) == n_rows and sum(r[1] for r in grp.rows()) == n_rows * (n_rows - 1) // 2
        # scan + filter keeps key order (handles strictly increasing) and splits consistently across batch sizes
        filt = Plan().table_scan(sc.TABLE, columns).selection(lt(col(2), const_int(10))).build(output_offsets=[0, 2])
        a = DagHandler(filt, sc.WHOLE, dev, batch_rows=1 << 22).handle_request()
        b = DagHandler(filt, sc.WHOLE, dev, batch_rows=300_000).handle_request()
        ha = np.asarray(a.columns[0]); assert np.all(np.diff(ha) > 0) and a.columns == b.columns
        assert all(0 <= v < 10 for v in a.columns[1][:1000])
        # checksum of the union == XOR of the parts, kv counts add (checksum.rs: order/partition independent)
        _, whole, _ = checksum(sc.WHOLE, dev)
        _, p0, _ = checksum([kvfmt.table_range(sc.TABLE, 0, n_rows // 3)], dev)
        _, p1, _ = checksum([kvfmt.table_range(sc.TABLE, n_rows // 3, n_rows)], dev)
        assert whole[0] == p0[0] ^ p1[0] and whole[1] == p0[1] + p1[1] == n_rows and whole[2] == p0[2] + p1[2]
    finally:
        for g in gens:
            ffi.lib().b2_gen_destroy(g)


@pytest.mark.parametrize("name,plan,exact,keys", sc.topn_plans(), ids=[t[0] for t in sc.topn_plans()])
def test_topn_matches_oracle(name, plan, exact, keys, regions):
    from compare import assert_topn
    for seed, n_blocks, ranges in ((1, 1, sc.WHOLE), (2, 3, sc.split_ranges())):
        host = regions[seed].build(read_ts=sc.READ_TS, n_write_blocks=n_blocks)
        exp = orc.dag_handle(plan, ranges, host)
        for region in (host, DeviceRegion(host)):
            assert_topn(DagHandler(plan, ranges, region).handle_request(), exp, exact, keys, ctx=f"{name}/seed{seed}")


def test_topn_large_generated():
    """TopN over 3e6 generated rows in 3 blocks: ORDER BY c2 DESC, c1 ASC LIMIT 1000 (BASELINE config 4 shape), every
    cell equal to the exact reference over the generator's closed form (topn_ref.py), on the whole table and on halves."""
    import topn_ref
    n_rows, n_cols, seed = 3_000_000, 4, 99
    spec = dict(n_cols=n_cols, seed=seed, lo=[0] * 4, rng=[0] * 4, nulls=[0, 10000, 0, 0])
    parts = [(i * (n_rows // 3), n_rows // 3) for i in range(3)]
    gens, blocks = [], []
    for first, n in parts:
        g, blk = _gen_block(n, n_cols, 2, seed, spec["lo"], spec["rng"], spec["nulls"], first_handle=first)
        gens.append(g); blocks.append(blk.block)
    try:
        dev = _source(blocks, ffi.LOC_DEVICE)
        columns = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(n_cols)]
        plan = Plan().table_scan(sc.TABLE, columns).topn([(col(2), True), (col(1), False)], 1000).build()
        ref = topn_ref.gen_rows(spec, parts)
        h, v, nl = ref["handle"], ref["vals"], ref["null"]
        for lo, hi in ((0, n_rows), (0, n_rows // 2), (n_rows // 2, n_rows)):
            idx = np.flatnonzero((h >= lo) & (h < hi))
            best = idx[topn_ref.topn_indices([(v[idx, 1], nl[idx, 1], True), (v[idx, 0], nl[idx, 0], False)], 1000)]
            want = [(int(h[i]),) + tuple(None if nl[i, c] else int(v[i, c]) for c in range(n_cols)) for i in best]
            got = DagHandler(plan, [kvfmt.table_range(sc.TABLE, lo, hi)], dev).handle_request()
            assert got.status == 0 and got.rows() == want, (lo, hi)
    finally:
        for g in gens:
            ffi.lib().b2_gen_destroy(g)


# ---- response encoding on the device (runner.rs:1051-1088) -----------------------------------------------------------
def _one_batch(plan, ranges, region):
    ex = BatchExecutor(plan, ranges, region, output=ffi.LOC_DEVICE)  # columns stay in HBM: only encoded bytes come back
    rc, b = ex.next_batch_raw(1 << 30)
    assert rc == ffi.B2_OK and b.is_drained != ffi.DRAIN_REMAIN
    return ex


def _elem_sizes(ex):
    return [40 if tp == ffi.TP_NEWDECIMAL else (4 if tp == ffi.TP_FLOAT else 8) for tp, _ in ex.schema()]


@pytest.mark.parametrize("name,plan", PLANS, ids=[n for n, _ in PLANS])
def test_encode_chunk_matches_oracle(name, plan, regions):
    """EncodeType::TypeChunk of the whole result: byte-identical to the oracle (as a multiset of rows for hash agg)."""
    region = regions[1].build(read_ts=sc.READ_TS, n_write_blocks=2)
    exp = orc.dag_handle(plan, sc.WHOLE, region)
    with _one_batch(plan, sc.WHOLE, region) as ex:
        got = ex.encode_batch(ffi.ENCODE_TYPE_CHUNK)
        if not sc.is_agg(name):
            assert got == exp.encoded[1]
        else:
            # group order is unspecified, and a MyDecimal cell is compared by value: its digitsInt keeps whatever
            # leading zero words the reference's order of additions left behind
            es = _elem_sizes(ex)
            norm = lambda cols: sorted(zip(*[[c if c is None or len(c) != 40 else kvfmt.decimal_struct_value(c) for c in col] for col in cols]),
                                       key=lambda t: tuple((0, 0) if x is None else (1, x) for x in t))
            a, b = norm(kvfmt.decode_chunk(got, es)), norm(kvfmt.decode_chunk(exp.encoded[1], es))
            if any(tp in (ffi.TP_DOUBLE, ffi.TP_FLOAT) for tp, _ in ex.schema()):
                continue_cmp = False  # f64 sums are order dependent; compared with tolerance by test_real_sum
            else:
                continue_cmp = True
            assert len(a) == exp.n_rows
            if continue_cmp:
                assert a == b


@pytest.mark.parametrize("name,plan", PLANS, ids=[n for n, _ in PLANS])
def test_encode_default_matches_oracle(name, plan):
    """EncodeType::TypeDefault, every plan, v2-only and mixed v1/v2 tables: the same rows after datum decode.  (Bytes can
    differ in exactly one way: a column no expression evaluated is still Raw in the reference and goes out as the stored
    v1 datum or the plan's default-value datum, e.g. VAR_INT; the device always writes the fixed-width INT/UINT/FLOAT
    datum the reference itself uses for decoded columns and for every v2 cell.  Same value, any TiDB client decodes both.)"""
    for only_fmt in (2, None):
        region = sc.dirty_region(5, n_keys=700, only_fmt=only_fmt).build(read_ts=sc.READ_TS, n_write_blocks=2)
        exp = orc.dag_handle(plan, sc.WHOLE, region)
        with _one_batch(plan, sc.WHOLE, region) as ex:
            got = ex.encode_batch(ffi.ENCODE_TYPE_DEFAULT)
            n_cols = len(ex.schema())
        a, b = kvfmt.decode_datum_rows(got, n_cols), kvfmt.decode_datum_rows(exp.encoded[0], n_cols)
        key = lambda t: tuple((0, 0) if x is None else (1, x) for x in t)
        norm = lambda rows: sorted(rows, key=key) if sc.is_agg(name) else rows
        assert len(a) == exp.n_rows
        if any(isinstance(x, float) for r in b for x in r) and sc.is_agg(name):
            continue  # f64 sums are order dependent; their values are compared (with tolerance) by test_real_sum
        assert norm(a) == norm(b), name


def test_encode_default_bytes_identical():
    """Where the reference's bytes are fully determined by the values (v2 rows, no default-filled cells; NULLs, unsigned,
    Real and the PK handle included) the TypeDefault stream is byte-identical; SUM/COUNT results (Decimal datums) too."""
    region = sc.dirty_region(9, n_keys=900, only_fmt=2).build(read_ts=sc.READ_TS, n_write_blocks=3)
    scan = lambda: Plan().table_scan(sc.TABLE, sc.COLUMNS)
    offs = [sc.C4, sc.C_H, sc.C2, sc.C3, sc.C1, sc.C6]
    for plan in (scan().build(output_offsets=offs), scan().selection(lt(col(sc.C1), const_int(0))).build(output_offsets=offs),
                 scan().aggregation([("count", const_int(1)), ("sum", col(sc.C1)), ("avg", col(sc.C3, unsigned=True)), ("sum", col(sc.C2))]).build()):
        exp = orc.dag_handle(plan, sc.split_ranges(), region)
        with _one_batch(plan, sc.split_ranges(), region) as ex:
            assert ex.encode_batch(ffi.ENCODE_TYPE_DEFAULT) == exp.encoded[0] and exp.n_rows > 0


def test_encode_empty_and_errors(regions):
    region = regions[1].build(read_ts=sc.READ_TS)
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).selection(lt(col(sc.C1), const_int(-(1 << 63)))).build()  # no row passes
    exp = orc.dag_handle(plan, sc.WHOLE, region)
    with _one_batch(plan, sc.WHOLE, region) as ex:
        assert ex.encode_batch(ffi.ENCODE_TYPE_DEFAULT) == exp.encoded[0] == b""
        assert ex.encode_batch(ffi.ENCODE_TYPE_CHUNK) == exp.encoded[1]
        with pytest.raises(Exception):
            ex.encode_batch(7)


def test_take_scanned_range_and_rows_per_range(regions):
    """BatchExecutor::take_scanned_range / collect_scanned_rows_per_range (scanner.rs:196-229) against the oracle's scan:
    consecutive takes tile the request's key space, each upper bound is the last returned row + 0x00, and the per-range
    row counts are what the MVCC scan returns range by range."""
    host = regions[2].build(read_ts=sc.READ_TS, n_write_blocks=2)
    ranges = sc.split_ranges()
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).selection(lt(col(sc.C1), const_int(0))).build()
    scans = [orc.mvcc_scan(host, kvfmt.enc_bytes_memcmp(lo), kvfmt.enc_bytes_memcmp(hi))[1] for lo, hi in ranges]
    all_rows = [kvfmt.dec_bytes_memcmp(k) for rows in scans for (k, _v) in rows]  # raw keys the scanner returns, in request order
    per_range = [len(rows) for rows in scans]
    with BatchExecutor(plan, ranges, host) as ex:
        prev_hi, seen, got_per_range = None, 0, [0] * len(ranges)
        while True:
            r = ex.next_batch(150)
            assert r.error is None
            lo, hi = ex.take_scanned_range()
            assert lo == (ranges[0][0] if prev_hi is None else prev_hi)
            seen = ex.collect_exec_stats().write_processed_keys
            for i, n in enumerate(ex.collect_scanned_rows_per_range()):
                got_per_range[i] += n
            if r.is_drained:
                assert hi == ranges[-1][1]
                break
            assert hi == (all_rows[seen - 1] + b"\x00" if seen and hi != lo else lo)
            prev_hi = hi
        assert seen == len(all_rows) and got_per_range == per_range and sum(per_range) > 300


@pytest.mark.parametrize("fmt", [2, 1])
@pytest.mark.parametrize("name,plan", sc.int_plans(), ids=[n for n, _ in sc.int_plans()])
def test_exact_layout_fast_path(name, plan, fmt):
    """All-integer table through the C ABI: SWAR width probe, conditions and outputs by stored position (every width mix,
    signed/unsigned), rows with NULL / missing columns on the general path of the same tiles."""
    region = sc.int_region(3, n_keys=3000, fmt=fmt).build(read_ts=sc.READ_TS, n_write_blocks=2)
    exp = orc.dag_handle(plan, sc.WHOLE, region)
    got = DagHandler(plan, sc.WHOLE, DeviceRegion(region)).handle_request()
    if name == "topn":
        from compare import assert_topn
        assert_topn(got, exp, True, None, ctx=name)
    else:
        assert_same_rows(got, exp, ordered=name != "agg", ctx=name)
    bad = sc.int_region(4, n_keys=3000, corrupt=True, fmt=fmt).build(read_ts=sc.READ_TS)
    exp = orc.dag_handle(plan, sc.WHOLE, bad)
    got = DagHandler(plan, sc.WHOLE, bad).handle_request()
    assert exp.status != 0 and got.status == exp.status
    if name not in ("agg", "topn"):
        assert_same_rows(got, exp, ordered=True, ctx=name + "/corrupt")


def test_plan_specialised_kernels_match_oracle(regions):
    """The run-time compiled, plan-specialised kernels (jit.cu) against the oracle: scan, selection, simple / hash
    aggregation and TopN, on the dirty region (every MVCC shape, v1 + v2 rows) and on the all-integer table."""
    from tikv_b200.executor import BatchExecutor as BE
    L = ffi.lib()
    cases = [(n, p, regions[1].build(read_ts=sc.READ_TS, n_write_blocks=2), sc.split_ranges()) for n, p in PLANS if n in
             ("scan_all", "sel_lt_const", "count_star", "group_by_small", "group_filter_offsets")]
    ir = sc.int_region(3, n_keys=3000).build(read_ts=sc.READ_TS, n_write_blocks=2)
    cases += [(n, p, ir, sc.WHOLE) for n, p in sc.int_plans() if n in ("const_on_left", "eq_ne", "agg", "topn")]
    assert len(cases) >= 7
    for name, plan, region, ranges in cases:
        rc = L.b2_plan_prepare(C.byref(plan.c), 0)
        assert rc == ffi.B2_OK, L.b2_last_error_message()
        exp = orc.dag_handle(plan, ranges, region)
        with BE(plan, ranges, region, jit=ffi.JIT_SYNC) as ex:
            cols, kinds, is_drained = None, None, False
            parts = []
            while not is_drained:
                r = ex.next_batch(700)
                assert r.error is None
                parts.append(r)
                is_drained = r.is_drained
            st = ex.collect_exec_stats()
            assert st.jit_launches > 0 and st.jit_launches <= st.kernel_launches
        got_rows = [row for r in parts for row in r.rows()]
        if name == "topn":
            assert got_rows == exp.rows(), name
        elif sc.is_agg(name) or name == "agg":
            key = lambda t: tuple((0, 0) if x is None else (1, x) for x in t)
            assert sorted(got_rows, key=key) == sorted(exp.rows(), key=key), name
        else:
            assert got_rows == exp.rows(), name


@pytest.mark.parametrize("name,plan", sc.limit_plans(), ids=[n for n, _ in sc.limit_plans()])
@pytest.mark.parametrize("batch", [64, 1 << 22])
def test_limit(name, plan, batch, regions):
    """BatchLimitExecutor on top of scan / selection (limit_executor.rs): the first n rows in key order, then drained."""
    region = regions[1].build(read_ts=sc.READ_TS, n_write_blocks=2)
    exp = orc.dag_handle(plan, sc.split_ranges(), region)
    got = DagHandler(plan, sc.split_ranges(), region, batch_rows=batch).handle_request()
    assert_same_rows(got, exp, ordered=True, ctx=name)


@pytest.mark.parametrize("name,plan", sc.minmax_plans(), ids=[n for n, _ in sc.minmax_plans()])
def test_min_max(name, plan, regions):
    """MAX / MIN (impl_max_min.rs): signed / unsigned / Real arguments, NULL inputs, GROUP BY, empty input."""
    for seed in (1, 2):
        region = regions[seed].build(read_ts=sc.READ_TS, n_write_blocks=2)
        exp = orc.dag_handle(plan, sc.split_ranges(), region)
        got = DagHandler(plan, sc.split_ranges(), DeviceRegion(region)).handle_request()
        assert exp.status == 0
        assert_same_rows(got, exp, ordered=False, ctx=f"{name}/seed{seed}")


@pytest.mark.parametrize("jit", [ffi.JIT_OFF, ffi.JIT_SYNC], ids=["aot", "jit"])
@pytest.mark.parametrize("name,plan", sc.multi_group_plans(), ids=[n for n, _ in sc.multi_group_plans()])
def test_multi_column_group_by(name, plan, jit, regions):
    """BatchSlowHashAggregation (slow_hash_aggr_executor.rs): composite keys of 2..4 Int / Real expressions."""
    for seed in ((1, 2) if jit == ffi.JIT_OFF else (2,)):
        region = regions[seed].build(read_ts=sc.READ_TS, n_write_blocks=2)
        exp = orc.dag_handle(plan, sc.split_ranges(), region)
        got = DagHandler(plan, sc.split_ranges(), DeviceRegion(region), jit=jit).handle_request()
        assert exp.status == 0 and (exp.n_rows > 0 or name == "mg_no_input")
        # f64 SUM: the addition order differs from the oracle's (atomics), tolerance 1e-12 relative; everything else bit-exact
        assert_same_rows(got, exp, ordered=False, float_rel_tol=1e-12 if name == "mg_same_expr_twice" else None, ctx=f"{name}/seed{seed}")


def test_multi_column_group_by_generated():
    """Generated table, 200k rows: (a) parity with the oracle for two- and three-column keys incl. a nullable column,
    (b) at 4M rows the group counts add up and the number of groups is the product of the key cardinalities."""
    n_cols = 8
    lo = [0, 0, -(1 << 40), 0, 0, 0, 0, 0]
    rng = [0, 37, 1 << 41, 0, 5, 0, 3, 0]
    nulls = [0, 0, 0, 10000, 200000, 0, 0, 0]
    columns = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(n_cols)]
    scan = lambda: Plan().table_scan(sc.TABLE, columns)
    plans = [("g2", scan().aggregation([("count", const_int(1)), ("sum", col(3))], group_by=[col(2), col(7)]).build()),
             ("g3null", scan().aggregation([("sum", col(1)), ("max", col(3))], group_by=[col(7), col(5), col(2)]).build())]
    g, blk = _gen_block(200_000, n_cols, 2, 99, lo, rng, nulls, extra=20000, delete=20000, lockrec=20000)
    try:
        hb, keep = _block_to_host(blk)
        host, dev = _source([hb], ffi.LOC_HOST), _source([blk.block], ffi.LOC_DEVICE)
        for name, plan in plans:
            e = orc.dag_handle(plan, sc.WHOLE, host)
            assert e.status == 0 and e.n_rows in (37 * 3, 37 * 3 * 6)
            assert_same_rows(DagHandler(plan, sc.WHOLE, dev).handle_request(), e, ordered=False, ctx=f"gen/{name}")
    finally:
        ffi.lib().b2_gen_destroy(g)
    n_rows = 4_000_000
    g, blk = _gen_block(n_rows, n_cols, 2, 5, lo, rng, nulls)
    try:
        dev = _source([blk.block], ffi.LOC_DEVICE)
        r = DagHandler(plans[1][1], sc.WHOLE, dev).handle_request()
        assert r.n_rows == 37 * 3 * 6
        cnt = DagHandler(scan().aggregation([("count", const_int(1))], group_by=[col(2), col(7)]).build(), sc.WHOLE, dev).handle_request()
        assert cnt.n_rows == 37 * 3 and sum(x[0] for x in cnt.rows()) == n_rows
        one = DagHandler(scan().aggregation([("count", const_int(1))], group_by=[col(0), col(7)]).build(), [kvfmt.table_range(sc.TABLE, 0, 500_000)], dev).handle_request()
        assert one.n_rows == 500_000 and all(x[0] == 1 for x in one.rows())  # one group per row
    finally:
        ffi.lib().b2_gen_destroy(g)


@pytest.mark.parametrize("name,plan", sc.scalar_plans(), ids=[n for n, _ in sc.scalar_plans()])
def test_scalar_functions(name, plan, regions):
    """DIV / MOD / unary minus / ABS / IFNULL / IF / CASE WHEN / COALESCE (impl_arithmetic.rs, impl_op.rs, impl_math.rs,
    impl_control.rs, impl_compare.rs) in projections, selections, aggregate arguments and group keys.  Plans with these
    functions always run on their plan-specialised kernel, also when the caller asked for JIT_OFF."""
    jit = ffi.JIT_OFF
    for seed in (2,):  # one region: every plan costs one run-time compilation (10-20 s for a wide projection)
        region = regions[seed].build(read_ts=sc.READ_TS, n_write_blocks=2)
        exp = orc.dag_handle(plan, sc.split_ranges(), region)
        got = DagHandler(plan, sc.split_ranges(), DeviceRegion(region), jit=jit).handle_request()
        if "_err_" in name:
            assert exp.status == ffi.B2_ERR_EVALUATE == got.status and exp.mysql_code == 1690 == got.mysql_code and got.message == exp.message
            assert got.rows()[:len(exp.rows())] == exp.rows()
            continue
        assert exp.status == 0 and exp.n_rows > 0
        assert_same_rows(got, exp, ordered="agg" not in name, ctx=f"{name}/seed{seed}")


def test_scalar_function_known_answers():
    """The reference's own unit-test vectors for these functions, through the CUDA path (the error vectors: one per kind
    here, all of them against the emulated device logic in test_device_logic_cpu.py — each is a kernel compilation)."""
    sc.check_scalar_known_answers(lambda plan, ranges, region: DagHandler(plan, ranges, DeviceRegion(region)).handle_request(),
                                  error_labels=("int_divide(-9223372036854775808,-1)", "neg_uint(9223372036854775809)", "abs(-9223372036854775808)"))


def test_units_of_a_single_entry():
    """A CF_WRITE block (and so a unit) holding one entry: every lane past the end of its only tile is clamped onto that
    entry.  The lean kernels once looked one entry back from it (index -1 into the staged offsets): an illegal address about
    one run in three (round 2: dirty_region(3, 2000 keys) splits into 3034 + 3034 + 1 entries)."""
    r = kvfmt.Region()
    for h in range(601):
        r.put(kvfmt.row_key(sc.TABLE, h), kvfmt.row_v2([(1, h * 7 - 300, "int"), (2, h % 5, "int"), (3, h, "uint"), (4, 0.5 * h, "f64"), (6, h % 9, "int")]), 10, 20)
    host = r.build(read_ts=sc.READ_TS, n_write_blocks=2)
    assert [b.n for b in host.wblocks] == [300, 300, 1]
    plans = [(n, p) for n, p in PLANS if n in ("count_star", "group_by_small", "agg_after_filter", "sel_lt_const")] + [(t[0], t[1]) for t in sc.topn_plans()[:2]]
    for region in (DeviceRegion(host), host, DeviceRegion(sc.dirty_region(3, n_keys=2000).build(read_ts=sc.READ_TS, n_write_blocks=2))):
        ref = region._host if isinstance(region, DeviceRegion) else region
        for _ in range(3):
            for name, plan in plans:
                assert_same_rows(DagHandler(plan, sc.WHOLE, region).handle_request(), orc.dag_handle(plan, sc.WHOLE, ref), ordered=not sc.is_agg(name), ctx=name)
            assert checksum(sc.WHOLE, region)[:2] == orc.checksum(sc.WHOLE, ref)[:2]


def test_like_known_answers():
    """impl_like.rs test_like / test_like_wide_character through the CUDA path (plan-specialised kernels, patterns in HBM)."""
    sc.check_like_known_answers(lambda plan, ranges, region: DagHandler(plan, ranges, DeviceRegion(region)).handle_request())


@pytest.mark.parametrize("name,plan", sc.in_plans(), ids=[n for n, _ in sc.in_plans()])
def test_in_lists(name, plan, regions):
    """IN (impl_compare_in.rs): NULL semantics, mixed signedness, Real, columns inside the list."""
    region = regions[2].build(read_ts=sc.READ_TS, n_write_blocks=2)
    exp = orc.dag_handle(plan, sc.split_ranges(), region)
    got = DagHandler(plan, sc.split_ranges(), DeviceRegion(region)).handle_request()
    assert exp.status == 0 and exp.n_rows > 0
    assert_same_rows(got, exp, ordered="group" not in name, ctx=name)


@pytest.mark.parametrize("name,plan", sc.projection_plans(), ids=[n for n, _ in sc.projection_plans()])
def test_projection(name, plan):
    """BatchProjectionExecutor (projection_executor.rs) on top of scan / selection, optionally under a Limit."""
    region = sc.dirty_region(1, n_keys=900, full_range=name == "proj_overflow").build(read_ts=sc.READ_TS, n_write_blocks=2)
    exp = orc.dag_handle(plan, sc.split_ranges(), region)
    got = DagHandler(plan, sc.split_ranges(), DeviceRegion(region)).handle_request()
    if name == "proj_real_chain":  # also through the plan-specialised kernel, where the evaluator is unrolled
        assert_same_rows(DagHandler(plan, sc.split_ranges(), DeviceRegion(region), jit=ffi.JIT_SYNC).handle_request(), exp, ordered=True, ctx=name + "/jit")
    if name == "proj_overflow":
        # an evaluation error ends the request; the reference drops the rows of the batch it happened in (projection_executor.rs
        # :207-211, batch = 32..1024 rows), the device keeps every row before the failing one: the oracle's rows are a prefix
        assert exp.status == ffi.B2_ERR_EVALUATE == got.status and exp.mysql_code == 1690 == got.mysql_code
        assert got.rows()[:len(exp.rows())] == exp.rows()
        return
    assert exp.status == 0
    assert_same_rows(got, exp, ordered=True, ctx=name)


_FIXTURES = sc.reference_executor_fixtures()


@pytest.mark.parametrize("fx", _FIXTURES, ids=[f[0] for f in _FIXTURES])
def test_reference_executor_fixtures(fx):
    """The reference's own aggregation / TopN test expectations (fast_hash_aggr_executor.rs:509-634, top_n_executor.rs:
    528-757, 1105-1212) through the CUDA path: generic and plan-specialised kernels, host- and device-resident sources."""
    jits = (ffi.JIT_OFF, ffi.JIT_SYNC) if fx[0] in ("hash_agg_fast_v2", "topn_integration_3", "topn_unsigned_col0_desc") else (ffi.JIT_OFF,)  # (a compile each)
    for jit in jits:
        sc.check_reference_fixture(fx, lambda plan, region: DagHandler(plan, sc.WHOLE, region, jit=jit).handle_request())
    sc.check_reference_fixture(fx, lambda plan, region: DagHandler(plan, sc.WHOLE, DeviceRegion(region)).handle_request())


# ---- backward scan (TableScan.desc; scan_executor.rs:89-101, backward.rs:78-225) ------------------------------------------
def test_desc_table_scan_matches_oracle(regions):
    """SURVEY §8 f3: the device path of `desc` scans (reversed chunks, rows reversed on the device) against the oracle's
    BackwardScanner pipeline: plain scan, selection, projection-free subsets, Limit, small batches, every isolation level,
    host- and device-resident sources, multi-range requests."""
    from tikv_b200.plan import gt
    scan = lambda: Plan().table_scan(sc.TABLE, sc.COLUMNS, desc=True)
    plans = [("all", scan().build()), ("sel", scan().selection(gt(col(sc.C6, tp=ffi.TP_LONG), const_int(3))).build(output_offsets=[sc.C_H, sc.C1, sc.C6])),
             ("limit", scan().selection(lt(col(sc.C1), const_int(0))).limit(41).build()), ("limit_plain", scan().limit(7).build())]
    for seed in (1, 2):
        host = regions[seed].build(read_ts=sc.READ_TS, n_write_blocks=3)
        for region in (host, DeviceRegion(host)):
            for ranges in (sc.WHOLE, sc.split_ranges()):
                for name, plan in plans:
                    exp = orc.dag_handle(plan, ranges, host)
                    for batch in (1 << 22, 97):
                        got = DagHandler(plan, ranges, region, batch_rows=batch).handle_request()
                        assert_same_rows(got, exp, ordered=True, ctx=f"desc/{name}/seed{seed}/batch{batch}")
                    if name == "all":
                        assert got.stats.write_processed_keys == exp.stats["processed_keys"] and got.stats.processed_size == exp.stats["processed_size"]
    for ts, iso in ((25, ffi.ISO_RC), (sc.READ_TS, ffi.ISO_RC_CHECK_TS)):
        region = regions[2].build(read_ts=ts, isolation=iso)
        exp, got = orc.dag_handle(plans[0][1], sc.WHOLE, region), DagHandler(plans[0][1], sc.WHOLE, region, batch_rows=200).handle_request()
        assert got.status == exp.status and got.rows() == exp.rows()


def test_desc_aggregation_topn_errors_and_locks(regions):
    """Direction-independent pipelines under `desc` (aggregates; TopN, whose ties go to the row scanned first = the larger
    key), the first error of a backward scan (the failing row with the largest key; the rows above it are still returned)
    and a conflicting lock (rows above the lock first, then KeyIsLocked)."""
    host = regions[1].build(read_ts=sc.READ_TS, n_write_blocks=2)
    scan = lambda: Plan().table_scan(sc.TABLE, sc.COLUMNS, desc=True)
    agg = scan().aggregation([("sum", col(sc.C1)), ("count", const_int(1))], group_by=[col(sc.C6, tp=ffi.TP_LONG)]).build()
    assert_same_rows(DagHandler(agg, sc.WHOLE, host).handle_request(), orc.dag_handle(agg, sc.WHOLE, host), ordered=False, ctx="desc agg")
    topn = scan().topn([(col(sc.C6), True)], 60).build()  # heavy ties on C6: only the scan order decides which rows stay
    exp, got = orc.dag_handle(topn, sc.WHOLE, host), DagHandler(topn, sc.WHOLE, host).handle_request()
    assert got.status == 0 == exp.status and [r[sc.C6] for r in got.rows()] == [r[sc.C6] for r in exp.rows()]
    # two corrupted rows: a backward scan reports the one with the larger key and returns the rows above it
    T = sc.TABLE
    r = kvfmt.Region()
    for h in range(500):
        r.put(kvfmt.row_key(T, h), kvfmt.row_v2([(1, h, "int"), (2, h % 5, "int"), (3, 7, "uint"), (4, 1.0, "f64"), (6, 1, "int")]), 10, 20)
    r.raw_write(kvfmt.row_key(T, 100), 50, b"Xjunk").raw_write(kvfmt.row_key(T, 400), 50, b"Xjunk")
    bad = r.build(read_ts=100)
    plan = scan().build()
    exp, got = orc.dag_handle(plan, sc.WHOLE, bad), DagHandler(plan, sc.WHOLE, bad, batch_rows=64).handle_request()
    assert exp.status == ffi.B2_ERR_STORAGE == got.status and got.rows() == exp.rows() and len(got.rows()) == 99
    # a Put lock in the middle: the rows with larger keys come out, then the request fails
    lk = kvfmt.Region()
    lk.write = [w for w in r.write if b"Xjunk" not in w[1]]
    lk.add_lock(kvfmt.row_key(T, 250), kvfmt.lock_record(b"P", kvfmt.row_key(T, 250), 60))
    locked = lk.build(read_ts=100)
    exp, got = orc.dag_handle(plan, sc.WHOLE, locked), DagHandler(plan, sc.WHOLE, locked, batch_rows=64).handle_request()
    assert exp.status == ffi.B2_ERR_KEY_IS_LOCKED == got.status and got.rows() == exp.rows() and len(got.rows()) == 249


@pytest.mark.parametrize("batch", [64, 1 << 22])
@pytest.mark.parametrize("desc", [False, True], ids=["forward", "backward"])
def test_scan_error_statistics_match_rows(desc, batch):
    """A failing row in the middle of a plain scan: the rows the scan meets before it come out, then the error, and the
    statistics describe exactly those rows (rows per range, processed keys) in both directions, also when the batch
    that meets the failing row has to be redone."""
    T = sc.TABLE
    r = kvfmt.Region()
    for h in range(500):
        r.put(kvfmt.row_key(T, h), kvfmt.row_v2([(1, h, "int"), (2, h % 5, "int"), (3, 7, "uint"), (4, 1.0, "f64"), (6, 1, "int")]), 10, 20)
    r.raw_write(kvfmt.row_key(T, 100), 50, b"Xjunk").raw_write(kvfmt.row_key(T, 400), 50, b"Xjunk")
    host = r.build(read_ts=100, n_write_blocks=2)
    ranges = [kvfmt.table_range(T, 0, 300), kvfmt.table_range(T, 300, 500)]
    plan = Plan().table_scan(T, sc.COLUMNS, desc=desc).build()
    exp = orc.dag_handle(plan, ranges, host)
    assert exp.status == ffi.B2_ERR_STORAGE and exp.n_rows == (99 if desc else 100)
    for region in (host, DeviceRegion(host)):
        with BatchExecutor(plan, ranges, region) as ex:
            rows, per_range = [], [0] * len(ranges)
            while True:
                b = ex.next_batch(batch)
                rows += b.rows()
                for i, n in enumerate(ex.collect_scanned_rows_per_range()):
                    per_range[i] += n
                if b.error is not None or b.is_drained:
                    break
            assert b.error is not None and b.error.status == exp.status
            assert rows == exp.rows()
            assert sum(per_range) == ex.collect_exec_stats().write_processed_keys == len(rows)


def test_desc_take_scanned_range(regions):
    """scanner.rs:204-229 with scan_backward_in_range: consecutive takes tile the key space from the top: each lower bound
    is the key of the last (smallest) row returned, the next take's upper bound; the last take reaches the first range's start."""
    host = regions[2].build(read_ts=sc.READ_TS, n_write_blocks=2)
    ranges = sc.split_ranges()
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS, desc=True).build()
    scans = [orc.mvcc_scan(host, kvfmt.enc_bytes_memcmp(lo), kvfmt.enc_bytes_memcmp(hi))[1] for lo, hi in ranges]
    all_rows = [kvfmt.dec_bytes_memcmp(k) for rows in scans for (k, _v) in rows][::-1]  # raw keys in the order a backward scan returns them
    with BatchExecutor(plan, ranges, host) as ex:
        prev_lo, seen = None, 0
        while True:
            r = ex.next_batch(150)
            assert r.error is None
            lo, hi = ex.take_scanned_range()
            assert hi == (ranges[-1][1] if prev_lo is None else prev_lo)
            seen = ex.collect_exec_stats().write_processed_keys
            if r.is_drained:
                assert lo == ranges[0][0]
                break
            assert lo == (all_rows[seen - 1] if seen and lo != hi else hi)
            prev_lo = lo
        assert seen == len(all_rows) > 300


# ---- ABI v2: deadline, async batches, warnings, paging, HBM block cache -----------------------------------------------
def test_deadline_exceeded(regions):
    """runner.rs:974 `self.deadline.check()?`: a request whose deadline has passed answers B2_ERR_DEADLINE (before any launch)."""
    import time
    host = regions[1].build(read_ts=sc.READ_TS)
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).build()
    with BatchExecutor(plan, sc.WHOLE, host, deadline_ns=time.monotonic_ns() - 1) as ex:
        r = ex.next_batch(1 << 20)
        assert r.error is not None and r.error.status == ffi.B2_ERR_DEADLINE and r.n_rows == 0 and r.is_drained
    with BatchExecutor(plan, sc.WHOLE, host, deadline_ns=time.monotonic_ns() + 60 * 10 ** 9) as ex:
        assert ex.next_batch(1 << 20).error is None


def test_async_next_batch_equals_sync(regions):
    """b2_exec_next_batch_async + b2_exec_poll (the reference's `async fn next_batch`): same batches as the blocking call."""
    import time
    host = regions[2].build(read_ts=sc.READ_TS, n_write_blocks=2)
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).selection(lt(col(sc.C1), const_int(0))).build()
    exp = DagHandler(plan, sc.WHOLE, host, batch_rows=300).handle_request()
    rows = []
    with BatchExecutor(plan, sc.WHOLE, host) as ex:
        while True:
            ex.next_batch_async(300)
            polls = 0
            while True:
                r = ex.poll()
                if r is not None:
                    break
                polls += 1
                time.sleep(0.0005)
            assert r.error is None
            rows += r.rows()
            if r.is_drained:
                break
    assert rows == exp.rows() and len(rows) > 100


def test_division_by_zero_warnings(regions):
    """DivideReal (impl_arithmetic.rs:515-533): x / 0 is NULL and raises warning 1365 "Division by 0" per evaluated row
    (expr/ctx.rs:267-286); the count equals the oracle's SelectResponse.warning_count, at most 64 details are kept."""
    from tikv_b200.plan import divide, multiply as mul, const_real
    host = regions[1].build(read_ts=sc.READ_TS)
    c4 = col(sc.C4, tp=ffi.TP_DOUBLE)
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).projection(col(sc.C_H), divide(c4, mul(c4, const_real(0.0))), divide(const_real(1.0), c4)).build()
    exp = orc.dag_handle(plan, sc.WHOLE, host)
    assert exp.status == 0 and exp.warning_count > 100
    for region in (host, DeviceRegion(host)):
        with BatchExecutor(plan, sc.WHOLE, region) as ex:
            rows, per_batch = [], 0
            while True:
                rc, b = ex.next_batch_raw(257)
                assert rc == 0
                per_batch += b.n_warnings
                r = ex._L  # noqa: F841
                from tikv_b200.executor import _read_batch
                cols, _, _ = _read_batch(b, ffi.LOC_HOST)
                rows += list(zip(*cols)) if cols else []
                if b.is_drained != ffi.DRAIN_REMAIN:
                    break
            total, details = ex.warnings()
        assert rows == exp.rows()
        assert total == exp.warning_count == per_batch and len(details) == 64 and details[0] == (1365, "Division by 0")


def test_region_block_cache(regions):
    """b2_region_pin: the CF blocks of a host-resident region are copied to HBM once (keyed by region id + data version);
    requests over the returned device source see the same data; a second pin is a cache hit; unpin releases the copy."""
    host = regions[1].build(read_ts=sc.READ_TS, n_write_blocks=3)
    L = ffi.lib()
    dev_src = ffi.RegionSource()
    h0, m0, b0 = C.c_uint64(), C.c_uint64(), C.c_uint64()
    L.b2_region_cache_stats(0, C.byref(b0), C.byref(h0), C.byref(m0))
    assert L.b2_region_pin(0, 4242, 7, C.byref(host.c), C.byref(dev_src)) == 0, L.b2_last_error_message()
    again = ffi.RegionSource()
    assert L.b2_region_pin(0, 4242, 7, C.byref(host.c), C.byref(again)) == 0
    b1, h1, m1 = C.c_uint64(), C.c_uint64(), C.c_uint64()
    L.b2_region_cache_stats(0, C.byref(b1), C.byref(h1), C.byref(m1))
    assert m1.value == m0.value + 1 and h1.value == h0.value + 1 and b1.value > b0.value
    assert dev_src.location == ffi.LOC_DEVICE and dev_src.n_write == 3 and again.write[0].keys == dev_src.write[0].keys

    class Pinned:  # a region object as the executors expect it
        c = dev_src
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).aggregation([("sum", col(sc.C1)), ("count", const_int(1))], group_by=[col(sc.C6, tp=ffi.TP_LONG)]).build()
    assert_same_rows(DagHandler(plan, sc.WHOLE, Pinned).handle_request(), orc.dag_handle(plan, sc.WHOLE, host), ordered=False, ctx="pinned agg")
    scan = Plan().table_scan(sc.TABLE, sc.COLUMNS).build()
    assert_same_rows(DagHandler(scan, sc.split_ranges(), Pinned).handle_request(), orc.dag_handle(scan, sc.split_ranges(), host), ctx="pinned scan")
    assert L.b2_region_unpin(0, 4242, 7) == 0 and L.b2_region_unpin(0, 4242, 7) == 0
    assert L.b2_region_unpin(0, 4242, 7) == ffi.B2_ERR_INVALID_ARG
    L.b2_region_cache_stats(0, C.byref(b1), C.byref(h1), C.byref(m1))
    assert b1.value == b0.value


def test_paging_request(regions):
    """b2_dag_handle with paging_size (runner.rs:790-806): a page of rows in key order, B2_DRAIN_PAGING, and the scanned
    range to resume from; resuming at its upper bound until drained yields the whole result exactly once."""
    from tikv_b200.executor import _read_batch
    from tikv_b200.plan import key_ranges
    host = regions[2].build(read_ts=sc.READ_TS, n_write_blocks=2)
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS).selection(lt(col(sc.C1), const_int(0))).build()
    exp = orc.dag_handle(plan, sc.WHOLE, host).rows()
    L = ffi.lib()
    rows, start, pages = [], sc.WHOLE[0][0], 0
    while True:
        kr, keep = key_ranges([(start, sc.WHOLE[0][1])])
        cfg = ffi.ExecConfig()
        cfg.output_location, cfg.paging_size = ffi.LOC_HOST, 100
        b, h = ffi.Batch(), C.c_void_p()
        rc = L.b2_dag_handle(C.byref(plan.c), kr, 1, C.byref(host.c), C.byref(cfg), C.byref(b), C.byref(h))
        assert rc == 0, L.b2_last_error_message()
        cols, _, _ = _read_batch(b, ffi.LOC_HOST)
        rows += list(zip(*cols)) if cols else []
        pages += 1
        lo, hi, ln, hn = C.c_void_p(), C.c_void_p(), C.c_uint32(), C.c_uint32()
        assert L.b2_exec_take_scanned_range(h, C.byref(lo), C.byref(ln), C.byref(hi), C.byref(hn)) == 0
        upper = C.string_at(hi, hn.value)
        drained = b.is_drained
        L.b2_exec_close(h)
        if drained != ffi.DRAIN_PAGING:
            assert drained == ffi.DRAIN_DRAINED
            break
        assert upper > start
        start = upper
    assert rows == exp and pages > 2
    agg = Plan().table_scan(sc.TABLE, sc.COLUMNS).aggregation([("count", const_int(1))]).build()
    kr, keep = key_ranges(sc.WHOLE)
    cfg = ffi.ExecConfig()
    cfg.paging_size = 10
    b, h = ffi.Batch(), C.c_void_p()
    assert L.b2_dag_handle(C.byref(agg.c), kr, 1, C.byref(host.c), C.byref(cfg), C.byref(b), C.byref(h)) == ffi.B2_ERR_UNSUPPORTED


def test_index_scan_matches_oracle():
    """SURVEY §8 f3: BatchIndexScan on the device (index_row_split: key datums -> columns, handle from the key tail or the
    value), forward and backward, with selection / aggregation / TopN on top, against the oracle (itself pinned on
    index_scan_executor.rs test_basic, tests/test_oracle_golden.py)."""
    import random
    rng = random.Random(5)
    T, IDX = 11, 4
    r = kvfmt.Region()
    for h in range(2000):
        a = None if rng.random() < 0.1 else rng.choice([rng.randrange(-(1 << 63), 1 << 63), rng.randrange(-5, 5)])
        b = rng.choice([0, 1, (1 << 64) - 1, rng.randrange(0, 1 << 64)])
        payload = (kvfmt.datum_null() if a is None else kvfmt.datum_int(a, comparable=True)) + kvfmt.datum_uint(b, comparable=True) + kvfmt.datum_int(h, comparable=True)
        key = kvfmt.index_key(T, IDX, payload)
        r.put(key, b"0", 3, 4)
        if rng.random() < 0.2:
            r.put(key, b"0", 50, 60)
        if rng.random() < 0.1:
            r.delete(key, 5, 6)
    host = r.build(read_ts=10, n_write_blocks=2)
    cols = [ColumnDef(1), ColumnDef(2, unsigned=True), ColumnDef(3, pk_handle=True), ColumnDef(-3)]
    whole = [(kvfmt.index_key(T, IDX), kvfmt.index_key(T, IDX, b"\xfa"))]
    scan = lambda desc=False: Plan().index_scan(T, cols, desc=desc)
    plans = [("asc", scan().build(), True), ("desc", scan(True).build(), True), ("sel", scan().selection(lt(col(0), const_int(3))).build(output_offsets=[2, 0]), True),
             ("agg", scan().aggregation([("count", const_int(1)), ("sum", col(0))], group_by=[col(1, unsigned=True)]).build(), False),
             ("topn", scan().topn([(col(0), True), (col(2), False)], 25).build(), True)]
    for region in (host, DeviceRegion(host)):
        for name, plan, ordered in plans:
            exp = orc.dag_handle(plan, whole, host)
            got = DagHandler(plan, whole, region, batch_rows=300).handle_request()
            assert exp.status == 0 and exp.n_rows > 5
            assert_same_rows(got, exp, ordered=ordered, ctx=f"index {name}")
    # unique index (handle in the value) and the error shapes
    T2, IDX2 = 7, 2
    u = kvfmt.Region()
    for a, h in ((1, 100), (2, -3), (9, 1 << 40)):
        u.put(kvfmt.index_key(T2, IDX2, kvfmt.datum_int(a, comparable=True)), (h & ((1 << 64) - 1)).to_bytes(8, "big"), 1, 2)
    w2 = [(kvfmt.index_key(T2, IDX2), kvfmt.index_key(T2, IDX2, b"\xfa"))]
    c2 = [ColumnDef(1), ColumnDef(2, pk_handle=True)]
    assert DagHandler(Plan().index_scan(T2, c2).build(), w2, u.build(read_ts=10)).handle_request().rows() == [(1, 100), (2, -3), (9, 1 << 40)]
    missing = DagHandler(Plan().index_scan(T2, [ColumnDef(1), ColumnDef(5), ColumnDef(2, pk_handle=True)]).build(), w2, u.build(read_ts=10)).handle_request()
    assert missing.status == ffi.B2_ERR_CORRUPTED
    rec = kvfmt.Region()
    rec.put(kvfmt.row_key(T2, 1), kvfmt.row_v2([(1, 5, "int")]), 1, 2)
    assert DagHandler(Plan().index_scan(T2, c2).build(), [kvfmt.table_range(T2)], rec.build(read_ts=10)).handle_request().status == ffi.B2_ERR_CORRUPTED


# ---- bytes / time / duration / decimal / json output columns (VERDICT r1 item 8) ---------------------------------------------
def test_reference_mixed_row_on_the_device():
    """The reference's own 12-column v2 row (encoder_for_test.rs:560-588) through the CUDA path: the values that test
    encoded, and a TypeChunk block byte-identical to the oracle's."""
    host = sc.ref_mixed_region().build(read_ts=sc.READ_TS)
    plan = Plan().table_scan(sc.TABLE, sc.REF_MIXED_COLUMNS).build()
    for region in (host, DeviceRegion(host)):
        got = DagHandler(plan, sc.WHOLE, region).handle_request()
        assert got.status == 0, got.message
        assert got.rows() == [sc.REF_MIXED_VALUES]
    with BatchExecutor(plan, sc.WHOLE, host) as ex:
        r = ex.next_batch(1 << 20)
        assert r.error is None and r.n_rows == 1
        assert ex.encode_batch(ffi.ENCODE_TYPE_CHUNK) == orc.dag_handle(plan, sc.WHOLE, host).encoded[1]


@pytest.mark.parametrize("seed", [1, 2])
def test_mixed_tables_match_oracle(seed):
    """Scans of a table with VARCHAR / BLOB / DATETIME / DATE / DECIMAL / DURATION / JSON columns (rows in both formats,
    NULLs, empty and 700-byte strings, values in CF_DEFAULT): every cell equals the oracle's, host- and device-resident
    sources, small batches and one big one; the TypeChunk encoding of the whole result is byte-identical."""
    sc.check_mixed(lambda plan, ranges, region: DagHandler(plan, ranges, region).handle_request(), seed=seed)
    sc.check_mixed(lambda plan, ranges, region: DagHandler(plan, ranges, DeviceRegion(region), batch_rows=97).handle_request(), seed=seed)
    host = sc.mixed_region(seed).build(read_ts=sc.READ_TS, n_write_blocks=2)
    for name, plan in sc.mixed_plans():
        if "limit" in name:
            continue
        with BatchExecutor(plan, sc.WHOLE, DeviceRegion(host)) as ex:
            r = ex.next_batch(1 << 22)
            assert r.error is None and r.is_drained
            assert ex.encode_batch(ffi.ENCODE_TYPE_CHUNK) == orc.dag_handle(plan, sc.WHOLE, host).encoded[1], name
