"""`-m gpu`: the device group tables at the places they go wrong: hash-tag collisions of the composite-key table, lanes of
one warp inserting the same new key, composite keys that differ only in their NULL mask or signedness, the slot
boundaries of the lean kernel's direct-addressed table, the general kernel's CTA table at its load limit, the empty-key
sentinel, and growth of the HBM table past its first capacity.  Every case is checked against the oracle, or against
closed-form sums where the table is too large for it."""
import pytest

import kvfmt
import orc
import scenarios as sc
from compare import assert_same_rows
from test_gpu_parity import _gen_block, _source
from tikv_b200 import ffi
from tikv_b200.executor import DagHandler, DeviceRegion
from tikv_b200.plan import ColumnDef, Plan, col, const_int

pytestmark = pytest.mark.gpu

U64 = (1 << 64) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
JITS = [ffi.JIT_OFF, ffi.JIT_SYNC]
JIT_IDS = ["aot", "jit"]

# schema of the hand-built regions: handle, a i64, b i64, u u64, r f64, v i64
COLS = [ColumnDef(100, pk_handle=True), ColumnDef(1), ColumnDef(2), ColumnDef(3, unsigned=True), ColumnDef(4, tp=ffi.TP_DOUBLE), ColumnDef(5)]
H, A, B, U, R, V = range(6)


def _scan():
    return Plan().table_scan(sc.TABLE, COLS)


def _region(rows, lock_records=False):
    """rows: list of dicts {column offset: value} (None = NULL), one key each.  lock_records=True puts a Lock and a
    Rollback record above every row, which makes the lean kernel hand the row over to the general kernel (list mode)."""
    kinds = {A: "int", B: "int", U: "uint", R: "f64", V: "int"}
    r = kvfmt.Region()
    for h, row in enumerate(rows):
        key = kvfmt.row_key(sc.TABLE, h)
        r.put(key, kvfmt.row_v2([(c, row.get(c), k) for c, k in kinds.items() if c in row]), 10, 20)
        if lock_records:
            r.lock_rec(key, 30, 31, last_change=(20, 1))
            r.rollback(key, 50)
    return r.build(read_ts=sc.READ_TS, n_write_blocks=1)


def _check(plan, host, ctx, jit=ffi.JIT_OFF, device=True, ranges=sc.WHOLE):
    exp = orc.dag_handle(plan, ranges, host)
    assert exp.status == 0, exp.message
    got = DagHandler(plan, ranges, DeviceRegion(host) if device else host, jit=jit).handle_request()
    assert_same_rows(got, exp, ordered=False, ctx=ctx)
    return got, exp


@pytest.fixture(scope="module")
def dirty():
    return sc.dirty_region(1, n_keys=900).build(read_ts=sc.READ_TS, n_write_blocks=2)


# ---- composite keys (BatchSlowHashAggregation) -----------------------------------------------------------------------

@pytest.mark.parametrize("jit", JITS, ids=JIT_IDS)
@pytest.mark.parametrize("bits", [1, 3, 8])
def test_forced_tag_collisions(bits, jit, dirty, monkeypatch):
    """B2_DEBUG_AGG_HASH_BITS keeps `bits` bits of the composite key's hash tag, so that up to 900 different keys share 2,
    8 or 256 tags: probes meet equal tags with different keys inside a warp and across CTAs, and only the word-by-word
    key compare keeps the groups apart.  The variable is read when a request opens."""
    monkeypatch.setenv("B2_DEBUG_AGG_HASH_BITS", str(bits))
    for name, plan in sc.multi_group_plans():
        exp = orc.dag_handle(plan, sc.split_ranges(), dirty)
        for device in (False, True):
            got = DagHandler(plan, sc.split_ranges(), DeviceRegion(dirty) if device else dirty, jit=jit).handle_request()
            assert_same_rows(got, exp, ordered=False, float_rel_tol=1e-12 if name == "mg_same_expr_twice" else None,
                             ctx=f"{name}/bits{bits}/{'device' if device else 'host'}")


def test_forced_tag_collisions_backward(dirty, monkeypatch):
    """The same with a backward table scan (TableScan.desc): rows reach the table in the opposite order."""
    monkeypatch.setenv("B2_DEBUG_AGG_HASH_BITS", "1")
    plan = Plan().table_scan(sc.TABLE, sc.COLUMNS, desc=True).aggregation(
        [("count", const_int(1)), ("sum", col(sc.C1))], group_by=[col(sc.C6, tp=ffi.TP_LONG), col(sc.C2), col(sc.C3, unsigned=True)]).build()
    _check(plan, dirty, "desc/bits1")


def _race_rows(n_windows):
    """32-row windows of 30 keys that none of the earlier windows holds, keys 0 and 1 of the window twice: with more than
    28 groups in a warp there is no warp pre-aggregation, so two lanes of one warp insert the same new key together."""
    rows = []
    for w in range(n_windows):
        ks = [30 * w + j for j in range(30)] + [30 * w, 30 * w + 1]
        for k in ks:
            rows.append({A: k // 5, B: k % 5 - 2, U: (k * 0x9E3779B97F4A7C15) & U64, R: float(-k), V: k * 7 - 1000})
    return rows


def race_plans():
    by = [col(A), col(B), col(U, unsigned=True), col(R, tp=ffi.TP_DOUBLE)]
    return [(f"race{n}", _scan().aggregation([("count", const_int(1)), ("sum", col(V)), ("max", col(V))], group_by=by[:n]).build()) for n in (2, 3, 4)]


@pytest.fixture(scope="module")
def race_region():
    return _region(_race_rows(400))


@pytest.mark.parametrize("jit", JITS, ids=JIT_IDS)
def test_same_new_key_in_one_warp(jit, race_region):
    """No knob: the production race between two lanes of one warp that insert the same new composite key."""
    for name, plan in race_plans():
        got, exp = _check(plan, race_region, f"{name}/{jit}", jit=jit)
        assert exp.n_rows == 400 * 30 and sorted(r[0] for r in got.rows())[-800:] == [2] * 800


@pytest.fixture(scope="module")
def edge_region():
    rows = []
    for rep in range(40):
        for a, b in ((None, 0), (0, None), (0, 0), (None, None)):
            rows.append({A: a, B: b, V: rep})
        for s in (-1, I64_MIN, 0, 1):
            for u in (U64, 1 << 63, 0, 1):
                rows.append({A: s, U: u, V: rep})
        for r in (0.0, -0.0):
            rows.append({R: r, A: 0, V: rep})
    return _region(rows)


@pytest.mark.parametrize("bits", [0, 1])
def test_composite_key_edges(bits, edge_region, monkeypatch):
    """Keys that differ only in their NULL mask ((NULL, 0), (0, NULL), (0, 0), (NULL, NULL)); a signed and an unsigned
    column whose value words are equal (-1 and 2^64-1, INT64_MIN and 2^63), in both orders; 0.0 and -0.0, which are
    different groups in the slow hash executor.  With bits=1 all of them share a tag, so the key compare decides."""
    monkeypatch.setenv("B2_DEBUG_AGG_HASH_BITS", str(bits))
    aggs = [("count", const_int(1)), ("sum", col(V))]
    for name, by in (("nullmask", [col(A), col(B)]), ("signed_unsigned", [col(A), col(U, unsigned=True)]),
                     ("unsigned_signed", [col(U, unsigned=True), col(A)]), ("negzero", [col(R, tp=ffi.TP_DOUBLE), col(A)])):
        got, exp = _check(_scan().aggregation(aggs, group_by=by).build(), edge_region, f"{name}/bits{bits}")
        assert all(r[0] % 40 == 0 for r in got.rows()), name
    got, _ = _check(_scan().aggregation(aggs, group_by=[col(R, tp=ffi.TP_DOUBLE), col(A)]).build(), edge_region, "negzero")
    assert sum(1 for r in got.rows() if r[2] == 0.0 and r[3] == 0) == 2  # 0.0 and -0.0


# ---- single-key tables ---------------------------------------------------------------------------------------------

# Aggregate lists and the lean kernel's direct-addressed table they get (engine.cu run_agg: 1024 slots, halved while
# slots * (4 + 8 * acc_words) > 28 KB; COUNT takes 1 accumulator word, MAX / MIN 2, integer SUM / AVG 3).  At most 8
# aggregates of 3 words fit a plan, so integer aggregates cannot bring the table below 128 slots.
LEAN_TABLES = [
    (1024, [("count", const_int(1)), ("max", col(V))]),                            # 3 words
    (512, [("sum", col(V)), ("count", const_int(1)), ("min", col(V))]),            # 6 words
    (256, [("sum", col(V))] * 2 + [("avg", col(V))] * 2),                          # 12 words
    (128, [("sum", col(V))] * 4 + [("avg", col(V))] * 4),                          # 24 words
]
SLOT_EDGES = [e for s in (64, 128, 256, 512, 1024) for e in (s - 1, s, s + 1)]
SPECIAL_KEYS = [0, -1, I64_MIN, I64_MAX, None]


def _single_key_rows():
    rows = []
    for rep in range(6):
        for k in SLOT_EDGES + SPECIAL_KEYS + list(range(rep, 1400, 7)):
            rows.append({A: k, B: rep, U: None if k is None else k & U64, R: 0.5, V: rep * 1000 + (k or 0) % 977})
    return rows


@pytest.fixture(scope="module")
def single_regions():
    rows = _single_key_rows()
    return {"lean": _region(rows), "general": _region(rows, lock_records=True)}


@pytest.mark.parametrize("slots,aggs", LEAN_TABLES, ids=[f"slots{s}" for s, _ in LEAN_TABLES])
def test_single_key_slot_boundaries(slots, aggs, single_regions):
    """Keys s-1, s and s+1 around every table size, and 0, -1 (the table's empty sentinel), INT64_MIN, INT64_MAX and NULL
    in the same request; grouped by a signed and by an unsigned column (2^64-1 is the sentinel there).  Single-version
    rows that hold every column of the plan take the lean kernel (exact row layout); keys below the slot count go to its
    direct-addressed table and are flushed to HBM.  The NULL-key rows lack a column and reach the general kernel."""
    n_keys = len({r[A] for r in _single_key_rows()})
    for c, uns in ((A, False), (U, True)):
        for where, host in single_regions.items():
            got, exp = _check(_scan().aggregation(aggs, group_by=[col(c, unsigned=uns)]).build(), host, f"{slots}/{c}/{where}")
            assert exp.n_rows == n_keys


def test_single_key_real_zero_and_subnormals():
    """Real keys: 0.0 and -0.0 are one group here (fast hash executor); subnormals whose bit patterns are below the slot
    count would share a direct slot with the integer of the same bits if the table ignored the key's type."""
    import struct
    subs = [struct.unpack("<d", struct.pack("<Q", b))[0] for b in (1, 2, 63, 64, 65, 1023, 1024)]
    rows = [{A: i, B: i, U: i, R: r, V: i} for i in range(30) for r in [0.0, -0.0, None, 1.0, -1.0] + subs]
    host = _region(rows)
    for aggs in (LEAN_TABLES[0][1], LEAN_TABLES[2][1]):
        got, _ = _check(_scan().aggregation(aggs, group_by=[col(R, tp=ffi.TP_DOUBLE)]).build(), host, "real")
        assert got.n_rows == 5 + len(subs) - 1


def test_general_cta_table_load_limit(single_regions):
    """The general kernel's 256-slot CTA table stops taking keys at 192; later keys go to HBM, and the CTA table is
    flushed at the end.  Every key has a Lock and a Rollback record above its row, so the lean kernel hands each run over
    to the general kernel (list mode); a 256-entry tile holds more than 192 distinct keys.  Integer aggregates only (an exact Real SUM
    or AVG turns the CTA table off)."""
    host = single_regions["general"]
    for aggs in (LEAN_TABLES[0][1], LEAN_TABLES[3][1]):
        for c, uns in ((A, False), (U, True)):
            _check(_scan().aggregation(aggs, group_by=[col(c, unsigned=uns)]).build(), host, f"general/{c}")


# ---- growth of the HBM table ---------------------------------------------------------------------------------------

def test_table_growth_and_redo():
    """4.5 M groups: more than the first capacity of the HBM table (2^22 slots), so the table overflows, grows x4 and
    the request runs again.  Checks the groups against closed forms and that the statistics describe one pass."""
    n_rows, n_cols, first = 4_500_000, 4, 1000
    lo, rng = [0, 0, 0, 0], [0, 37, 0, 0]
    g, blk = _gen_block(n_rows, n_cols, 2, 11, lo, rng, None, first_handle=first)
    try:
        dev = _source([blk.block], ffi.LOC_DEVICE)
        columns = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(n_cols)]
        scan = lambda: Plan().table_scan(sc.TABLE, columns)
        few = DagHandler(scan().aggregation([("count", const_int(1))], group_by=[col(2)]).build(), sc.WHOLE, dev).handle_request()
        assert few.status == 0 and few.n_rows == 37 and sum(r[0] for r in few.rows()) == n_rows
        want_sum = n_rows * first + n_rows * (n_rows - 1) // 2
        for name, by in (("single", [col(0)]), ("composite", [col(0), const_int(7)])):
            r = DagHandler(scan().aggregation([("count", const_int(1)), ("max", col(0))], group_by=by).build(), sc.WHOLE, dev).handle_request()
            assert r.status == 0, (name, r.message)
            assert r.n_rows == n_rows, name
            cnt, mx = r.columns[0], r.columns[1]
            assert all(x == 1 for x in cnt), name
            assert sum(mx) == want_sum, name
            assert sum(r.columns[2]) == want_sum, name  # the group key column
            assert r.stats.write_processed_keys == few.stats.write_processed_keys == n_rows, name
            assert r.stats.processed_size == few.stats.processed_size, name
    finally:
        ffi.lib().b2_gen_destroy(g)
