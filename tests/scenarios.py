"""Seeded synthetic regions + DAG plans shared by the CPU (device-logic emulation) and GPU parity tests.

Data shape follows SURVEY.md §8(d)'s "dirty" variant: several versions per key, Deletes, Lock/Rollback records
(with and without last_change jumps), versions newer than read_ts, long values in CF_DEFAULT, NULLs, missing
columns with defaults, both row formats in one region.
"""
import random
import struct

import kvfmt
from tikv_b200 import ffi
from tikv_b200.plan import (divide, fn, ColumnDef, Plan, and_, col, const_int, const_real, const_uint, eq, ge, gt, is_null, le, lt, minus, multiply,
                            in_, ne, not_, null, nulleq, or_, plus, xor_, int_divide, mod, neg, abs_, if_null, if_, case_when, coalesce, const_time, const_duration,
                            bit_and, bit_or, bit_xor, bit_neg, cast_int_as_int, cast_int_as_real, cast_real_as_real, const_bytes, like, const_decimal)

TABLE = 1000
READ_TS = 1000

# schema: handle PK, c1 i64, c2 i64 (small domain, nullable), c3 u64, c4 f64, c5 i64 with default 77, c6 i32-domain key
COLUMNS = [
    ColumnDef(100, pk_handle=True),
    ColumnDef(1),
    ColumnDef(2),
    ColumnDef(3, unsigned=True),
    ColumnDef(4, tp=ffi.TP_DOUBLE),
    ColumnDef(5, default=kvfmt.datum_int(77)),
    ColumnDef(6, tp=ffi.TP_LONG),
]
C_H, C1, C2, C3, C4, C5, C6 = range(7)


def _row_value(rng, fmt, full_range=True):
    c1 = rng.randrange(-(1 << 63), 1 << 63) if full_range else rng.randrange(-(1 << 40), 1 << 40)
    c2 = None if rng.random() < 0.1 else rng.randrange(-50, 50)
    c3 = rng.choice([0, 1, (1 << 64) - 1, 1 << 63, rng.randrange(0, 1 << 64)])
    c4 = None if rng.random() < 0.05 else rng.choice([0.0, -0.0, 1.5, -2.25, rng.uniform(-1e6, 1e6)])
    c5 = None if rng.random() < 0.5 else rng.randrange(-1000, 1000)  # None => column missing => default 77
    c5_explicit_null = rng.random() < 0.1
    c6 = rng.randrange(0, 16)
    if fmt == 2:
        cols = [(1, c1, "int"), (2, c2, "int"), (3, c3, "uint"), (4, c4, "f64"), (6, c6, "int")]
        if c5 is not None:
            cols.append((5, None if c5_explicit_null else c5, "int"))
        rng.shuffle(cols)
        return kvfmt.row_v2(cols)
    d = [(1, kvfmt.datum_int(c1)), (2, kvfmt.datum_null() if c2 is None else kvfmt.datum_int(c2)),
         (3, kvfmt.datum_uint(c3) if rng.random() < 0.5 else kvfmt.datum_uint(c3, comparable=True)),
         (4, kvfmt.datum_null() if c4 is None else kvfmt.datum_f64(c4)), (6, kvfmt.datum_int(c6, comparable=rng.random() < 0.3))]
    if c5 is not None:
        d.append((5, kvfmt.datum_null() if c5_explicit_null else kvfmt.datum_int(c5)))
    if rng.random() < 0.2:
        d.append((99, kvfmt.datum_bytes(b"unknown column")))  # unknown column ids are skipped
    rng.shuffle(d)
    return kvfmt.row_v1(d)


def dirty_region(seed, n_keys=600, full_range=True, long_values=True, only_fmt=None):
    """Region with every MVCC shape the forward scanner handles."""
    rng = random.Random(seed)
    r = kvfmt.Region()
    for h in range(n_keys):
        key = kvfmt.row_key(TABLE, h * 3 - 100)
        shape = rng.random()
        fmt = 2 if rng.random() < 0.6 else 1
        if only_fmt:
            fmt = only_fmt
        val = _row_value(rng, fmt, full_range)
        if shape < 0.45:  # single visible put
            r.put(key, val, 10, 20)
        elif shape < 0.55:  # older + visible + newer-than-read_ts versions
            r.put(key, _row_value(rng, fmt, full_range), 5, 8)
            r.put(key, val, 10, 20)
            r.put(key, _row_value(rng, fmt, full_range), READ_TS + 5, READ_TS + 9)
        elif shape < 0.62:  # visible version is a Delete
            r.put(key, val, 10, 20)
            r.delete(key, 30, 40)
        elif shape < 0.70:  # Lock / Rollback records above the visible put (step by next)
            r.put(key, val, 10, 20)
            r.lock_rec(key, 30, 31, last_change=(20, 1))
            r.rollback(key, 50)
            r.lock_rec(key, 60, 61)  # last_change unknown
        elif shape < 0.76:  # many lock records: last_change jump (estimated versions >= SEEK_BOUND)
            r.put(key, _row_value(rng, fmt, full_range), 2, 3)
            r.put(key, val, 10, 20)
            for i in range(10):
                r.lock_rec(key, 100 + 2 * i, 101 + 2 * i, last_change=(20, i + 1))
        elif shape < 0.80:  # only lock records, last change does not exist
            for i in range(3):
                r.lock_rec(key, 100 + 2 * i, 101 + 2 * i, last_change=(0, 1))
        elif shape < 0.85 and long_values:  # long value -> CF_DEFAULT
            big = kvfmt.row_v2([(1, rng.randrange(-100, 100), "int"), (2, 1, "int"), (3, 5, "uint"), (4, 2.5, "f64"), (6, 3, "int"),
                                (7, bytes(rng.randrange(256) for _ in range(300)), "bytes")])
            r.put(key, big, 10, 20)
        elif shape < 0.90:  # gc fence: fenced (invisible) or not
            r.put(key, val, 10, 20, overlapped_rollback=True, gc_fence=rng.choice([0, 500, READ_TS, READ_TS + 1, 30]))
        elif shape < 0.95:  # only versions newer than read_ts
            r.put(key, val, READ_TS + 1, READ_TS + 2)
        else:  # 12 newer versions: move_write_cursor_to_ts goes over SEEK_BOUND
            r.put(key, val, 10, 20)
            for i in range(12):
                r.put(key, _row_value(rng, fmt, full_range), READ_TS + 10 + 2 * i, READ_TS + 11 + 2 * i)
    return r


WHOLE = [kvfmt.table_range(TABLE)]


def plans():
    """(name, Plan) list.  Column offsets refer to COLUMNS."""
    P = []

    def scan():
        return Plan().table_scan(TABLE, COLUMNS)

    P.append(("scan_all", scan().build()))
    P.append(("scan_subset_cols", scan().build(output_offsets=[C4, C_H, C2])))
    P.append(("sel_lt_const", scan().selection(lt(col(C1), const_int(0))).build()))
    P.append(("sel_handle_range", scan().selection(ge(col(C_H), const_int(50)), le(col(C_H), const_int(900))).build()))
    P.append(("sel_null_semantics", scan().selection(gt(col(C2), const_int(-10))).build()))
    P.append(("sel_nulleq", scan().selection(nulleq(col(C2), null())).build()))
    P.append(("sel_is_null_or", scan().selection(or_(is_null(col(C2)), eq(col(C2), const_int(7)))).build()))
    P.append(("sel_not_xor", scan().selection(xor_(not_(gt(col(C2), const_int(0))), lt(col(C6), const_int(8)))).build()))
    P.append(("sel_unsigned_cmp", scan().selection(gt(col(C3, unsigned=True), const_uint(1 << 63))).build()))
    P.append(("sel_mixed_sign_cmp", scan().selection(lt(col(C2), col(C3, unsigned=True))).build()))
    P.append(("sel_uint_vs_int", scan().selection(ge(col(C3, unsigned=True), col(C2))).build()))
    P.append(("sel_real", scan().selection(le(col(C4, tp=ffi.TP_DOUBLE), const_real(1.5))).build()))
    P.append(("sel_real_ne", scan().selection(ne(col(C4, tp=ffi.TP_DOUBLE), const_real(0.0))).build()))
    P.append(("sel_default_col", scan().selection(eq(col(C5), const_int(77))).build()))
    P.append(("sel_arith", scan().selection(lt(plus(col(C2), multiply(col(C6), const_int(3))), const_int(20))).build()))
    P.append(("sel_arith_minus", scan().selection(gt(minus(col(C6), col(C2)), const_int(10))).build()))
    P.append(("sel_and_two_conds", scan().selection(and_(lt(col(C2), const_int(25)), gt(col(C6), const_int(2))), ne(col(C5), const_int(0))).build()))
    P.append(("count_star", scan().aggregation([("count", const_int(1))]).build()))
    P.append(("count_col_sum_avg", scan().aggregation([("count", col(C2)), ("sum", col(C2)), ("avg", col(C6))]).build()))
    P.append(("sum_fullrange", scan().aggregation([("sum", col(C1)), ("count", const_int(1))]).build()))
    P.append(("sum_unsigned", scan().aggregation([("sum", col(C3, unsigned=True))]).build()))
    P.append(("agg_after_filter", scan().selection(lt(col(C1), const_int(0))).aggregation([("count", const_int(1)), ("sum", col(C1))]).build()))
    P.append(("agg_no_input", scan().selection(lt(col(C6), const_int(-5))).aggregation([("count", const_int(1)), ("sum", col(C1))]).build()))
    P.append(("group_by_small", scan().aggregation([("sum", col(C1)), ("count", const_int(1))], group_by=[col(C6, tp=ffi.TP_LONG)]).build()))
    P.append(("group_by_nullable", scan().aggregation([("count", const_int(1)), ("avg", col(C1)), ("sum", col(C5))], group_by=[col(C2)]).build()))
    P.append(("group_by_handle_many", scan().aggregation([("sum", col(C6)), ("count", col(C2))], group_by=[col(C_H)]).build()))
    P.append(("group_by_expr", scan().aggregation([("count", const_int(1))], group_by=[plus(col(C6), const_int(100))]).build()))
    P.append(("group_by_real", scan().aggregation([("count", const_int(1))], group_by=[col(C4, tp=ffi.TP_DOUBLE)]).build()))
    P.append(("group_filter_offsets", scan().selection(ge(col(C6), const_int(4))).aggregation([("sum", col(C2)), ("count", const_int(1))], group_by=[col(C6, tp=ffi.TP_LONG)]).build(output_offsets=[2, 0])))
    return P


def real_sum_plans():
    def scan():
        return Plan().table_scan(TABLE, COLUMNS)
    return [("sum_real", scan().aggregation([("sum", col(C4, tp=ffi.TP_DOUBLE)), ("avg", col(C4, tp=ffi.TP_DOUBLE))]).build()),
            ("sum_real_group", scan().aggregation([("sum", col(C4, tp=ffi.TP_DOUBLE))], group_by=[col(C6, tp=ffi.TP_LONG)]).build())]


def check_exact_real_sums(run, region):
    """SUM / AVG over Real are exactly rounded on the device path (b2_device.h f64_acc_add / f64_acc_round): the result is
    the correctly rounded sum of the group's values whatever the order — compare bit for bit with math.fsum over the
    values the oracle's plain scan returns, and (loosely) with the oracle's own sequential sum."""
    import math
    import orc
    rows = orc.dag_handle(Plan().table_scan(TABLE, COLUMNS).build(output_offsets=[C6, C4]), WHOLE, region).rows()
    by = {}
    for g, v in rows:
        if v is not None:
            by.setdefault(g, []).append(v)
    assert by and max(len(v) for v in by.values()) > 10
    plans = dict(real_sum_plans())
    got = run(plans["sum_real_group"])
    assert got.status == 0
    assert {g: s for s, g in got.rows()} == {g: math.fsum(v) for g, v in by.items()}  # bit-exact: 0 ULP from the true sum's rounding
    allv = [x for v in by.values() for x in v]
    got = run(plans["sum_real"])  # [SUM, AVG count, AVG sum]
    assert got.rows() == [(math.fsum(allv), len(allv), math.fsum(allv))]
    seq = orc.dag_handle(plans["sum_real"], WHOLE, region).rows()[0][0]
    assert math.isclose(seq, math.fsum(allv), rel_tol=1e-12)  # the reference's sequential sum is only this close to it


def topn_plans(desc=False):
    """(name, Plan, exact) — exact=False when ties at the cut make the surviving rows ambiguous in the reference too
    (TopNHeap keeps whichever tied rows its binary heap happens to hold): then only the sort keys are compared.
    desc=True: the same plans over a backward scan."""
    def scan():
        return Plan().table_scan(TABLE, COLUMNS, desc=desc)
    return [
        ("topn_two_keys", scan().topn([(col(C2), True), (col(C1), False)], 50).build(), True, None),
        ("topn_real_desc_handle", scan().topn([(col(C4, tp=ffi.TP_DOUBLE), True), (col(C_H), False)], 30).build(), True, None),
        ("topn_expr", scan().topn([(plus(col(C6), col(C2)), False), (col(C_H), True)], 40).build(), True, None),
        ("topn_all_rows", scan().topn([(col(C1), False), (col(C_H), False)], 2000).build(), True, None),
        ("topn_all_rows_ties", scan().topn([(col(C1), False)], 2000).build(), False, [C1]),
        ("topn_zero", scan().topn([(col(C1), False)], 0).build(), True, None),
        ("topn_after_filter", scan().selection(lt(col(C6), const_int(8))).topn([(col(C1), True)], 25).build(output_offsets=[C1, C6, C_H]), True, None),
        ("topn_unsigned_ties", scan().topn([(col(C3, unsigned=True), False)], 20).build(), False, [C3]),
        ("topn_small_domain_ties", scan().topn([(col(C6), True), (col(C2), False)], 60).build(), False, [C6, C2]),
    ]


def is_agg(name):
    return name.startswith(("count", "sum", "agg", "group"))


def split_ranges():
    return [kvfmt.table_range(TABLE, -1000, 50), kvfmt.table_range(TABLE, 50, 51), kvfmt.table_range(TABLE, 400, 1000), kvfmt.table_range(TABLE, 1200, 5000)]


# ---- all-integer table: exercises the exact-layout fast path (SWAR width probe, conditions and outputs by stored position)
INT_COLUMNS = [ColumnDef(100, pk_handle=True), ColumnDef(7, unsigned=True), ColumnDef(2), ColumnDef(11), ColumnDef(3, unsigned=True),
               ColumnDef(5, tp=ffi.TP_LONG), ColumnDef(9), ColumnDef(4), ColumnDef(6, unsigned=True)]


def int_region(seed, n_keys=500, corrupt=False, fmt=2, ts=(5, 8)):
    """v2 rows holding exactly the 8 stored columns above with every width mix (1/2/4/8 bytes), some rows with a NULL or a
    missing column (general path), optionally rows with a 3-byte integer or decreasing offsets (errors)."""
    rng = random.Random(seed)
    r = kvfmt.Region()
    mags = [1 << 6, 1 << 14, 1 << 30, 1 << 62]
    for h in range(n_keys):
        cols = []
        for cid, uns in ((7, True), (2, False), (11, False), (3, True), (5, False), (9, False), (4, False), (6, True)):
            m = rng.choice(mags)
            v = rng.randrange(0, 2 * m) if uns else rng.randrange(-m, m)
            if cid == 5:
                v = rng.randrange(-(1 << 31), 1 << 31) if rng.random() < 0.5 else rng.randrange(-100, 100)
            cols.append((cid, v, "uint" if uns else "int"))
        x = rng.random()
        if x < 0.05:
            k = rng.randrange(8)
            cols[k] = (cols[k][0], None, "null")
        elif x < 0.08:
            cols.pop(rng.randrange(8))
        if fmt == 1:
            # v1: `08 id datum` per column; INT / UINT / VAR_INT / VAR_UINT flags mixed, sometimes out of id order, an
            # unknown extra column, a NIL datum: all but the plain in-order rows take the general datum walk
            d = []
            for cid, v, kind in cols:
                if v is None:
                    d.append((cid, kvfmt.datum_null()))
                elif kind == "uint":
                    d.append((cid, kvfmt.datum_uint(v, comparable=rng.random() < 0.3)))
                else:
                    d.append((cid, kvfmt.datum_int(v, comparable=rng.random() < 0.3)))
            d.sort(key=lambda t: t[0])
            y = rng.random()
            if y < 0.04:
                rng.shuffle(d)
            elif y < 0.07:
                d.append((40, kvfmt.datum_int(1)))
            val = bytearray(kvfmt.row_v1(d))
            if corrupt and 0.5 < x < 0.52 and len(cols) == 8:
                val = val[:-1] if val[-1] >= 0x80 or rng.random() < 0.5 else val + b"\x08"  # truncated datum / dangling id marker
            r.put(kvfmt.row_key(TABLE, h * 2 + 5), bytes(val), ts[0], ts[1])
            continue
        val = bytearray(kvfmt.row_v2(cols))
        if corrupt and 0.5 < x < 0.52 and len(cols) == 8:
            # widen the first value to 3 bytes by shifting every offset up by one where possible: rewrite offsets by hand
            offs_at = 6 + 8
            ends = list(struct.unpack_from("<8H", val, offs_at))
            if rng.random() < 0.5 and ends[1] - ends[0] >= 2:
                ends[0] += 1            # first width + 1 (3, 5 or 9 bytes), second width - 1: not 1/2/4/8 somewhere
            else:
                ends[3], ends[4] = ends[4], ends[3]  # decreasing offsets
            struct.pack_into("<8H", val, offs_at, *ends)
        r.put(kvfmt.row_key(TABLE, h * 2 + 5), bytes(val), ts[0], ts[1])
    return r


def int_plans():
    from tikv_b200.plan import ne
    scan = lambda: Plan().table_scan(TABLE, INT_COLUMNS)
    c = lambda i, **k: col(i, unsigned=INT_COLUMNS[i].flag & ffi.FLAG_UNSIGNED != 0, **k)
    P = [("all", scan().build()),
         ("lt_signed", scan().selection(lt(c(2), const_int(0))).build()),
         ("const_on_left", scan().selection(gt(const_int(1000), c(3))).build(output_offsets=[3, 0, 8, 1, 1, 5])),
         ("unsigned_vs_negative", scan().selection(gt(c(1), const_int(-5)), le(c(4), const_int(1 << 40))).build()),
         ("eq_ne", scan().selection(ne(c(5), const_int(7)), ge(c(7), const_int(-(1 << 20)))).build(output_offsets=[7, 6, 5, 4, 3, 2, 1, 0])),
         ("agg", scan().selection(lt(c(6), const_int(1 << 20))).aggregation([("count", const_int(1)), ("sum", c(1)), ("sum", c(2)), ("avg", c(8))], group_by=[c(5, tp=ffi.TP_LONG)]).build()),
         ("topn", scan().selection(ge(c(3), const_int(0))).topn([(c(4), True), (c(2), False)], 40).build())]
    return P


def limit_plans():
    scan = lambda: Plan().table_scan(TABLE, COLUMNS)
    return [("limit_scan", scan().limit(37).build()),
            ("limit_after_selection", scan().selection(lt(col(C1), const_int(0))).limit(100).build(output_offsets=[C_H, C1, C3])),
            ("limit_zero", scan().limit(0).build()),
            ("limit_beyond_table", scan().selection(ge(col(C6), const_int(0))).limit(1 << 20).build())]


def minmax_plans():
    """MAX / MIN over signed, unsigned and Real arguments (impl_max_min.rs), with and without GROUP BY, NULL inputs, an
    empty input (no row passes -> no output row for simple agg), groups whose argument is always NULL."""
    scan = lambda: Plan().table_scan(TABLE, COLUMNS)
    return [("minmax_simple", scan().aggregation([("max", col(C1)), ("min", col(C1)), ("max", col(C3, unsigned=True)), ("min", col(C3, unsigned=True)),
                                                   ("max", col(C4, tp=ffi.TP_DOUBLE)), ("min", col(C4, tp=ffi.TP_DOUBLE)), ("min", col(C2)), ("count", const_int(1))]).build()),
            ("minmax_group", scan().selection(lt(col(C1), const_int(1 << 62))).aggregation([("min", col(C2)), ("max", col(C1)), ("sum", col(C2)), ("max", col(C4, tp=ffi.TP_DOUBLE)),
                                                                                            ("min", col(C3, unsigned=True))], group_by=[col(C6, tp=ffi.TP_LONG)]).build()),
            ("minmax_expr", scan().aggregation([("max", plus(col(C6, tp=ffi.TP_LONG), const_int(5))), ("min", col(C_H))], group_by=[col(C2)]).build(output_offsets=[2, 1, 0])),
            ("minmax_empty", scan().selection(lt(col(C1), const_int(-(1 << 63)))).aggregation([("max", col(C1)), ("min", col(C3, unsigned=True))]).build())]


def multi_group_plans():
    """BatchSlowHashAggregation (slow_hash_aggr_executor.rs): GROUP BY over 2..4 expressions; NULLs in any key position,
    Real keys (0.0 and -0.0 stay apart here), one group per row, repeated expressions, reordered output offsets."""
    scan = lambda: Plan().table_scan(TABLE, COLUMNS)
    c6 = col(C6, tp=ffi.TP_LONG)
    return [("mg_two_ints", scan().aggregation([("count", const_int(1)), ("sum", col(C1))], group_by=[c6, col(C2)]).build()),
            ("mg_with_handle", scan().aggregation([("sum", c6), ("count", col(C2))], group_by=[col(C_H), c6]).build()),
            ("mg_real_negzero", scan().aggregation([("count", const_int(1)), ("max", col(C1))], group_by=[multiply(col(C4, tp=ffi.TP_DOUBLE), const_real(-0.0)), c6]).build()),
            ("mg_four", scan().aggregation([("avg", col(C1)), ("min", col(C2))], group_by=[c6, col(C2), is_null(col(C5)), col(C3, unsigned=True)]).build()),
            ("mg_filter_offsets", scan().selection(ge(c6, const_int(4))).aggregation([("sum", col(C2)), ("count", const_int(1))], group_by=[col(C2), c6]).build(output_offsets=[3, 0, 2])),
            ("mg_same_expr_twice", scan().aggregation([("sum", col(C4, tp=ffi.TP_DOUBLE))], group_by=[c6, c6]).build()),
            ("mg_no_input", scan().selection(lt(c6, const_int(-5))).aggregation([("count", const_int(1))], group_by=[c6, col(C2)]).build())]


def one_():
    return const_int(1)


def scalar_plans():
    """More scalar functions (SURVEY 8(f) rank 4): DIV / MOD in every signedness mix (x / 0 and x % 0 are NULL), MOD over
    Real, unary minus, ABS, IFNULL, IF, CASE WHEN (with and without ELSE), COALESCE; as projection outputs, selection
    conditions, aggregate arguments and group keys; and the overflow errors of DIV, unary minus and ABS."""
    scan = lambda: Plan().table_scan(TABLE, COLUMNS)
    c1, c2, c3, c4, c5, c6, ch = col(C1), col(C2), col(C3, unsigned=True), col(C4, tp=ffi.TP_DOUBLE), col(C5), col(C6, tp=ffi.TP_LONG), col(C_H)
    zero, r0 = const_int(0), const_real(0.0)
    return [("sc_div_signed", scan().projection(ch, int_divide(c1, c2), mod(c1, c2), int_divide(c2, c6), mod(c2, c6), mod(c1, const_int(-1))).build()),
            ("sc_div_unsigned", scan().projection(ch, int_divide(c3, c3), mod(c3, c3), mod(c3, c2), mod(c2, c3), int_divide(c3, plus(c6, const_int(1))),
                                                  int_divide(c2, const_uint(1000)), int_divide(const_uint(0), c2), int_divide(c3, abs_(c2))).build()),
            ("sc_real", scan().projection(ch, mod(c4, const_real(2.5)), mod(c4, multiply(c4, r0)), neg(c4), abs_(c4), if_null(c4, const_real(9.5)),
                                          coalesce(c4, null(ffi.TP_DOUBLE), const_real(1.0)), if_(c2, c4, neg(c4)),
                                          case_when(lt(c4, r0), const_real(-1.0), gt(c4, r0), const_real(1.0))).build()),
            ("sc_divide_real", scan().projection(ch, divide(c4, const_real(0.5)), divide(c4, multiply(c4, r0)), divide(const_real(1.0), c4)).build()),
            ("sc_unary", scan().projection(ch, neg(c2), abs_(c2), abs_(c3), neg(c6), neg(const_uint(1 << 63))).build()),
            ("sc_control", scan().projection(ch, if_null(c2, c6), if_(lt(c2, zero), c1, c5), case_when(lt(c2, const_int(-10)), const_int(1), is_null(c2), const_int(2), gt(c6, const_int(8)), c6, c5),
                                             case_when(lt(c2, zero), c1), coalesce(c2, null(), c5), coalesce(null(), null()), if_(null(), c1, c3), case_when(c5)).build()),
            ("sc_in_selection_agg", scan().selection(gt(mod(ch, const_int(7)), const_int(2)), ne(if_null(c2, zero), int_divide(c6, const_int(2))))
                                          .aggregation([("sum", abs_(c2)), ("count", case_when(gt(c6, const_int(5)), c6)), ("max", neg(c6))], group_by=[mod(ch, const_int(5))]).build()),
            ("sc_bits_casts", scan().projection(ch, bit_and(c1, c3), bit_or(c2, c6), bit_xor(c1, c2), bit_neg(c2), cast_int_as_int(c2, unsigned=True), cast_int_as_real(c2),
                                                cast_int_as_real(c3), cast_int_as_real(c2, unsigned=True), cast_real_as_real(c4)).build()),
            ("sc_bits_sel_agg", scan().selection(ne(bit_and(ch, const_int(3)), zero), lt(cast_int_as_real(c6), const_real(7.5)))
                                      .aggregation([("sum", bit_and(c1, const_int(0xffff))), ("count", one_())], group_by=[bit_and(ch, const_int(7))]).build()),
            ("sc_err_div_overflow", scan().projection(ch, int_divide(c2, c3)).build()),
            ("sc_err_div_overflow2", scan().projection(ch, int_divide(c3, c2)).build()),
            ("sc_err_neg_uint", scan().projection(ch, neg(c3)).build()),
            ("sc_err_abs_min", scan().projection(ch, abs_(plus(const_int(-(1 << 63)), multiply(c2, zero)))).build()),
            ("sc_err_neg_min", scan().selection(lt(neg(plus(const_int(-(1 << 63)), c6)), zero)).build())]


def scalar_known_answers():
    """(label, Expr over constants, expected value | None | "error"): the reference's own unit-test vectors for the scalar
    functions above — impl_arithmetic.rs test_mod_int :735-760, test_mod_int_unsigned :763-805, test_mod_real :808-835,
    test_int_divide_int :902-948, test_int_divide_int_overflow :951-983; impl_op.rs test_unary_minus_int :425-472;
    impl_math.rs test_abs_int :854-866; impl_control.rs test_if_null :150-165, test_case_when :168-207, test_if :243-250;
    test_plus_int / test_plus_real / test_minus_int / test_minus_real; the bit operators and casts (cited where they are added)."""
    MAX, MIN, UMAX = (1 << 63) - 1, -(1 << 63), (1 << 64) - 1

    def I(v, unsigned=False):
        if v is None:
            return null()
        return const_uint(v & UMAX) if unsigned else const_int(v)

    def R(v):
        return null(ffi.TP_DOUBLE) if v is None else const_real(v)
    K = []
    for a, b, e in [(13, 11, 2), (-13, 11, -2), (13, -11, 2), (-13, -11, -2), (33, 11, 0), (33, -11, 0), (-33, -11, 0), (-11, None, None), (None, -11, None),
                    (11, 0, None), (-11, 0, None), (MAX, MIN, MAX), (MIN, MAX, -1)]:
        K.append((f"mod_int({a},{b})", mod(I(a), I(b)), e))
    K.append(("mod_int(u64max u, i64min)", mod(I(UMAX, True), I(MIN)), MAX))
    K.append(("mod_int(i64min, u64max u)", mod(I(MIN), I(UMAX, True)), MIN))
    for a, b, e in [(1.0, None, None), (None, 1.0, None), (1.0, 1.1, 1.0), (-1.0, 1.1, -1.0), (1.0, -1.1, 1.0), (-1.0, -1.1, -1.0), (1.0, 0.0, None)]:
        K.append((f"mod_real({a},{b})", mod(R(a), R(b)), e))
    for a, au, b, bu, e in [(13, False, 11, False, 1), (13, False, -11, False, -1), (-13, False, 11, False, -1), (-13, False, -11, False, 1), (33, False, 11, False, 3),
                            (33, False, -11, False, -3), (-33, False, 11, False, -3), (-33, False, -11, False, 3), (11, False, 0, False, None), (-11, False, 0, False, None),
                            (-3, False, 5, True, 0), (3, False, -5, False, 0), (MIN + 1, False, -1, False, MAX), (MIN, False, 1, False, MIN), (MAX, False, 1, False, MAX),
                            (UMAX, True, 1, False, -1),  # u64::MAX as i64
                            (MIN, False, -1, False, "error"), (-1, False, 1, True, "error"), (-2, False, 1, True, "error"), (1, True, -1, False, "error"), (2, True, -1, False, "error")]:
        K.append((f"int_divide({a}{'u' if au else ''},{b}{'u' if bu else ''})", int_divide(I(a, au), I(b, bu)), e))
    for a, e in [(None, None), (MAX + 1, MIN), (12345, -12345), (0, 0), (MAX + 2, "error")]:
        K.append((f"neg_uint({a})", neg(I(a, True)), e))
    for a, e in [(None, None), (MAX, -MAX), (-MAX, MAX), (MIN + 1, MAX), (0, 0), (MIN, "error")]:
        K.append((f"neg_int({a})", neg(I(a)), e))
    for a, au, e in [(-3, False, 3), (MAX, False, MAX), (UMAX, True, -1), (MIN, False, "error")]:
        K.append((f"abs({a})", abs_(I(a, au)), e))
    for a, b, e in [(None, None, None), (None, 1, 1), (2, None, 2), (2, 1, 2)]:
        K.append((f"if_null({a},{b})", if_null(I(a), I(b)), e))
    for args, e in [([I(1), R(3.0), I(1), R(5.0)], 3.0), ([I(0), R(3.0), I(1), R(5.0)], 5.0), ([I(None), R(2.0), I(1), R(6.0)], 6.0), ([R(7.0)], 7.0), ([I(0), R(None)], None),
                    ([I(1), R(None)], None), ([I(1), R(3.5)], 3.5), ([I(2), R(3.5)], 3.5), ([I(0), R(None), I(None), R(None), R(5.5)], 5.5)]:
        K.append((f"case_when#{len(K)}", case_when(*args) if len(args) > 1 else fn("CASE_WHEN_REAL", args[0], ret_tp=ffi.TP_DOUBLE), e))
    import math
    for c, e in [(0, math.pi), (1, math.e), (None, math.pi)]:
        K.append((f"if({c})", if_(I(c), R(math.e), R(math.pi)), e))
    # impl_op.rs test_bit_and :589-605, test_bit_or :608-624, test_bit_xor :627-643, test_bit_neg :646-660
    for a, b, e in [(123, 321, 65), (-123, 321, 257), (None, 1, None), (1, None, None), (None, None, None)]:
        K.append((f"bit_and({a},{b})", bit_and(I(a), I(b)), e))
    for a, b, e in [(123, 321, 379), (-123, 321, -59), (None, 1, None), (1, None, None), (None, None, None)]:
        K.append((f"bit_or({a},{b})", bit_or(I(a), I(b)), e))
    for a, b, e in [(123, 321, 314), (-123, 321, -316), (None, 1, None), (1, None, None), (None, None, None)]:
        K.append((f"bit_xor({a},{b})", bit_xor(I(a), I(b)), e))
    for a, e in [(123, -124), (-123, 122), (0, -1), (None, None)]:
        K.append((f"bit_neg({a})", bit_neg(I(a)), e))
    # impl_cast.rs test_int_as_int_others :1878-1890, test_signed_int_as_unsigned_int :1893-1916 (in_union false),
    # test_signed_int_as_signed_real :3250-3266, test_signed_int_as_unsigned_real :3269-3297 (in_union false),
    # test_unsigned_int_as_signed_or_unsigned_real :3300-3315, test_real_as_signed_real :3318-3338
    for a in (MAX, MIN, -1, None):
        K.append((f"cast_int_as_int({a})", cast_int_as_int(I(a)), a))
    for a in (-10, 10, MIN, MAX):
        K.append((f"cast_int_as_uint({a})", cast_int_as_int(I(a), unsigned=True), a))  # the same bits, read as u64 by the caller
    for a in (MIN, 0, MAX, None):
        K.append((f"cast_int_as_real({a})", cast_int_as_real(I(a)), None if a is None else float(a)))
    for a in (MAX, 0):
        K.append((f"cast_int_as_ureal({a})", cast_int_as_real(I(a), unsigned=True), float(a)))
    K.append(("cast_int_as_ureal(-1)", cast_int_as_real(I(-1), unsigned=True), float(UMAX)))  # `as u64 as f64`
    for a in (0, UMAX, MAX):
        K.append((f"cast_uint_as_real({a})", cast_int_as_real(I(a, True)), float(a)))
    # impl_arithmetic.rs test_plus_int :551-588, test_plus_real :591-617, test_minus_int :636-678, test_minus_real :681-713
    FMAX = 1.7976931348623157e308
    for a, au, b, bu, e in [(None, False, 1, False, None), (1, False, None, False, None), (17, False, 25, False, 42), (MIN, False, MAX + 1, True, 0)]:
        K.append((f"plus_int({a}{'u' if au else ''},{b}{'u' if bu else ''})", plus(I(a, au), I(b, bu)), e))
    for a, au, b, bu, e in [(None, False, 1, False, None), (1, False, None, False, None), (12, False, 1, False, 11), (0, True, MIN, False, MIN),  # (i64::MAX as u64 + 1) as i64
                            (MIN, False, MAX, False, "error"), (MAX, False, MIN, False, "error"), (-1, False, 2, True, "error"), (1, True, 2, False, "error")]:
        K.append((f"minus_int({a}{'u' if au else ''},{b}{'u' if bu else ''})", minus(I(a, au), I(b, bu)), e))
    for a, b, e in [(1.01001, -0.01, 1.00001), (1e308, 1e308, "error"), (FMAX - 1.0, 2.0, FMAX)]:
        K.append((f"plus_real({a},{b})", plus(R(a), R(b)), e))
    for a, b, e in [(1.01001, -0.01, 1.02001), (-FMAX, FMAX, "error"), (-FMAX, 1.0, -FMAX)]:
        K.append((f"minus_real({a},{b})", minus(R(a), R(b)), e))
    for a in (float.fromhex("-0x1.fffffep+127"), float.fromhex("0x1.fffffep+127"), -1.7976931348623157e308, 0.0, 1.7976931348623157e308, float(MIN), float(MAX), float(UMAX), None):
        K.append((f"cast_real_as_real({a})", cast_real_as_real(R(a)), a))
    # impl_op.rs test_logical_and / _or / _xor, test_unary_not_int / _real, test_is_null (Int, Real, Decimal, Time, Duration arms)
    for a, b, e in [(1, 1, 1), (1, 0, 0), (0, 0, 0), (2, -1, 1), (0, None, 0), (None, 1, None)]:
        K.append((f"and({a},{b})", and_(I(a), I(b)), e))
    for a, b, e in [(1, 1, 1), (1, 0, 1), (0, 0, 0), (2, -1, 1), (1, None, 1), (None, 0, None)]:
        K.append((f"or({a},{b})", or_(I(a), I(b)), e))
    for a, b, e in [(1, 1, 0), (1, 0, 1), (0, 0, 0), (2, -1, 0), (-1, 0, 1), (0, None, None), (None, 1, None)]:
        K.append((f"xor({a},{b})", xor_(I(a), I(b)), e))
    for a, e in [(None, None), (0, 1), (1, 0), (2, 0), (-1, 0)]:
        K.append((f"not_int({a})", not_(I(a)), e))
    for a, e in [(None, None), (0.0, 1), (1.0, 0), (0.3, 0)]:
        K.append((f"not_real({a})", not_(R(a)), e))
    K += [("is_null(int NULL)", is_null(I(None)), 1), ("is_null(int 0)", is_null(I(0)), 0), ("is_null(real NULL)", is_null(R(None)), 1), ("is_null(real 0)", is_null(R(0.0)), 0),
          ("is_null(decimal NULL)", is_null(null(ffi.TP_NEWDECIMAL)), 1), ("is_null(decimal 1)", is_null(const_decimal(kvfmt.decimal_bin("1", 1, 0))), 0),
          ("is_null(time NULL)", is_null(null(ffi.TP_DATETIME)), 1), ("is_null(time zero)", is_null(const_time(0)), 0),
          ("is_null(duration NULL)", is_null(null(ffi.TP_DURATION)), 1), ("is_null(duration 1ns)", is_null(const_duration(1)), 0)]
    return K


def like_known_answers():
    """(target, pattern, escape, collation of the LikeSig node, of the target, of the pattern, expected): impl_like.rs
    test_like :80-258 and test_like_wide_character :261-405, the cases under the collations the device path takes
    (binary and *_bin; the _ci cases are answered B2_ERR_UNSUPPORTED, see like_unsupported_cases)."""
    B, U = 63, -46  # Collation::Binary, Collation::Utf8Mb4Bin (field_type.rs:110-111)
    bs = "\\"
    one = [("hello", "%HELLO%", bs, B, 0), ("Hello, World", "Hello, World", bs, B, 1), ("Hello, World", "Hello, %", bs, B, 1), ("Hello, World", "%, World", bs, B, 1),
           ("test", "te%st", bs, B, 1), ("test", "te%%st", bs, B, 1), ("test", "test%", bs, B, 1), ("test", "%test%", bs, B, 1), ("test", "%%test%", bs, B, 1),
           ("test", "%test%%", bs, B, 1), ("testAAA", "%test%", bs, B, 1), ("testBBB", "%test%%", bs, B, 1), ("test", "t%e%s%t", bs, B, 1), ("test", "_%_%_%_", bs, B, 1),
           ("test", "_%_%st", bs, B, 1), ("C:", "%\\", bs, B, 0), ("C:\\", "%\\", bs, B, 1), ("C:\\Programs", "%\\", bs, B, 0), ("C:\\Programs\\", "%\\", bs, B, 1),
           ("C:", "%\\\\", bs, B, 0), ("C:\\", "%\\\\", bs, B, 1), ("C:\\\\", "C:\\\\", bs, B, 0), ("C:\\Programs", "%\\\\", bs, B, 0), ("C:\\Programs\\", "%\\\\", bs, B, 1),
           ("C:\\Programs\\", "%Prog%", bs, B, 1), ("C:\\Programs\\", "%Pr_g%", bs, B, 1), ("C:\\Programs\\", "%%\\", "%", B, 1), ("C:\\Programs%", "%%%", "%", B, 1),
           ("C:\\Programs%", "%%%%", "%", B, 1), ("hello", "\\%", bs, B, 0), ("%", "\\%", bs, B, 1), ("3hello", "%%hello", "%", B, 1), ("3hello", "3%hello", "3", B, 0),
           ("3hello", "__hello", "_", B, 0), ("3hello", "%_hello", "%", B, 1), ("aaaaaaaaaaaaaaaaaaaaaaaaaaa", "a%a%a%a%a%a%a%a%b", bs, B, 0),
           ("IpHONE", "iPhone", bs, U, 0), ("baab", "b_%b", bs, U, 1), ("baab", "b%_b", bs, U, 1), ("bab", "b_%b", bs, U, 1), ("bab", "b%_b", bs, U, 1), ("bb", "b_%b", bs, U, 0),
           ("bb", "b%_b", bs, U, 0), ("baabccc", "b_%b%", bs, U, 1)]
    out = [(t, p, e, c, c, c, x) for t, p, e, c, x in one]
    out += [("夏威夷吉他", "_____", bs, B, B, B, 0), ("🐶🍐🍳➕🥜🎗🐜", "_______", bs, U, U, U, 1), ("🕺_", "🕺🕺🕺_", "🕺", B, B, B, 0), ("夏威夷吉他", "_____", bs, B, U, U, 1),
            ("🐶🍐🍳➕🥜🎗🐜", "_______", bs, B, U, U, 1), ("🕺_", "🕺🕺🕺_", "🕺", B, U, U, 1), ("测试", "测_", bs, B, U, B, 0), ("测试", "测%", bs, B, U, B, 1), ("测试", "测_", bs, B, U, U, 1)]
    return [(t.encode(), p.encode(), ord(e), c, ct, cp, x) for t, p, e, c, ct, cp, x in out]


def check_like_known_answers(run):
    """The LIKE vectors through `run(plan, ranges, region)` (oracle, emulated device logic, CUDA path): constants only,
    projected over a one-row table, 12 per plan."""
    r = kvfmt.Region()
    r.put(kvfmt.row_key(TABLE, 1), kvfmt.row_v2([(1, 5, "int")]), 1, 2)
    region = r.build(read_ts=10)
    cols = [ColumnDef(100, pk_handle=True), ColumnDef(1)]
    cases = like_known_answers()
    assert len(cases) >= 50
    for i in range(0, len(cases), 12):
        chunk = cases[i:i + 12]
        exprs = [like(const_bytes(t, ct), const_bytes(p, cp), e, collation=c) for t, p, e, c, ct, cp, _ in chunk]
        res = run(Plan().table_scan(TABLE, cols).projection(*exprs).build(), [kvfmt.table_range(TABLE)], region)
        assert res.status == 0, res.message
        assert list(res.rows()[0]) == [x for *_, x in chunk], [(c[0], c[1]) for c, g in zip(chunk, res.rows()[0]) if g != c[-1]]


def in_plans():
    """IN lists (impl_compare_in.rs): constants, NULL in the list, NULL base, columns in the list, signed vs unsigned, Real."""
    scan = lambda: Plan().table_scan(TABLE, COLUMNS)
    return [("in_consts", scan().selection(in_(col(C6, tp=ffi.TP_LONG), const_int(1), const_int(5), const_int(7), const_int(14))).build()),
            ("in_with_null", scan().selection(in_(col(C2), const_int(3), null(), const_int(-2))).build(output_offsets=[C_H, C2])),
            ("in_null_result", scan().selection(is_null(in_(col(C2), const_int(3), null()))).build(output_offsets=[C_H, C2])),
            ("in_not", scan().selection(not_(in_(col(C2), const_int(3), const_int(4)))).build(output_offsets=[C_H, C2])),
            ("in_null_base_and_columns", scan().selection(in_(col(C2), col(C6, tp=ffi.TP_LONG), const_int(0))).build(output_offsets=[C_H, C2, C6])),
            ("in_signedness", scan().selection(in_(col(C3, unsigned=True), const_int(-1), const_uint((1 << 64) - 1), col(C1), const_int(77))).build(output_offsets=[C_H, C3, C1])),
            ("in_real", scan().selection(in_(col(C4, tp=ffi.TP_DOUBLE), const_real(2.5), const_real(-0.0), const_real(1e300))).build(output_offsets=[C_H, C4])),
            ("in_as_group_key", scan().aggregation([("count", const_int(1))], group_by=[in_(col(C6, tp=ffi.TP_LONG), const_int(2), const_int(3), null())]).build())]


def projection_plans():
    """BatchProjectionExecutor on top of scan / selection: arithmetic, compares, IN, plain column refs, Real results, NULLs;
    an overflowing expression (error), Projection followed by Limit, a subset of the projected columns."""
    scan = lambda: Plan().table_scan(TABLE, COLUMNS)
    c6 = col(C6, tp=ffi.TP_LONG)
    return [("proj_mixed", scan().projection(plus(c6, const_int(100)), col(C_H), lt(col(C2), const_int(3)), multiply(col(C4, tp=ffi.TP_DOUBLE), const_real(0.5)),
                                             in_(c6, const_int(1), const_int(2)), col(C3, unsigned=True)).build()),
            ("proj_after_selection_limit", scan().selection(ge(c6, const_int(3))).projection(minus(col(C_H), c6), col(C2)).limit(55).build()),
            ("proj_subset", scan().projection(col(C1), plus(c6, c6), is_null(col(C2))).build(output_offsets=[2, 1])),
            ("proj_overflow", scan().projection(col(C_H), multiply(col(C1), const_int(1 << 40))).build()),
            # Real multiply feeding an add / subtract: separately rounded steps (a fused multiply-add would differ in the last bit)
            ("proj_real_chain", scan().projection(col(C_H), plus(multiply(col(C4, tp=ffi.TP_DOUBLE), const_real(1.1)), const_real(0.3)),
                                                  minus(multiply(col(C4, tp=ffi.TP_DOUBLE), col(C4, tp=ffi.TP_DOUBLE)), multiply(col(C4, tp=ffi.TP_DOUBLE), const_real(1e-3)))).build())]


def check_scalar_known_answers(run, error_labels=None):
    """Evaluate every scalar_known_answers() expression through `run(plan, ranges, region)` (oracle, emulator or the CUDA
    path) as a projection over a one-row table and compare with the reference's expected value."""
    r = kvfmt.Region()
    r.put(kvfmt.row_key(TABLE, 1), kvfmt.row_v2([(1, 5, "int")]), 1, 2)
    region = r.build(read_ts=10)
    cols = [ColumnDef(100, pk_handle=True), ColumnDef(1)]
    cases = scalar_known_answers()
    assert len(cases) >= 170
    scan = lambda: Plan().table_scan(TABLE, cols)
    ok = [c for c in cases if c[2] != "error"]
    for label, expr, _ in [c for c in cases if c[2] == "error"]:  # an error ends the request: one plan per case
        if error_labels is not None and label not in error_labels:
            continue
        res = run(scan().projection(expr).build(), [kvfmt.table_range(TABLE)], region)
        assert res.status == ffi.B2_ERR_EVALUATE and getattr(res, "mysql_code", 1690) == 1690, (label, res.status, res.message)
    for i in range(0, len(ok), 12):  # the others: 12 expressions per projection (one specialised kernel per plan on the GPU)
        chunk = ok[i:i + 12]
        res = run(scan().projection(*[c[1] for c in chunk]).build(), [kvfmt.table_range(TABLE)], region)
        assert res.status == 0, ([c[0] for c in chunk], res.message)
        got = res.rows()
        assert len(got) == 1 and len(got[0]) == len(chunk)
        for (label, _, want), v in zip(chunk, got[0]):
            if isinstance(want, float):
                assert v is not None and struct.pack("<d", v) == struct.pack("<d", want), (label, v, want)
            else:
                assert v == want, (label, v, want)


# ---- the reference's own executor fixtures (MockExecutor batches restated as table rows) ------------------------------
def reference_executor_fixtures():
    """[(name, region, plan, expected rows, ordered, compared columns)] for
      * BatchFastHashAggregationExecutor / BatchSlowHashAggregationExecutor test_it_works_integration
        (fast_hash_aggr_executor.rs:509-634 over util/aggr_executor.rs:434-520 make_src_executor_1),
      * BatchTopNExecutor test_integration_1/2/3 (top_n_executor.rs:463-757) and test_top_unsigned (:1022-1212).
    The MockExecutor's logical rows become table rows (handle = logical position), so that the whole path — MVCC scan,
    row decode, expression evaluation, the executor — must reproduce the reference's expected output."""
    from tikv_b200.plan import plus
    TP_D = ffi.TP_DOUBLE
    out = []

    def table(col_defs, rows, fmt=2):
        r = kvfmt.Region()
        for h, vals in enumerate(rows):
            cells = []
            for (cid, kind), v in zip(col_defs, vals):
                cells.append((cid, v, kind if v is not None else "null"))
            if fmt == 2:
                val = kvfmt.row_v2(cells)
            else:
                d = []
                for cid, v, kind in cells:
                    d.append((cid, kvfmt.datum_null() if v is None else (kvfmt.datum_f64(v) if kind == "f64" else (kvfmt.datum_uint(v) if kind == "uint" else kvfmt.datum_int(v)))))
                val = kvfmt.row_v1(d)
            r.put(kvfmt.row_key(TABLE, h + 1), val, 5, 8)
        return r.build(read_ts=READ_TS)

    # --- hash aggregation: COUNT(1), COUNT(col_1 + 5.0), AVG(col_0) GROUP BY col_0 + col_1
    rows = [(None, 1.0, 1), (7.0, 2.0, None), (None, None, None), (None, 4.5, None), (1.5, 4.5, 5)]
    cols = [ColumnDef(1, tp=TP_D), ColumnDef(2, tp=TP_D), ColumnDef(4)]
    c0, c1 = col(0, tp=TP_D), col(1, tp=TP_D)
    for fmt in (2, 1):
        region = table([(1, "f64"), (2, "f64"), (4, "int")], rows, fmt)
        for n_groups, label in ((1, "fast"), (2, "slow")):
            gb = [plus(c0, c1)] * n_groups if n_groups == 1 else [plus(c0, c1), c0]  # the slow executor, keyed on two expressions
            plan = Plan().table_scan(TABLE, cols).aggregation([("count", const_int(1)), ("count", plus(c1, const_real(5.0))), ("avg", c0)], group_by=gb).build()
            if n_groups == 1:
                exp = [(1, 1, 1, 7.0, 9.0), (1, 1, 1, 1.5, 6.0), (3, 2, 0, None, None)]
            else:  # (col_0 + col_1, col_0): the NULL group stays whole — col_0 is NULL in all three of its rows
                exp = [(1, 1, 1, 7.0, 9.0, 7.0), (1, 1, 1, 1.5, 6.0, 1.5), (3, 2, 0, None, None, None)]
            out.append((f"hash_agg_{label}_v{fmt}", region, plan, exp, False, None))

    # --- TopN: Col0 (Int) Col1 (Int) Col2 (Real)
    rows = [(None, -1, -1.0), (None, None, 2.0), (None, 1, 4.0), (-1, None, None), (-10, 10, 3.0), (-10, None, -5.0), (-10, -10, 0.0)]
    cols = [ColumnDef(1), ColumnDef(2), ColumnDef(3, tp=TP_D)]
    region = table([(1, "int"), (2, "int"), (3, "f64")], rows)
    scan = lambda: Plan().table_scan(TABLE, cols)
    out.append(("topn_integration_1", region, scan().topn([(col(2, tp=TP_D), False)], 100).build(),
                [(-1, None, None), (-10, None, -5.0), (None, -1, -1.0), (-10, -10, 0.0), (None, None, 2.0), (-10, 10, 3.0), (None, 1, 4.0)], True, None))
    out.append(("topn_integration_2", region, scan().topn([(col(0), True), (col(1), False)], 7).build(),
                [(-1, None, None), (-10, None, -5.0), (-10, -10, 0.0), (-10, 10, 3.0), (None, None, 2.0), (None, -1, -1.0), (None, 1, 4.0)], True, None))
    out.append(("topn_integration_3", region, scan().topn([(is_null(col(0)), False), (col(0), False), (plus(col(1), const_int(1)), True)], 5).build(),
                [(-10, 10, 3.0), (-10, -10, 0.0), (-10, None, -5.0), (-1, None, None), (None, 1, 4.0)], True, None))

    # --- TopN over unsigned columns: Col0 (u64) Col1 (i64) Col2 (u32)
    U = (1 << 64)
    rows = [(U - 1, -3, 4294967295), (None, None, None), (U - 3, -1, 4294967295), (2000, 2000, 2000), ((1 << 63) - 1, (1 << 63) - 1, 2147483647),
            (300, 300, 300), (1 << 63, -(1 << 63), 2147483648)]
    cols = [ColumnDef(1, unsigned=True), ColumnDef(2), ColumnDef(3, tp=ffi.TP_LONG, unsigned=True)]
    region = table([(1, "uint"), (2, "int"), (3, "uint")], rows)
    s64 = lambda v: None if v is None else (v - U if v >= (1 << 63) else v)  # columns come back as i64 bits
    cases = [(0, False, [None, 300, 2000, (1 << 63) - 1, 1 << 63]), (0, True, [U - 1, U - 3, 1 << 63, (1 << 63) - 1, 2000]),
             (1, False, [None, -(1 << 63), -3, -1, 300]), (1, True, [(1 << 63) - 1, 2000, 300, -1, -3]),
             (2, False, [None, 300, 2000, 2147483647, 2147483648]), (2, True, [4294967295, 4294967295, 2147483648, 2147483647, 2000])]
    for ci, desc, exp in cases:
        c = col(ci, unsigned=ci != 1, tp=ffi.TP_LONG if ci == 2 else ffi.TP_LONGLONG)
        plan = Plan().table_scan(TABLE, cols).topn([(c, desc)], 5).build()
        out.append((f"topn_unsigned_col{ci}_{'desc' if desc else 'asc'}", region, plan, [(s64(v),) for v in exp], True, [ci]))
    return out


def check_reference_fixture(fx, run):
    """run(plan, region) -> result with .status / .rows(); compares with the reference's expected rows."""
    name, region, plan, exp, ordered, cols = fx
    got = run(plan, region)
    assert got.status == 0, (name, getattr(got, "message", ""))
    rows = got.rows()
    if cols is not None:
        rows = [tuple(r[c] for c in cols) for r in rows]
    if not ordered:
        key = lambda r: tuple((0, 0) if v is None else (1, v) for v in r)
        rows, exp = sorted(rows, key=key), sorted(exp, key=key)
    assert rows == exp, f"{name}: {rows} != reference {exp}"


# ---- tables with bytes / time / duration / decimal / json columns (they stay Raw in the reference until the response) ------
MIXED_COLUMNS = [
    ColumnDef(100, pk_handle=True),
    ColumnDef(1),                                   # BIGINT
    ColumnDef(2, tp=ffi.TP_VARCHAR),
    ColumnDef(3, tp=ffi.TP_DATETIME, decimal=3),
    ColumnDef(4, tp=ffi.TP_DATE),
    ColumnDef(5, tp=ffi.TP_NEWDECIMAL),
    ColumnDef(6, tp=ffi.TP_DURATION, decimal=2),
    ColumnDef(7, tp=ffi.TP_JSON),
    ColumnDef(8, tp=ffi.TP_DOUBLE),
    ColumnDef(9, tp=ffi.TP_BLOB),
]
M_H, M_INT, M_STR, M_DT, M_DATE, M_DEC, M_DUR, M_JSON, M_F64, M_BLOB = range(10)


def mixed_region(seed, n_keys=700, json_in_v1=False):
    """Rows of MIXED_COLUMNS in row formats v2 and v1 (v1 rows carry no JSON cell: the device does not size binary JSON
    datums), with NULLs, empty and long strings, zero dates, negative / fractional decimals, several versions per key and a
    few long values in CF_DEFAULT."""
    rng = random.Random(seed)
    r = kvfmt.Region()

    def cells(fmt):
        out = {}
        out[1] = None if rng.random() < 0.1 else rng.randrange(-1000, 1000)
        out[2] = None if rng.random() < 0.1 else bytes(rng.randrange(32, 127) for _ in range(rng.choice([0, 1, 3, 8, 9, 40, 300])))
        out[3] = None if rng.random() < 0.1 else (0 if rng.random() < 0.1 else kvfmt.time_packed(rng.randrange(1000, 9999), rng.randrange(1, 13), rng.randrange(1, 29), rng.randrange(24), rng.randrange(60), rng.randrange(60), rng.randrange(1000) * 1000))
        out[4] = None if rng.random() < 0.1 else (0 if rng.random() < 0.1 else kvfmt.time_packed(rng.randrange(1, 9999), rng.randrange(1, 13), rng.randrange(1, 29)))
        if rng.random() < 0.1:
            out[5] = None
        else:
            prec, frac = rng.choice([(1, 0), (9, 0), (10, 2), (14, 4), (18, 9), (30, 10), (65, 30), (5, 5)])
            digs = "".join(rng.choice("0123456789") for _ in range(prec)) if rng.random() < 0.9 else "0" * prec
            txt = (digs[:prec - frac] or "0") + ("." + digs[prec - frac:] if frac else "")
            out[5] = (("-" if rng.random() < 0.5 else "") + txt, prec, frac)
        out[6] = None if rng.random() < 0.1 else rng.choice([0, 1, -1, 10 ** 9, -3 * 10 ** 12, rng.randrange(-10 ** 15, 10 ** 15)])
        out[7] = None if rng.random() < 0.2 else rng.choice([kvfmt.json_string("x" * rng.randrange(0, 50)), kvfmt.json_i64(rng.randrange(-5, 5)), bytes([0x04, 0x01])])
        out[8] = None if rng.random() < 0.1 else rng.uniform(-5, 5)
        out[9] = None if rng.random() < 0.3 else bytes(rng.randrange(256) for _ in range(rng.choice([0, 5, 17, 700])))
        if fmt == 2:
            kinds = {1: "int", 2: "bytes", 3: "time", 4: "time", 5: "decimal", 6: "duration", 7: "bytes", 8: "f64", 9: "bytes"}
            return kvfmt.row_v2([(cid, v, kinds[cid]) for cid, v in out.items()])
        d = []
        for cid, v in out.items():
            if cid == 7 and not json_in_v1:
                continue
            if v is None:
                if rng.random() < 0.5:
                    d.append((cid, kvfmt.datum_null()))
                continue  # (a missing cell of a nullable column is NULL as well)
            enc = {1: lambda: kvfmt.datum_int(v), 2: lambda: kvfmt.datum_bytes(v), 3: lambda: kvfmt.datum_time(v), 4: lambda: kvfmt.datum_time(v, comparable=rng.random() < 0.3),
                   5: lambda: kvfmt.datum_decimal(*v), 6: lambda: kvfmt.datum_duration(v, fixed=rng.random() < 0.5), 7: lambda: bytes([10]) + v,
                   8: lambda: kvfmt.datum_f64(v), 9: lambda: kvfmt.datum_bytes(v)}[cid]()
            d.append((cid, enc))
        rng.shuffle(d)
        return kvfmt.row_v1(d)

    for h in range(n_keys):
        key = kvfmt.row_key(TABLE, h * 2 - 50)
        fmt = 2 if rng.random() < 0.6 else 1
        shape = rng.random()
        if shape < 0.7:
            r.put(key, cells(fmt), 10, 20)
        elif shape < 0.85:
            r.put(key, cells(fmt), 5, 8)
            r.put(key, cells(fmt), 10, 20)
            r.put(key, cells(fmt), READ_TS + 5, READ_TS + 9)
        elif shape < 0.92:
            r.put(key, cells(fmt), 10, 20)
            r.delete(key, 30, 40)
        else:
            r.put(key, cells(fmt), 10, 20, force_long=True)
    return r


def mixed_plans():
    scan = lambda: Plan().table_scan(TABLE, MIXED_COLUMNS)
    return [("mixed_all", scan().build()),
            ("mixed_sel", scan().selection(lt(col(M_INT), const_int(0))).build(output_offsets=[M_STR, M_H, M_DEC, M_DT, M_JSON])),
            ("mixed_sel_real_limit", scan().selection(gt(col(M_F64, tp=ffi.TP_DOUBLE), const_real(0.0))).limit(120).build(output_offsets=[M_BLOB, M_DATE, M_DUR, M_INT])),
            ("mixed_only_fixed", scan().build(output_offsets=[M_DT, M_DATE, M_DUR, M_H])),
            # DATE / DATETIME / DURATION predicates (impl_compare.rs over `Ord for Time` / `Ord for Duration`)
            ("mixed_sel_datetime", scan().selection(lt(col(M_DT, tp=ffi.TP_DATETIME), const_time(kvfmt.time_packed(5000, 6, 15, 12, 30, 0, 0)))).build(output_offsets=[M_H, M_DT, M_STR])),
            ("mixed_sel_date_in_null", scan().selection(or_(is_null(col(M_DATE, tp=ffi.TP_DATE)),
                                                            in_(col(M_DATE, tp=ffi.TP_DATE), const_time(0, ffi.TP_DATE), null(ffi.TP_DATE), const_time(kvfmt.time_packed(2000, 1, 1), ffi.TP_DATE)))).build(output_offsets=[M_H, M_DATE])),
            ("mixed_sel_datetime_vs_date", scan().selection(ge(col(M_DT, tp=ffi.TP_DATETIME), col(M_DATE, tp=ffi.TP_DATE))).build(output_offsets=[M_H, M_DT, M_DATE])),
            ("mixed_sel_duration", scan().selection(ge(col(M_DUR, tp=ffi.TP_DURATION), const_duration(0)), ne(col(M_DUR, tp=ffi.TP_DURATION), const_duration(10 ** 9))).build(output_offsets=[M_H, M_DUR, M_BLOB])),
            # LIKE over VARCHAR / BLOB cells (impl_like.rs): binary and utf8mb4_bin, `_` / `%` / escape, NULL operands
            ("mixed_sel_like_contains", scan().selection(like(col(M_STR, tp=ffi.TP_VARCHAR, collation=63), const_bytes(b"%a%"))).build(output_offsets=[M_H, M_STR])),
            ("mixed_sel_like_underscores", scan().selection(or_(like(col(M_STR, tp=ffi.TP_VARCHAR, collation=-46), const_bytes(b"___", -46), collation=-46),
                                                                 like(col(M_STR, tp=ffi.TP_VARCHAR, collation=-46), const_bytes(b"_%z", -46), collation=-46))).build(output_offsets=[M_H, M_STR, M_INT])),
            ("mixed_sel_like_blob_escape", scan().selection(not_(like(col(M_BLOB, tp=ffi.TP_BLOB, collation=63), const_bytes(b"%!%%"), escape=ord("!")))).build(output_offsets=[M_H, M_BLOB])),
            ("mixed_count_like_prefix", scan().selection(like(col(M_STR, tp=ffi.TP_VARCHAR, collation=63), const_bytes(b"a%"))).aggregation([("count", const_int(1))]).build()),
            # DECIMAL comparisons (impl_compare.rs over `Ord for Decimal`): column vs constant in several (precision, fraction)
            # shapes, IN with a NULL, IS NULL, column vs itself
            ("mixed_sel_decimal_lt", scan().selection(lt(col(M_DEC, tp=ffi.TP_NEWDECIMAL), const_decimal(kvfmt.decimal_bin("0.5", 3, 2)))).build(output_offsets=[M_H, M_DEC])),
            ("mixed_sel_decimal_ge_big", scan().selection(ge(col(M_DEC, tp=ffi.TP_NEWDECIMAL), const_decimal(kvfmt.decimal_bin("1000000000.000000001", 30, 9)))).build(output_offsets=[M_H, M_DEC, M_STR])),
            ("mixed_sel_decimal_in_null", scan().selection(or_(is_null(col(M_DEC, tp=ffi.TP_NEWDECIMAL)),
                                                               in_(col(M_DEC, tp=ffi.TP_NEWDECIMAL), const_decimal(kvfmt.decimal_bin("0", 1, 0)), null(ffi.TP_NEWDECIMAL),
                                                                   const_decimal(kvfmt.decimal_bin("-0.00000", 5, 5))))).build(output_offsets=[M_H, M_DEC])),
            ("mixed_count_decimal_eq_self", scan().selection(eq(col(M_DEC, tp=ffi.TP_NEWDECIMAL), col(M_DEC, tp=ffi.TP_NEWDECIMAL)), ne(col(M_DEC, tp=ffi.TP_NEWDECIMAL), const_decimal(kvfmt.decimal_bin("7", 1, 0))))
                                                  .aggregation([("count", const_int(1))]).build()),
            ("mixed_count_nulleq_duration", scan().selection(nulleq(col(M_DUR, tp=ffi.TP_DURATION), const_duration(1))).aggregation([("count", const_int(1))]).build()),
            ("mixed_count_zero_dates", scan().selection(eq(col(M_DT, tp=ffi.TP_DATETIME), const_time(0))).aggregation([("count", const_int(1)), ("count", col(M_INT))]).build()),
            ("mixed_only_strings", scan().build(output_offsets=[M_STR, M_BLOB, M_JSON]))]


# The reference's own 12-column row (row/v2/encoder_for_test.rs:560-588 `test_encode`): the expected bytes of that test
# are the stored row value here; the values are the ones the test encodes.
REF_MIXED_ROW = bytes([
    128, 0, 11, 0, 1, 0, 1, 3, 6, 7, 8, 9, 12, 13, 14, 15, 16, 33, 2, 0, 3, 0, 11, 0, 14, 0, 16, 0, 24, 0, 25, 0, 33, 0, 36, 0, 65, 0, 69, 0, 232, 3, 3, 64, 3, 51, 51, 51, 51,
    51, 50, 97, 98, 99, 255, 127, 191, 252, 204, 204, 204, 204, 204, 205, 2, 0, 0, 0, 135, 51, 230, 158, 25, 1, 0, 129, 1, 1, 0, 0, 0, 28, 0, 0, 0, 19, 0, 0, 0, 3, 0, 12, 22, 0,
    0, 0, 107, 101, 121, 5, 118, 97, 108, 117, 101, 0, 202, 154, 59])
REF_MIXED_COLUMNS = [ColumnDef(1), ColumnDef(12), ColumnDef(33), ColumnDef(3, unsigned=True), ColumnDef(8), ColumnDef(7, tp=ffi.TP_VARCHAR), ColumnDef(9, tp=ffi.TP_DOUBLE),
                     ColumnDef(6, tp=ffi.TP_DOUBLE), ColumnDef(13, tp=ffi.TP_DATETIME), ColumnDef(14, tp=ffi.TP_NEWDECIMAL), ColumnDef(15, tp=ffi.TP_JSON),
                     ColumnDef(16, tp=ffi.TP_DURATION), ColumnDef(100, pk_handle=True)]
REF_MIXED_JSON = bytes([1, 1, 0, 0, 0, 28, 0, 0, 0, 19, 0, 0, 0, 3, 0, 12, 22, 0, 0, 0, 107, 101, 121, 5, 118, 97, 108, 117, 101])  # {"key":"value"}
REF_MIXED_VALUES = (1000, 2, None, 3, 32767, b"abc", 1.8, -1.8, kvfmt.time_bits(2018, 1, 19, 3, 14, 7), 1, REF_MIXED_JSON, 10 ** 9, 7)


def ref_mixed_region():
    r = kvfmt.Region()
    r.put(kvfmt.row_key(TABLE, 7), REF_MIXED_ROW, 10, 20)
    return r


def check_mixed(run, seed=1, n_keys=700):
    """Every mixed_plans() result of `run(plan, ranges, region)` equals the oracle's, cell for cell."""
    import orc
    region = mixed_region(seed, n_keys).build(read_ts=READ_TS, n_write_blocks=2)
    for name, plan in mixed_plans():
        exp = orc.dag_handle(plan, WHOLE, region)
        got = run(plan, WHOLE, region)
        assert exp.status == 0 and exp.n_rows > (0 if "count" in name else (25 if "like" in name else 50)), (name, exp.status, exp.message)
        if "count" in name:
            assert exp.rows()[0][0] > 2, (name, exp.rows())
        assert got.status == 0, (name, got.status, got.message)
        assert got.kinds == exp.kinds, (name, got.kinds, exp.kinds)
        assert got.rows() == exp.rows(), name
