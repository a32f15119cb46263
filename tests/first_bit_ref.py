"""Reference results for FIRST and BIT_AND / BIT_OR / BIT_XOR aggregation plans.

The oracle executes the scan (and selection) of a plan and returns its rows in scan order; the aggregates are then
applied here as the reference defines them:
  FIRST  (impl_first.rs AggrFnStateFirst::update / push_result): the argument of the first row of the group, NULL
         included; no row -> NULL
  BIT_*  (impl_bit_op.rs BitOp::init_state, AggrFnStateBitOp): u64 state from !0 / 0 / 0, NULL arguments skipped, never NULL
Every other aggregate of a plan is checked against the oracle running the plan without the new aggregates.
Values are compared as bits (u64 for integers, IEEE bits for doubles): -0.0 and NaN payloads must survive unchanged."""
import struct

import kvfmt
import orc
import scenarios as sc
from tikv_b200 import ffi
from tikv_b200.plan import ColumnDef, Plan, col, const_int, lt

U64 = (1 << 64) - 1
NEW_KINDS = ("first", "bit_and", "bit_or", "bit_xor")
WIDTH = {"count": 1, "sum": 1, "avg": 2, "min": 1, "max": 1, "first": 1, "bit_and": 1, "bit_or": 1, "bit_xor": 1}


def bits(v):
    if v is None:
        return None
    if isinstance(v, float):
        return ("f", struct.unpack("<Q", struct.pack("<d", v))[0])
    return ("i", v & U64)


def _group_key(vals, fast_hash):
    out = []
    for v in vals:
        if fast_hash and isinstance(v, float) and v == 0.0:
            v = 0.0  # the fast hash executor groups -0.0 with 0.0
        out.append(bits(v))
    return tuple(out)


def fold(kind, values):
    """The aggregate of `values` (python ints / floats / None, in scan order) as the reference computes it."""
    if kind == "first":
        return values[0] if values else None
    acc = {"bit_and": U64, "bit_or": 0, "bit_xor": 0}[kind]
    for v in values:
        if v is None:
            continue
        v &= U64
        acc = acc & v if kind == "bit_and" else (acc | v if kind == "bit_or" else acc ^ v)
    return acc


class Spec:
    """An aggregation over plain column arguments and plain column group keys.  cols: the table's ColumnDefs;
    aggs: [(kind, column offset, col kwargs)]; group_by: [(column offset, col kwargs)]."""

    def __init__(self, table, cols, aggs, group_by=(), selection=(), desc=False):
        self.table, self.cols, self.aggs, self.group_by = table, cols, list(aggs), list(group_by)
        self.selection, self.desc = list(selection), desc

    def _scan(self):
        p = Plan().table_scan(self.table, self.cols, desc=self.desc)
        return p.selection(*self.selection) if self.selection else p

    def _agg(self, aggs):
        from tikv_b200.plan import col
        return self._scan().aggregation([(k, col(c, **kw)) for k, c, kw in aggs],
                                        group_by=[col(c, **kw) for c, kw in self.group_by]).build()

    def plan(self):
        return self._agg(self.aggs)

    def old_aggs(self):
        return [a for a in self.aggs if a[0] not in NEW_KINDS]

    def expected(self, ranges, region):
        """{group key: [normalised output cells of every aggregate, in plan order]}: new aggregates from the scan rows,
        the others from the oracle."""
        scan = orc.dag_handle(self._scan().build(), ranges, region)
        assert scan.status == 0, scan.message
        fast_hash = len(self.group_by) == 1
        groups = {}
        for row in scan.rows():
            groups.setdefault(_group_key([row[c] for c, _ in self.group_by], fast_hash), []).append(row)
        if not self.group_by and not groups:
            groups[()] = []  # aggregation without GROUP BY answers one row even over no input
        out = {k: [] for k in groups}
        old = {}
        if self.old_aggs():
            res = orc.dag_handle(self._agg(self.old_aggs()), ranges, region)
            assert res.status == 0, res.message
            n_old = sum(WIDTH[a[0]] for a in self.old_aggs())
            for r in res.rows():
                old[_group_key(r[n_old:], fast_hash)] = list(r[:n_old])
            assert set(old) == set(groups), "oracle groups differ from the scan's"
        for k, rows in groups.items():
            pos = 0
            for kind, c, _ in self.aggs:
                if kind in NEW_KINDS:
                    out[k].append(bits(fold(kind, [r[c] for r in rows])))
                else:
                    out[k] += [bits(v) for v in old[k][pos:pos + WIDTH[kind]]]
                    pos += WIDTH[kind]
        return out

    def got(self, result):
        n = sum(WIDTH[a[0]] for a in self.aggs)
        fast_hash = len(self.group_by) == 1
        out = {}
        for r in result.rows():
            k = _group_key(r[n:], fast_hash)
            assert k not in out, f"group {k} answered twice"
            out[k] = [bits(v) for v in r[:n]]
        return out

    def check(self, result, ranges, region, ctx=""):
        assert result.status == 0, f"{ctx}: {getattr(result, 'message', '')}"
        exp, got = self.expected(ranges, region), self.got(result)
        assert set(got) == set(exp), f"{ctx}: groups differ: {len(got)} vs {len(exp)}"
        for k in exp:
            assert got[k] == exp[k], f"{ctx}: group {k}: {got[k]} != {exp[k]}"
        return exp


I64, UNS, REAL, LONG = {}, {"unsigned": True}, {"tp": ffi.TP_DOUBLE}, {"tp": ffi.TP_LONG}


def scenario_specs(desc):
    """(name, Spec) over sc.COLUMNS: C1 full-range i64, C2 small nullable i64, C3 u64 (0, 1, 2^63, 2^64-1 ...), C4 f64 with
    NULL / 0.0 / -0.0, C5 nullable with a default, C6 small key."""
    S = lambda aggs, by=(), sel=(): Spec(sc.TABLE, sc.COLUMNS, aggs, by, sel, desc)
    return [
        ("first_nokey", S([("first", sc.C1, I64)])),
        ("bits_nokey", S([("bit_and", sc.C2, I64), ("bit_or", sc.C3, UNS), ("bit_xor", sc.C1, I64)])),
        ("first_real_nokey", S([("first", sc.C4, REAL), ("count", sc.C2, I64), ("first", sc.C2, I64)])),
        ("mixed_key_c6", S([("first", sc.C2, I64), ("sum", sc.C1, I64), ("bit_xor", sc.C3, UNS), ("max", sc.C1, I64), ("count", sc.C5, I64),
                            ("first", sc.C4, REAL)], [(sc.C6, LONG)])),
        ("nullable_key", S([("first", sc.C1, I64), ("bit_and", sc.C2, I64), ("bit_or", sc.C5, I64)], [(sc.C2, I64)])),
        ("real_key", S([("first", sc.C3, UNS), ("bit_or", sc.C1, I64), ("min", sc.C2, I64)], [(sc.C4, REAL)])),
        ("two_keys", S([("first", sc.C1, I64), ("bit_and", sc.C3, UNS), ("count", sc.C1, I64)], [(sc.C2, I64), (sc.C6, LONG)])),
        ("four_keys", S([("first", sc.C4, REAL), ("bit_xor", sc.C2, I64), ("max", sc.C1, I64)], [(sc.C2, I64), (sc.C6, LONG), (sc.C3, UNS), (sc.C4, REAL)])),
        ("filtered", S([("bit_or", sc.C2, I64), ("first", sc.C5, I64), ("avg", sc.C6, I64)], [(sc.C6, LONG)], [lt(col(sc.C1), const_int(0))])),
    ]


# tests/integrations/coprocessor/test_select.rs test_aggr_first and test_aggr_bit_ops, with the VARCHAR column `name`
# ("name:N") restated as an INT column holding N (NULL stays NULL): the reference's expected rows apply unchanged.
SELECT_COLS = [ColumnDef(100, pk_handle=True), ColumnDef(1), ColumnDef(2)]  # id, name, count
ID, NAME, COUNT = range(3)
FIRST_ROWS = [(1, 0, 2), (2, 3, 3), (3, 5, 3), (4, 0, 1), (5, 5, 4), (6, 5, 4), (7, None, 4), (8, None, 5), (9, 5, 5), (10, None, 6)]
BIT_ROWS = [(1, 0, 2), (2, 3, 3), (4, 0, 1), (5, 5, 4), (6, 5, 5), (7, None, 4), (8, 5, None), (9, 6, None)]


def select_region(rows, n_write_blocks=1):
    r = kvfmt.Region()
    for i, name, count in rows:
        r.put(kvfmt.row_key(sc.TABLE, i), kvfmt.row_v2([(1, name, "int"), (2, count, "int")]), 10, 20)
    return r.build(read_ts=sc.READ_TS, n_write_blocks=n_write_blocks)


def select_cases(desc=False):
    """(name, rows, Spec, {group key: expected cells}) with the reference's expected answers (forward scans; a backward
    scan keeps the BIT_* answers and takes the last row of each group for FIRST)."""
    k = lambda v: (bits(v),)
    cells = lambda *vs: [bits(v) for v in vs]
    first_id = {k(None): cells(7), k(0): cells(1), k(3): cells(2), k(5): cells(3)}
    first_name = {k(5): cells(None), k(6): cells(None), k(2): cells(0), k(1): cells(0), k(3): cells(3), k(4): cells(5)}
    if desc:
        first_id = {k(None): cells(10), k(0): cells(4), k(3): cells(2), k(5): cells(9)}
        first_name = {k(5): cells(5), k(6): cells(None), k(2): cells(0), k(1): cells(0), k(3): cells(5), k(4): cells(None)}
    return [("first_id_by_name", FIRST_ROWS, Spec(sc.TABLE, SELECT_COLS, [("first", ID, I64)], [(NAME, I64)], (), desc), first_id),
            ("first_name_by_count", FIRST_ROWS, Spec(sc.TABLE, SELECT_COLS, [("first", NAME, I64)], [(COUNT, I64)], (), desc), first_name),
            ("bit_ops_by_name", BIT_ROWS, Spec(sc.TABLE, SELECT_COLS, [("bit_and", COUNT, I64), ("bit_or", COUNT, I64), ("bit_xor", COUNT, I64)],
                                               [(NAME, I64)], (), desc),
             {k(None): cells(4, 4, 4), k(0): cells(0, 3, 3), k(3): cells(3, 3, 3), k(5): cells(4, 5, 1), k(6): cells(-1, 0, 0)})]
