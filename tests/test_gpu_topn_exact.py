"""`-m gpu`: TopN on the device against the exact reference of topn_ref.py, every cell of every row, in order.

Generated tables at about 2M rows per block (clean, and dirty: extra versions, Deletes, lock records and NULLs that send
runs to the list-mode kernel while the lean kernel takes the rest of the same chunks), rows whose MVCC runs straddle
the first chunk boundaries of a unit, Int / unsigned / Real value edges, and sort keys after the first that fail or
warn on rows the CTA's bound would drop.  Ties go to the row scanned first (b2_device.h item_less), so every row is
determined and a payload taken from the wrong list or chunk shows up as a wrong cell."""
import math
import random
import struct

import numpy as np
import pytest

import kvfmt
import orc
import scenarios as sc
import topn_ref
from test_gpu_parity import _block_to_host, _gen_block, _source
from tikv_b200 import ffi
from tikv_b200.executor import BatchExecutor, DeviceRegion
from tikv_b200.plan import ColumnDef, Plan, cast_int_as_real, col, const_int, const_real, divide, in_, multiply

pytestmark = pytest.mark.gpu

T = sc.TABLE
I64_MAX = (1 << 63) - 1


def _columns(n_cols):
    return [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(n_cols)]


def _run(plan, ranges, region, jit=None):
    """Drain one request: (rows, error or None, warning count, exec stats)."""
    kw = {} if jit is None else dict(jit=jit)
    with BatchExecutor(plan, ranges, region, **kw) as ex:
        rows, err = [], None
        while True:
            b = ex.next_batch(1 << 22)
            rows += b.rows()
            if b.error is not None:
                err = b.error
                break
            if b.is_drained:
                break
        return rows, err, ex.warnings()[0], ex.collect_exec_stats()


def _same_as_oracle(plan, ranges, host, got, ctx, sort_key=None):
    """Status, MySQL code, rows, warning count and processed keys equal the oracle's.  sort_key: where rows tie on every
    sort key, compare only these (the oracle's heap keeps an arbitrary one of the tied rows)."""
    rows, err, warns, st = got
    exp = orc.dag_handle(plan, ranges, host)
    assert (err.status if err else 0) == exp.status, f"{ctx}: status {err and (err.status, err.message)} != oracle {exp.status} ({exp.message})"
    assert (err.mysql_code if err else 0) == exp.mysql_code, ctx
    assert warns == exp.warning_count, f"{ctx}: {warns} warnings != oracle {exp.warning_count}"
    if exp.status == 0:
        assert [sort_key(r) for r in rows] == [sort_key(r) for r in exp.rows()] if sort_key else rows == exp.rows(), ctx
        assert st.write_processed_keys == exp.stats["processed_keys"], ctx
    return exp


def _gen_table_rows(g, idx):
    """Rows (handle, c1, ...) of gen_rows output `g` at indices `idx`; None = NULL."""
    h, v, nl = g["handle"][idx], g["vals"][idx], g["null"][idx]
    return [(int(h[i]),) + tuple(None if nl[i, c] else int(v[i, c]) for c in range(v.shape[1])) for i in range(len(idx))]


class _Gen:
    """Generated blocks in HBM (b2_gen_create) and their reference rows; the blocks are freed at teardown."""

    def __init__(self, spec, blocks, fmt=2):
        self.spec, self.gens, self.blks = spec, [], []
        for first, n in blocks:
            g, blk = _gen_block(n, spec["n_cols"], fmt, spec["seed"], spec.get("lo"), spec.get("rng"), spec.get("nulls"),
                                extra=spec.get("extra", 0), delete=spec.get("delete", 0), lockrec=spec.get("lockrec", 0), first_handle=first)
            self.gens.append(g); self.blks.append(blk)
        self.rows = topn_ref.gen_rows(spec, blocks)
        assert [b.block.n for b in self.blks] == self.rows["n_entries"]
        self.dev = _source([b.block for b in self.blks], ffi.LOC_DEVICE)
        self._host = None

    def host(self):
        if self._host is None:
            copies = [_block_to_host(b) for b in self.blks]
            self._host = (_source([hb for hb, _ in copies], ffi.LOC_HOST), copies)
        return self._host[0]

    def key_arrays(self, order):
        """[(values, nulls, desc)] of sort keys given as (column offset, desc); offset 0 is the handle."""
        g = self.rows
        return [(g["handle"], None, d) if o == 0 else (g["vals"][:, o - 1], g["null"][:, o - 1], d) for o, d in order]

    def free(self):
        for g in self.gens:
            ffi.lib().b2_gen_destroy(g)


# ---- 1. the reference is trustworthy ------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [2, 1])
def test_generated_rows_match_oracle_scan(fmt):
    """gen_rows == the oracle's MVCC scan of a D2H copy of the generated block, cell for cell, and each row's first
    CF_WRITE entry holds the row's key (its predecessor another key)."""
    spec = dict(n_cols=6, seed=0x6A09E667F3BCC909, lo=[0, -500, 0, 7, 0, -(1 << 40)], rng=[0, 1000, 3, 1, 1 << 20, 1 << 41],
                nulls=[0, 30000, 0, 0, 0, 10000], extra=200000, delete=50000, lockrec=50000)
    gen = _Gen(spec, [(-7, 20000)], fmt=fmt)
    try:
        hb, (keys, _vals, koff, _voff) = _block_to_host(gen.blks[0])
        host = _source([hb], ffi.LOC_HOST)
        exp = orc.dag_handle(Plan().table_scan(T, _columns(6)).build(), sc.WHOLE, host)
        g = gen.rows
        assert exp.status == 0 and 0.9 * 20000 < exp.n_rows < 0.97 * 20000
        assert exp.rows() == _gen_table_rows(g, np.arange(len(g["handle"])))
        # memcomparable row key: the handle's 8 big-endian bytes are key bytes 12..16 and 18..20 (after a group marker)
        starts = koff[:-1].astype(np.int64)
        hb8 = np.stack([keys[starts + i] for i in (12, 13, 14, 15, 16, 18, 19, 20)], axis=1)
        key_handle = (hb8.astype(np.uint64) << np.arange(56, -1, -8, dtype=np.uint64)).sum(axis=1, dtype=np.uint64) ^ np.uint64(1 << 63)
        key_handle = key_handle.view(np.int64)
        assert np.array_equal(key_handle[g["entry"]], g["handle"])
        prev = g["entry"][g["entry"] > 0] - 1
        assert np.all(key_handle[prev] != key_handle[prev + 1])
    finally:
        gen.free()


# ---- 2. scale: ~6M rows, both kernels, every limit up to 2048 ----------------------------------------------------------
N_BLOCK = 2_000_000
SCALE_BLOCKS = [(i * N_BLOCK, N_BLOCK) for i in range(3)]
# c1 full-range i64, c2 narrow [-500, 500), c3 [0, 3), c4 always 7, c5 [0, 2^20)
SCALE_SPEC = dict(n_cols=5, lo=[0, -500, 0, 7, 0], rng=[0, 1000, 3, 1, 1 << 20])
ORDERS = {
    "full_desc_narrow": [(1, True), (2, False)],
    "handle_desc": [(0, True)],  # forward: every row beats the bound, each chunk replaces the running list
    "handle_asc": [(0, False)],  # the bound is tight after the first chunk
    "range1_first": [(4, False), (2, True)],  # every row ties on the first key: the prefilter passes them all
    "range3_handle_desc": [(3, False), (0, True)],
    "four_keys": [(3, True), (2, False), (5, True), (1, False)],
}
LIMITS = [1, 255, 256, 257, 1000, 2047, 2048]


def _scale_ranges(g):
    """Five ranges that split blocks: across a block boundary, a one-row range, an empty one, a long one inside the
    first block, and the table's last rows."""
    one = int(g["handle"][np.searchsorted(g["handle"], 3 * N_BLOCK // 2)])
    return [(N_BLOCK - 1000, N_BLOCK + 1500), (one, one + 1), (4_500_000, 4_500_000), (100, 1_500_000), (3 * N_BLOCK - 700, 3 * N_BLOCK + 10)]


@pytest.fixture(scope="module")
def scale_sets():
    sets = {}
    try:
        sets["clean"] = _Gen(dict(SCALE_SPEC, seed=0x3C6EF372FE94F82B), SCALE_BLOCKS)
        sets["dirty"] = _Gen(dict(SCALE_SPEC, seed=0xA54FF53A5F1D36F1, nulls=[0, 10000, 0, 0, 0], extra=200000, delete=50000, lockrec=50000), SCALE_BLOCKS)
        yield sets
    finally:
        for s in sets.values():
            s.free()


def _topn_plan(n_cols, order, limit, desc):
    return Plan().table_scan(T, _columns(n_cols), desc=desc).topn([(col(o), d) for o, d in order], limit).build()


@pytest.mark.parametrize("desc", [False, True], ids=["forward", "backward"])
@pytest.mark.parametrize("order", list(ORDERS), ids=list(ORDERS))
@pytest.mark.parametrize("which", ["clean", "dirty"])
def test_topn_at_scale(which, order, desc, scale_sets):
    gen = scale_sets[which]
    g = gen.rows
    perm = topn_ref.topn_indices(gen.key_arrays(ORDERS[order]), len(g["handle"]), desc_scan=desc)  # the whole order, best first
    for limit in LIMITS:
        plan = _topn_plan(5, ORDERS[order], limit, desc)
        rows, err, _, _ = _run(plan, sc.WHOLE, gen.dev)
        assert err is None, (err.status, err.message)
        assert rows == _gen_table_rows(g, perm[:limit]), f"{which}/{order}/limit{limit}"
    for lo, hi in _scale_ranges(g):
        inside = (g["handle"] >= lo) & (g["handle"] < hi)
        sub = perm[inside[perm]]
        for limit in (257, 2048):
            rows, err, _, _ = _run(_topn_plan(5, ORDERS[order], limit, desc), [kvfmt.table_range(T, lo, hi)], gen.dev)
            assert err is None and rows == _gen_table_rows(g, sub[:limit]), f"{which}/{order}/[{lo},{hi})/limit{limit}"


@pytest.mark.parametrize("which", ["clean", "dirty"])
def test_topn_at_scale_plan_specialised_and_host_resident(which, scale_sets):
    """The run-time compiled kernels (JIT_SYNC) on the widest sort keys, and one request over host-resident blocks."""
    gen = scale_sets[which]
    g = gen.rows
    for order in ("full_desc_narrow", "four_keys"):
        for desc in (False, True):
            perm = topn_ref.topn_indices(gen.key_arrays(ORDERS[order]), 2048, desc_scan=desc)
            for limit in (1000, 2048):
                rows, err, _, st = _run(_topn_plan(5, ORDERS[order], limit, desc), sc.WHOLE, gen.dev, jit=ffi.JIT_SYNC)
                assert err is None and rows == _gen_table_rows(g, perm[:limit]), f"jit/{which}/{order}/desc{desc}/limit{limit}"
                assert st.jit_launches > 0
    if which == "dirty":
        perm = topn_ref.topn_indices(gen.key_arrays(ORDERS["full_desc_narrow"]), 1000)
        rows, err, _, _ = _run(_topn_plan(5, ORDERS["full_desc_narrow"], 1000, False), sc.WHOLE, gen.host())
        assert err is None and rows == _gen_table_rows(g, perm), "host-resident"


# ---- 3. MVCC runs across chunk boundaries --------------------------------------------------------------------------------
def _straddling_seed(spec, n_rows, b1, b2):
    """First seed whose block has a 3-entry run (extra versions) across entry `b1` and a 2-entry run (lock record over
    the visible Put) across `b2`."""
    for seed in range(1, 5000):
        g = topn_ref.gen_rows(dict(spec, seed=seed), [(0, n_rows)])
        e = g["entry"]  # (no Deletes in `spec`: the entry gap to the next row is the row's own run)
        i1, i2 = np.searchsorted(e, b1, "right") - 1, np.searchsorted(e, b2, "right") - 1
        if e[i1] < b1 and e[i1 + 1] - e[i1] == 3 and e[i2] == b2 - 1 and e[i2 + 1] - e[i2] == 2:
            return seed, int(g["handle"][i1]), int(g["handle"][i2])
    raise AssertionError("no seed found")


@pytest.mark.parametrize("desc", [False, True], ids=["forward", "backward"])
def test_runs_straddling_chunk_boundaries(desc):
    n_rows = 60_000
    spec = dict(n_cols=3, lo=[0, -500, 0], rng=[0, 1000, 3], extra=200000, lockrec=100000)
    n_entries = topn_ref.gen_rows(dict(spec, seed=1), [(0, n_rows)])["n_entries"][0]  # (about: only the boundaries below matter)
    starts, _ = topn_ref.chunk_bounds(0, n_entries)
    b1, b2 = starts[1], starts[2]
    seed, h1, h2 = _straddling_seed(spec, b2 + 100, b1, b2)
    gen = _Gen(dict(spec, seed=seed), [(0, n_rows)])
    try:
        g = gen.rows
        starts, _ = topn_ref.chunk_bounds(0, g["n_entries"][0])
        assert starts[1:3] == [b1, b2] and len(starts) >= 3
        hit = np.isin(g["handle"], [h1, h2]).astype(np.int64)
        for limit in (2, 10, 2048):
            order = [(in_(col(0), const_int(h1), const_int(h2)), True), (col(2), False), (col(0), desc)]
            plan = Plan().table_scan(T, _columns(3), desc=desc).topn(order, limit).build()
            want = _gen_table_rows(g, topn_ref.topn_indices([(hit, None, True), (g["vals"][:, 1], None, False), (g["handle"], None, desc)], limit, desc))
            assert {want[0][0], want[1][0]} == {h1, h2}
            got = _run(plan, sc.WHOLE, gen.dev)
            assert got[1] is None and got[0] == want, f"limit{limit}"
            _same_as_oracle(plan, sc.WHOLE, gen.host(), got, f"straddle/limit{limit}")
    finally:
        gen.free()


# ---- 4. value edges: Real, unsigned and signed sort keys -----------------------------------------------------------------
REAL_EDGES = [0.0, -0.0, math.inf, -math.inf, 1.7976931348623157e308, -1.7976931348623157e308, 5e-324, -5e-324, 1.0,
              math.nextafter(1.0, 2.0), math.nan, None]
UINT_EDGES = [0, I64_MAX, 1 << 63, (1 << 64) - 1]
INT_EDGES = [-(1 << 63), -1, 0, I64_MAX]
EDGE_COLS = [ColumnDef(100, pk_handle=True), ColumnDef(1, tp=ffi.TP_DOUBLE), ColumnDef(2, unsigned=True), ColumnDef(3), ColumnDef(4)]


@pytest.fixture(scope="module")
def edge_region():
    """50k keys, v1 and v2 rows: a Real, an unsigned and a signed column over their edge values (±0.0 half the
    time, so zeros tie across the cut), and a small grouping column; three or more chunks in the one unit."""
    rng = random.Random(4242)
    r = kvfmt.Region()
    for h in range(50_000):
        real = rng.choice((0.0, -0.0)) if rng.random() < 0.5 else rng.choice(REAL_EDGES)
        u, i, grp = rng.choice(UINT_EDGES), rng.choice(INT_EDGES), rng.randrange(50)
        if rng.random() < 0.5:
            row = kvfmt.row_v2([(1, real, "f64"), (2, u, "uint"), (3, i, "int"), (4, grp, "int")])
        else:
            row = kvfmt.row_v1([(1, kvfmt.datum_null() if real is None else kvfmt.datum_f64(real)), (2, kvfmt.datum_uint(u)),
                                (3, kvfmt.datum_int(i)), (4, kvfmt.datum_int(grp))])
        r.put(kvfmt.row_key(T, h * 2 - 30_000), row, 10, 20)
    host = r.build(read_ts=sc.READ_TS)
    assert len(topn_ref.chunk_bounds(0, host.wblocks[0].n)[0]) >= 3
    return host, DeviceRegion(host)


EDGE_ORDERS = {
    "real_asc": [(1, False, "real"), (0, False, "int")],
    "real_desc": [(1, True, "real")],
    "grp_real_asc": [(4, False, "int"), (1, False, "real")],
    "grp_real_desc": [(4, True, "int"), (1, True, "real")],
    "uint_asc": [(2, False, "uint")],
    "grp_uint_desc": [(4, False, "int"), (2, True, "uint")],
    "int_asc": [(3, False, "int")],
    "grp_int_desc": [(4, True, "int"), (3, True, "int")],
}


@pytest.mark.parametrize("desc", [False, True], ids=["forward", "backward"])
@pytest.mark.parametrize("order", list(EDGE_ORDERS), ids=list(EDGE_ORDERS))
def test_value_edges(order, desc, edge_region):
    host, dev = edge_region
    scan = orc.dag_handle(Plan().table_scan(T, EDGE_COLS).build(), sc.WHOLE, host)
    assert scan.status == 0 and scan.n_rows == 50_000
    keys = EDGE_ORDERS[order]
    for limit in (1, 100, 2048):
        plan = Plan().table_scan(T, EDGE_COLS, desc=desc).topn([(col(o, tp=ffi.TP_DOUBLE if k == "real" else ffi.TP_LONGLONG, unsigned=k == "uint"), d)
                                                                for o, d, k in keys], limit).build()
        want = topn_ref.expected_topn(scan.rows(), keys, limit, desc_scan=desc)
        for region in (dev, host):
            got = _run(plan, sc.WHOLE, region)
            assert got[1] is None, got[1].message
            # bit for bit: -0.0 stays -0.0 in the payload, NaN came back as NULL
            assert [tuple(struct.pack("<d", x) if isinstance(x, float) else x for x in r) for r in got[0]] == \
                   [tuple(struct.pack("<d", x) if isinstance(x, float) else x for x in r) for r in want], f"{order}/limit{limit}"
        if limit == 2048:
            _same_as_oracle(plan, sc.WHOLE, host, got, f"{order}/limit{limit}", sort_key=lambda r: tuple(r[o] for o, _, _ in keys))


# ---- 5. errors and warnings in later sort keys ---------------------------------------------------------------------------
ERR_ROWS = 1_000_000


def _error_case():
    """Seed, multiplier K and handle: c_b * K overflows on exactly one row, whose c_a loses against the 10 smallest,
    which lies past the first three chunks of a forward scan and of a backward one, and whose c3 is NULL when the
    table has NULLs in c3 (50 %)."""
    spec = dict(n_cols=3, lo=[0, 0, 0], rng=[1 << 40, 1 << 40, 100])
    for seed in range(1, 500):
        g = topn_ref.gen_rows(dict(spec, seed=seed, nulls=[0, 0, 500000]), [(0, ERR_ROWS)])
        ca, cb = g["vals"][:, 0], g["vals"][:, 1]
        top2 = np.argsort(cb)[-2:]
        i = int(top2[1])
        K = I64_MAX // int(cb[i]) + 1
        starts, _ = topn_ref.chunk_bounds(0, g["n_entries"][0])
        middle = starts[3] <= g["entry"][i] < g["n_entries"][0] - starts[3]
        if middle and int(cb[top2[0]]) * K <= I64_MAX and ca[i] > np.sort(ca)[10] and g["null"][i, 2]:
            return spec, seed, K, int(g["handle"][i])
    raise AssertionError("no seed found")


@pytest.fixture(scope="module")
def error_tables():
    spec, seed, K, h = _error_case()
    gens = {}
    try:
        gens["lean"] = _Gen(dict(spec, seed=seed), [(0, ERR_ROWS)])
        gens["list"] = _Gen(dict(spec, seed=seed, nulls=[0, 0, 500000]), [(0, ERR_ROWS)])
        yield gens, K, h
    finally:
        for x in gens.values():
            x.free()


@pytest.mark.parametrize("desc", [False, True], ids=["forward", "backward"])
@pytest.mark.parametrize("path", ["lean", "list"])
def test_later_sort_key_overflow_fails_the_request(path, desc, error_tables):
    """ORDER BY c_a, c_b * K LIMIT 10: one row's product overflows, and its c_a can never make the top 10.  The reference
    evaluates every sort key of every row, so the request fails with ER_DATA_OUT_OF_RANGE (1690) on whichever kernel
    meets that row: the lean one (all cells present) or the list-mode one (the row has a NULL cell)."""
    gens, K, h = error_tables
    gen = gens[path]
    assert gen.rows["null"][gen.rows["handle"] == h, 2][0] == (path == "list")
    plan = Plan().table_scan(T, _columns(3), desc=desc).topn([(col(1), False), (multiply(col(2), const_int(K)), False)], 10).build()
    jits = (None, ffi.JIT_SYNC) if path == "lean" and not desc else (None,)
    for jit in jits:
        got = _run(plan, sc.WHOLE, gen.dev, jit=jit)
        assert got[1] is not None and got[1].status == ffi.B2_ERR_EVALUATE and got[1].mysql_code == 1690, \
            f"{path}: status {got[1] and got[1].status}, expected B2_ERR_EVALUATE / 1690"
    _same_as_oracle(plan, sc.WHOLE, gen.host(), got, f"overflow/{path}")
    # the same plan without the overflowing row: the 10 smallest c_a
    ok = _run(plan, [kvfmt.table_range(T, 0, h), kvfmt.table_range(T, h + 1, ERR_ROWS)], gen.dev)
    g = gen.rows
    keep = g["handle"] != h
    want = topn_ref.topn_indices([(g["vals"][keep, 0], None, False), (g["vals"][keep, 1], None, False)], 10, desc)
    assert ok[1] is None and ok[0] == _gen_table_rows({k: v[keep] for k, v in g.items() if k != "n_entries"}, want)


@pytest.mark.parametrize("desc", [False, True], ids=["forward", "backward"])
@pytest.mark.parametrize("path", ["lean", "list"])
def test_sort_key_warnings_count_every_row(path, desc, error_tables):
    """x / 0.0 in a sort key is NULL with warning 1365 once per row and key evaluation, as in the reference: in a later
    key (rows the bound drops warn too) and in the first key (candidates evaluate it once, not twice)."""
    gens, _, _ = error_tables
    gen = gens[path]
    zero = lambda c: divide(cast_int_as_real(col(c)), const_real(0.0))
    for name, order in (("later", [(col(1), False), (zero(2), False)]), ("first", [(zero(1), True), (col(2), False)])):
        plan = Plan().table_scan(T, _columns(3), desc=desc).topn(order, 10).build()
        got = _run(plan, sc.WHOLE, gen.dev)
        exp = _same_as_oracle(plan, sc.WHOLE, gen.host(), got, f"warnings/{name}/{path}")
        assert exp.warning_count == len(gen.rows["handle"]), name
