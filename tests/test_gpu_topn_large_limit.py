"""`-m gpu`: TopN with LIMIT 2049..4096 on the device, every cell of every row, in order, against topn_ref.py and the oracle.

Above LIMIT 2048 a CTA's candidate buffer (capacity 8192) lives in HBM in both TopN kernels (engine.cu run_topn).  The
cases below cover the generated ~6M-row sets of test_gpu_topn_exact.py at the large limits, tables on which every
scanned row is a candidate so that CTAs of both kernels must compact their HBM buffers mid-launch, the reference's own
LIMIT 4000 benchmark shapes, errors and warnings in sort keys, and the merge of several regions' partial results."""
import random

import numpy as np
import pytest
import torch

import kvfmt
import orc
import scenarios as sc
import topn_ref
from test_gpu_parity import _one_batch
from test_gpu_topn_exact import ORDERS, SCALE_BLOCKS, SCALE_SPEC, _Gen, _gen_table_rows, _run, _same_as_oracle, _scale_ranges, _topn_plan
from test_gpu_topn_exact import error_tables  # noqa: F401  (the fixture of the error tables, shared)
from tikv_b200 import dist as bd
from tikv_b200 import ffi
from tikv_b200.executor import DeviceRegion
from tikv_b200.plan import ColumnDef, Plan, cast_int_as_real, col, const_int, const_real, divide, gt, is_null, multiply

pytestmark = pytest.mark.gpu

T = sc.TABLE
LIMITS = [2049, 3000, 4000, 4095, 4096]
CAP = 8192  # engine.cu run_topn: a CTA's candidate capacity above LIMIT 2048


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


# ---- 1. the generated sets at the large limits -------------------------------------------------------------------------
@pytest.mark.parametrize("desc", [False, True], ids=["forward", "backward"])
@pytest.mark.parametrize("order", list(ORDERS), ids=list(ORDERS))
@pytest.mark.parametrize("which", ["clean", "dirty"])
def test_large_limits_at_scale(which, order, desc, scale_sets):
    gen = scale_sets[which]
    g = gen.rows
    perm = topn_ref.topn_indices(gen.key_arrays(ORDERS[order]), len(g["handle"]), desc_scan=desc)
    for limit in LIMITS:
        rows, err, _, _ = _run(_topn_plan(5, ORDERS[order], limit, desc), sc.WHOLE, gen.dev)
        assert err is None, (err.status, err.message)
        assert rows == _gen_table_rows(g, perm[:limit]), f"{which}/{order}/limit{limit}"
    for lo, hi in _scale_ranges(g):
        inside = (g["handle"] >= lo) & (g["handle"] < hi)
        sub = perm[inside[perm]]
        rows, err, _, _ = _run(_topn_plan(5, ORDERS[order], 4096, desc), [kvfmt.table_range(T, lo, hi)], gen.dev)
        assert err is None and rows == _gen_table_rows(g, sub[:4096]), f"{which}/{order}/[{lo},{hi})"


@pytest.mark.parametrize("which", ["clean", "dirty"])
def test_large_limits_plan_specialised_and_host_resident(which, scale_sets):
    gen = scale_sets[which]
    g = gen.rows
    for order in ("full_desc_narrow", "four_keys"):
        for desc in (False, True):
            perm = topn_ref.topn_indices(gen.key_arrays(ORDERS[order]), 4096, desc_scan=desc)
            for limit in (2049, 4096):
                rows, err, _, st = _run(_topn_plan(5, ORDERS[order], limit, desc), sc.WHOLE, gen.dev, jit=ffi.JIT_SYNC)
                assert err is None and rows == _gen_table_rows(g, perm[:limit]), f"jit/{which}/{order}/desc{desc}/limit{limit}"
                assert st.jit_launches > 0
    if which == "dirty":
        perm = topn_ref.topn_indices(gen.key_arrays(ORDERS["full_desc_narrow"]), 4000)
        rows, err, _, _ = _run(_topn_plan(5, ORDERS["full_desc_narrow"], 4000, False), sc.WHOLE, gen.host())
        assert err is None and rows == _gen_table_rows(g, perm), "host-resident"


# ---- 2. compaction of the HBM buffers, in both kernels -------------------------------------------------------------------
N_COMPACT = 8_000_000
LEAN_CTAS_PER_SM, GENERAL_CTAS_PER_SM = 3, 2  # the most either TopN kernel fits on an SM (launch bounds / shared memory)
# clean: the lean kernel takes every row; dirty: rows with a NULL in c1 (60 %) go to the general kernel in list mode;
# wide: nine value columns, which the lean kernel does not decode, so the general kernel scans whole chunks
COMPACT_SETS = {
    "clean": dict(n_cols=2, lo=[0, 0], rng=[1000, 1000]),
    "dirty": dict(n_cols=2, lo=[0, 0], rng=[1000, 1000], nulls=[600000, 0]),
    "wide": dict(n_cols=9, lo=[0] * 9, rng=[1000] * 9),
}


@pytest.mark.parametrize("which", list(COMPACT_SETS))
def test_every_row_a_candidate_compacts_in_hbm(which):
    """ORDER BY handle DESC: a unit's chunks are scanned from its lower end in both scan directions (engine.cu run_topn),
    so every chunk holds larger handles than all before it and each CTA's buffer takes every row it scans.  The largest
    chunk hands more than CAP rows to each CTA of the kernel that scans them, so CTAs compact mid-launch, not only at
    the end."""
    spec = dict(COMPACT_SETS[which], seed=0x510E527FADE682D1)
    gen = _Gen(spec, [(0, N_COMPACT)])
    try:
        g = gen.rows
        starts, _ = topn_ref.chunk_bounds(0, g["n_entries"][0])
        ends = starts[1:] + [g["n_entries"][0]]
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        lo, hi = max(zip(starts, ends), key=lambda b: b[1] - b[0])
        in_chunk = (g["entry"] >= lo) & (g["entry"] < hi)
        if which == "clean":
            per_cta = in_chunk.sum() / (LEAN_CTAS_PER_SM * sms)
        elif which == "dirty":
            per_cta = (in_chunk & g["null"][:, 0]).sum() / (GENERAL_CTAS_PER_SM * sms)
        else:
            per_cta = in_chunk.sum() / (GENERAL_CTAS_PER_SM * sms)
        assert per_cta > CAP, f"{which}: {per_cta:.0f} candidates per CTA in the largest chunk do not force a compaction"
        n_cols = spec["n_cols"]
        for desc in (False, True):
            order = [(0, True)]
            want = _gen_table_rows(g, topn_ref.topn_indices(gen.key_arrays(order), 4096, desc_scan=desc))
            for jit in (None, ffi.JIT_SYNC):
                rows, err, _, _ = _run(_topn_plan(n_cols, order, 4096, desc), sc.WHOLE, gen.dev, jit=jit)
                assert err is None and rows == want, f"{which}/desc{desc}/jit{jit}"
    finally:
        gen.free()


# ---- 3. the reference's LIMIT 4000 benchmark shapes ----------------------------------------------------------------------
REF_ROWS = 200_000


class _Built:
    """A hand-built region (kvfmt) where the generator's 24 columns are too few: host copy and HBM copy."""

    def __init__(self, host):
        self._h, self.dev = host, DeviceRegion(host)

    def host(self):
        return self._h

    def free(self):
        pass


def _fifty_columns(n_rows):
    """id + 49 value columns of random i64 values, row format v2."""
    rng = random.Random(0x5BE0CD19)
    r = kvfmt.Region()
    for h in range(n_rows):
        r.put(kvfmt.row_key(T, h), kvfmt.row_v2([(c + 1, rng.randrange(-(1 << 63), 1 << 63), "int") for c in range(49)]), 10, 20)
    return _Built(r.build(read_ts=sc.READ_TS))


@pytest.fixture(scope="module")
def ref_tables():
    """id + col1 (NULL in 30 % of rows) + col2, full-range random values; and id + 49 value columns."""
    t = {}
    try:
        t["3col"] = _Gen(dict(n_cols=2, seed=0x1F83D9ABFB41BD6B, nulls=[300000, 0]), [(0, REF_ROWS)])
        t["50col"] = _fifty_columns(12_000)
        yield t
    finally:
        for x in t.values():
            x.free()


def _ref_shapes():
    cols3 = [ColumnDef(100, pk_handle=True), ColumnDef(1), ColumnDef(2)]
    order3 = lambda: [(is_null(col(1)), False), (col(1), False), (col(2), True)]
    cols50 = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(49)]
    return {
        "order_by_3_col": ("3col", lambda n: Plan().table_scan(T, cols3).topn(order3(), n).build()),
        "where_order_by_3_col": ("3col", lambda n: Plan().table_scan(T, cols3).selection(gt(col(0), const_int(REF_ROWS // 2))).topn(order3(), n).build()),
        "50_col_order_by_1_col": ("50col", lambda n: Plan().table_scan(T, cols50).topn([(col(1), False)], n).build()),
    }


@pytest.mark.parametrize("shape", list(_ref_shapes()))
def test_reference_limit_large_shapes(shape, ref_tables):
    table, mk = _ref_shapes()[shape]
    gen = ref_tables[table]
    host = gen.host()
    # the whole table (NULLs sort last under isnull(col1) and do not reach the top 4000), and 5000 rows around the
    # WHERE bound, among which they do
    for ranges in (sc.WHOLE, [kvfmt.table_range(T, REF_ROWS // 2 - 1000, REF_ROWS // 2 + 4000)] if table == "3col" else [kvfmt.table_range(T, 3000, 8000)]):
        for limit in (10, 4000):
            plan = mk(limit)
            got = _run(plan, ranges, gen.dev)
            assert got[1] is None, got[1].message
            exp = _same_as_oracle(plan, ranges, host, got, f"{shape}/limit{limit}")
            assert 0 < exp.n_rows <= limit and (exp.n_rows == limit or ranges is not sc.WHOLE)
            if table == "3col" and ranges is not sc.WHOLE and limit == 4000 and shape == "order_by_3_col":
                assert any(r[1] is None for r in got[0]) and got[0][0][1] is not None  # NULL col1 rows made it, last
            ex = _one_batch(plan, ranges, gen.dev)
            try:
                assert ex.encode_batch(ffi.ENCODE_TYPE_CHUNK) == exp.encoded[1], f"{shape}/limit{limit}: chunk bytes"
            finally:
                ex.close()


# ---- 4. errors and warnings in sort keys under LIMIT 4096 ----------------------------------------------------------------
@pytest.mark.parametrize("desc", [False, True], ids=["forward", "backward"])
@pytest.mark.parametrize("path", ["lean", "list"])
def test_later_sort_key_overflow_fails_at_limit_4096(path, desc, error_tables):  # noqa: F811
    gens, K, h = error_tables
    gen = gens[path]
    plan = Plan().table_scan(T, [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(3)], desc=desc) \
        .topn([(col(1), False), (multiply(col(2), const_int(K)), False)], 4096).build()
    got = _run(plan, sc.WHOLE, gen.dev)
    assert got[1] is not None and got[1].status == ffi.B2_ERR_EVALUATE and got[1].mysql_code == 1690, got[1] and got[1].message
    _same_as_oracle(plan, sc.WHOLE, gen.host(), got, f"overflow/{path}")


@pytest.mark.parametrize("path", ["lean", "list"])
def test_sort_key_warnings_count_every_row_at_limit_4096(path, error_tables):  # noqa: F811
    gens, _, _ = error_tables
    gen = gens[path]
    zero = lambda c: divide(cast_int_as_real(col(c)), const_real(0.0))
    cols = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(3)]
    for name, order in (("later", [(col(1), False), (zero(2), False)]), ("first", [(zero(1), True), (col(2), False)])):
        plan = Plan().table_scan(T, cols).topn(order, 4096).build()
        got = _run(plan, sc.WHOLE, gen.dev)
        exp = _same_as_oracle(plan, sc.WHOLE, gen.host(), got, f"warnings/{name}/{path}", sort_key=lambda r: (r[1],) if name == "later" else (r[2],))
        assert exp.warning_count == len(gen.rows["handle"]), name


# ---- 5. several regions' partial results merged ----------------------------------------------------------------------------
def test_region_partials_merge_at_4096(scale_sets):
    """Each of four ranges (regions) is a request of its own; their device results go through dist.merge_topn, which
    must give the TopN of the union."""
    gen = scale_sets["dirty"]
    g = gen.rows
    order = ORDERS["full_desc_narrow"]
    bounds = [(-1, 1_000_000), (1_000_000, 2_600_000), (2_600_000, 5_999_000), (5_999_000, 7_000_000)]
    cols, nulls = None, None
    for lo, hi in bounds:
        rows, err, _, _ = _run(_topn_plan(5, order, 4096, False), [kvfmt.table_range(T, lo, hi)], gen.dev)
        in_range = int(((g["handle"] >= lo) & (g["handle"] < hi)).sum())
        assert err is None and len(rows) == min(4096, in_range)
        c = [torch.tensor([0 if r[j] is None else r[j] for r in rows], dtype=torch.int64) for j in range(6)]
        n = [torch.tensor([r[j] is None for r in rows], dtype=torch.bool) for j in range(6)]
        cols = c if cols is None else [torch.cat([a, b]) for a, b in zip(cols, c)]
        nulls = n if nulls is None else [torch.cat([a, b]) for a, b in zip(nulls, n)]
    mc, mn = bd.merge_topn(cols, nulls, [(o, d, "i64") for o, d in order], 4096)
    got = [tuple(None if mn[j][i] else int(mc[j][i]) for j in range(6)) for i in range(mc[0].shape[0])]
    inside = np.zeros(len(g["handle"]), dtype=bool)
    for lo, hi in bounds:
        inside |= (g["handle"] >= lo) & (g["handle"] < hi)
    perm = topn_ref.topn_indices(gen.key_arrays(order), len(g["handle"]))
    assert got == _gen_table_rows(g, perm[inside[perm]][:4096])
