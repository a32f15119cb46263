"""The TopN reference of topn_ref.py pinned down on the CPU: against the oracle on the shared TopN plans, forward and
backward, and its numpy mixer against the scalar formula."""
import numpy as np
import pytest

import orc
import scenarios as sc
import topn_ref
from tikv_b200.plan import Plan

C_H, C1, C2, C3, C4, C6 = sc.C_H, sc.C1, sc.C2, sc.C3, sc.C4, sc.C6


def _sum(r):
    return None if r[C6] is None or r[C2] is None else r[C6] + r[C2]


# sort keys, limit, row filter and output offsets of each plan of sc.topn_plans()
KEYS = {
    "topn_two_keys": ([(C2, True, "int"), (C1, False, "int")], 50, None, None),
    "topn_real_desc_handle": ([(C4, True, "real"), (C_H, False, "int")], 30, None, None),
    "topn_expr": ([(_sum, False, "int"), (C_H, True, "int")], 40, None, None),
    "topn_all_rows": ([(C1, False, "int"), (C_H, False, "int")], 2000, None, None),
    "topn_all_rows_ties": ([(C1, False, "int")], 2000, None, None),
    "topn_zero": ([(C1, False, "int")], 0, None, None),
    "topn_after_filter": ([(C1, True, "int")], 25, lambda r: r[C6] < 8, [C1, C6, C_H]),
    "topn_unsigned_ties": ([(C3, False, "uint")], 20, None, None),
    "topn_small_domain_ties": ([(C6, True, "int"), (C2, False, "int")], 60, None, None),
}


@pytest.fixture(scope="module")
def regions():
    return {seed: sc.dirty_region(seed, n_keys=900).build(read_ts=sc.READ_TS, n_write_blocks=3) for seed in (1, 2)}


@pytest.mark.parametrize("desc", [False, True], ids=["forward", "backward"])
def test_reference_matches_oracle_on_topn_plans(desc, regions):
    assert sorted(KEYS) == sorted(t[0] for t in sc.topn_plans())
    for seed, ranges in ((1, sc.WHOLE), (2, sc.split_ranges())):
        region = regions[seed]
        scan = orc.dag_handle(Plan().table_scan(sc.TABLE, sc.COLUMNS).build(), ranges, region)
        assert scan.status == 0 and scan.n_rows > 500
        for name, plan, exact, key_cols in sc.topn_plans(desc=desc):
            keys, limit, keep, offsets = KEYS[name]
            rows = [r for r in scan.rows() if keep is None or keep(r)]
            want = topn_ref.expected_topn(rows, keys, limit, desc_scan=desc)
            if offsets:
                want = [tuple(r[o] for o in offsets) for r in want]
            exp = orc.dag_handle(plan, ranges, region)
            assert exp.status == 0 and exp.n_rows == len(want) == min(limit, len(rows)), name
            if exact:
                assert exp.rows() == want, f"{name}/seed{seed}"
            else:
                assert [tuple(r[c] for c in key_cols) for r in exp.rows()] == [tuple(r[c] for c in key_cols) for r in want], name


def test_ties_go_to_the_row_scanned_first():
    rows = [(h, h % 3, None if h % 5 == 0 else float(h % 2) - 0.5, -0.0 if h % 2 else 0.0) for h in range(30)]
    fwd = topn_ref.expected_topn(rows, [(1, False, "int")], 4)
    assert [r[0] for r in fwd] == [0, 3, 6, 9]
    bwd = topn_ref.expected_topn(rows, [(1, True, "int")], 4, desc_scan=True)
    assert [r[0] for r in bwd] == [29, 26, 23, 20]
    # NULL before any value ascending, after every value descending; -0.0 ties with 0.0
    assert [r[0] for r in topn_ref.expected_topn(rows, [(2, False, "real")], 3)] == [0, 5, 10]
    assert [r[0] for r in topn_ref.expected_topn(rows, [(2, True, "real")], 2)] == [1, 3]
    assert [r[0] for r in topn_ref.expected_topn(rows, [(3, True, "real")], 3, desc_scan=True)] == [29, 28, 27]
    big = [(0, (1 << 64) - 1), (1, 1 << 63), (2, 0), (3, (1 << 63) - 1)]
    assert [r[0] for r in topn_ref.expected_topn(big, [(1, False, "uint")], 4)] == [2, 3, 1, 0]


def test_numpy_mixer_matches_the_scalar_formula():
    from test_gpu_parity import _gen_mix
    edges = [0, 1, 2, 255, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, (1 << 64) - 2, (1 << 64) - 1]
    handles = np.array(edges, dtype=np.uint64)
    for seed in (0, 99, 0x525C682A2F7CE3DB, (1 << 64) - 1):
        for salt in (0, 1, 7, 500, 503, 1000):
            got = topn_ref.gen_mix(seed, handles, salt)
            assert [int(x) for x in got] == [_gen_mix(seed, h, salt) for h in edges] == [topn_ref.gen_mix_scalar(seed, h, salt) for h in edges]


def test_chunk_bounds_follow_the_engine_rule():
    starts, seeded = topn_ref.chunk_bounds(0, 600_000)
    assert starts[:3] == [0, 16 * topn_ref.TILE, 16 * topn_ref.TILE * 8] and seeded == 600_000
    assert all(b > a for a, b in zip(starts, starts[1:]))
    assert topn_ref.chunk_bounds(10, 20, seeded_rows=10 ** 6) == ([10], 10 ** 6 + 10)
