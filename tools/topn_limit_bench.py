"""TopN request time against LIMIT, on one GPU: the C4 table and ORDER BY of bench.py at LIMIT 1000 .. 4096 (both sides
of the 2048 switch to HBM candidate buffers), and the reference benchmark's three `limit_large` shapes at LIMIT 4000
next to their LIMIT 10 twins, over tables built row by row (the region generator makes at most 24 columns).

Every arm's rows are first checked against tests/topn_ref.py: on a 1M-row prefix of the C4 table, over the whole of the
others.  The arms then run alternately
(round-robin, --rounds times); the median ms per request is reported.  One extra profiled request per arm splits out the
device time of the merge kernels (topn_rank_merge / topn_merge2 / topn_copy) and of the payload gather (topn_gather).
Prints one JSON object with the card's name and power limit.

Usage: python tools/topn_limit_bench.py [--rows 100000000] [--ref-rows 200000] [--rounds 5] [--out FILE]"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import bench  # noqa: E402
import kvfmt  # noqa: E402
import scenarios as sc  # noqa: E402
import topn_ref  # noqa: E402
from test_gpu_parity import _source  # noqa: E402
from tikv_b200 import ffi  # noqa: E402
from tikv_b200.executor import BatchExecutor, DeviceRegion  # noqa: E402
from tikv_b200.plan import ColumnDef, Plan, col, const_int, gt, is_null  # noqa: E402

T = sc.TABLE
PREFIX = 1_000_000  # rows of the C4 table checked against topn_ref before timing


class Table:
    """The C4 table of bench.py (gen_blocks, 8 regions as in its C4 record) and the spec topn_ref.gen_rows restates."""

    def __init__(self, n_rows):
        n_cols, lo, rng, nulls = bench.TABLES["c4"]
        self.spec = dict(n_cols=n_cols, seed=bench.SEED, lo=lo, rng=rng, nulls=nulls)
        self.gens, self.blks = bench.gen_blocks(ffi, 0, "c4", n_rows, 8)
        self.src = _source([b.block for b in self.blks], ffi.LOC_DEVICE)

    def free(self):
        for g in self.gens:
            ffi.lib().b2_gen_destroy(g)


def built_table(n_rows, n_cols, seed, null_pct=0):
    """id + n_cols random full-range i64 columns (col1 NULL in null_pct % of rows), built row by row: (rows, HBM region)."""
    rnd = random.Random(seed)
    r, rows = kvfmt.Region(), []
    for h in range(n_rows):
        vals = [rnd.randrange(-(1 << 63), 1 << 63) for _ in range(n_cols)]
        if rnd.randrange(100) < null_pct:
            vals[0] = None
        r.put(kvfmt.row_key(T, h), kvfmt.row_v2([(c + 1, v, "int") for c, v in enumerate(vals)]), 10, 20)
        rows.append((h,) + tuple(vals))
    return rows, DeviceRegion(r.build(read_ts=sc.READ_TS))


def run(plan, ranges, src):
    with BatchExecutor(plan, ranges, src) as ex:
        rows = []
        while True:
            b = ex.next_batch(1 << 30)
            if b.error is not None:
                raise RuntimeError(b.error.message)
            rows += b.rows()
            if b.is_drained:
                return rows


def timed(plan, src):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(plan, sc.WHOLE, src)  # (next_batch returns after the stream has finished)
    return (time.perf_counter() - t0) * 1e3


def profiled(plan, src):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(plan, sc.WHOLE, src)
        torch.cuda.synchronize()
    merge = gather = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if "topn_gather" in e.key:
            gather += us
        elif "topn_rank_merge" in e.key or "topn_merge2" in e.key or "topn_copy" in e.key:
            merge += us
    return merge / 1e3, gather / 1e3


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # the name from torch, the power limit unknown
        return f"{torch.cuda.get_device_name(0)}, power limit not read ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000, help="rows of the C4 table")
    ap.add_argument("--ref-rows", type=int, default=200_000, help="rows of the 3-column table of the reference shapes (the 50-column one has a tenth)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"

    c4 = Table(args.rows)
    rows3, src3 = built_table(args.ref_rows, 2, 0x1F83D9AB, null_pct=30)
    rows50, src50 = built_table(args.ref_rows // 10, 49, 0x5BE0CD19)
    c4_cols = [ColumnDef(100, pk_handle=True), ColumnDef(1), ColumnDef(2)]
    c4_order = [(1, True), (2, False)]
    order3 = [(is_null(col(1)), False), (col(1), False), (col(2), True)]
    keys3 = [(lambda r: int(r[1] is None), False, "int"), (1, False, "int"), (2, True, "int")]
    cols50 = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(49)]
    bound = args.ref_rows // 2
    g4 = topn_ref.gen_rows(c4.spec, [(0, PREFIX)])
    c4_want = lambda n: [(int(g4["handle"][i]),) + tuple(None if g4["null"][i, c] else int(g4["vals"][i, c]) for c in range(2))
                         for i in topn_ref.topn_indices([(g4["vals"][:, o - 1], g4["null"][:, o - 1], d) for o, d in c4_order], n)]
    # name -> (source, plan, the key range the check reads, expected rows there, limit)
    arms = {}
    for limit in (1000, 2048, 2049, 4000, 4096):
        arms[f"c4/limit{limit}"] = (c4.src, Plan().table_scan(bench.TABLE_ID, c4_cols).topn([(col(o), d) for o, d in c4_order], limit).build(),
                                    [kvfmt.table_range(T, 0, PREFIX)], c4_want, limit)
    for limit in (10, 4000):
        arms[f"order_by_3_col/limit{limit}"] = (src3, Plan().table_scan(T, c4_cols).topn(order3, limit).build(), sc.WHOLE,
                                                lambda n: topn_ref.expected_topn(rows3, keys3, n), limit)
        arms[f"where_order_by_3_col/limit{limit}"] = (src3, Plan().table_scan(T, c4_cols).selection(gt(col(0), const_int(bound))).topn(order3, limit).build(), sc.WHOLE,
                                                      lambda n: topn_ref.expected_topn([r for r in rows3 if r[0] > bound], keys3, n), limit)
        arms[f"50_col_order_by_1_col/limit{limit}"] = (src50, Plan().table_scan(T, cols50).topn([(col(1), False)], limit).build(), sc.WHOLE,
                                                       lambda n: topn_ref.expected_topn(rows50, [(1, False, "int")], n), limit)

    checked, failed = {}, {}
    for name, (src, plan, rng, want_of, limit) in arms.items():
        want = want_of(limit)
        try:
            got = run(plan, rng, src)
        except RuntimeError as e:  # reported, and the arm is not timed
            failed[name] = str(e)
            continue
        if got != want:  # reported with the first difference, and the arm is not timed
            i = next((k for k, (a, b) in enumerate(zip(got, want)) if a != b), min(len(got), len(want)))
            failed[name] = f"rows differ from topn_ref: {len(got)} vs {len(want)} rows, first at {i}: " \
                           f"{got[i] if i < len(got) else None} vs {want[i] if i < len(want) else None}"
            continue
        checked[name] = len(got)

    plans = {name: (src, plan) for name, (src, plan, _, _, _) in arms.items() if name in checked}
    for src, plan in plans.values():  # warm-up: module loads, plan-specialised kernels, pools
        run(plan, sc.WHOLE, src)
    times = {name: [] for name in plans}
    for _ in range(args.rounds):
        for name, (src, plan) in plans.items():
            times[name].append(timed(plan, src))
    res = {}
    for name, (src, plan) in plans.items():
        m, gth = profiled(plan, src)
        res[name] = {"ms_per_request": round(statistics.median(times[name]), 3), "ms_all": [round(x, 3) for x in times[name]],
                     "merge_ms": round(m, 3), "gather_ms": round(gth, 3), "rows_checked": checked[name]}
    out = {"card": card(), "c4_rows": args.rows, "ref_rows": args.ref_rows, "rounds": args.rounds,
           "timing": "host clock around a drained request (median of alternating rounds); merge / gather: device time of one profiled request",
           "arms": res, "failed": failed}
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")
    c4.free()


if __name__ == "__main__":
    main()
