"""Cost of the FIRST and BIT_* aggregates on the C3 table (bench.py's headline table and size), one process, arms
alternating step by step:

  c3            SUM(val) GROUP BY key WHERE val < 0                     (bench.py's C3)
  c3_first      C3 + FIRST(val)
  c3_bit_xor    C3 + BIT_XOR(val)
  c3_count      C3 + COUNT(val)          (older kinds of the same state width, for comparison)
  c3_max        C3 + MAX(val)
  bit_or_nokey  BIT_OR(val) WHERE val < 0, no GROUP BY
  first_nokey   FIRST(val) WHERE val < 0, no GROUP BY

Each arm is first checked against the reference on a prefix of the table (the oracle's rows, aggregated as the reference
defines FIRST / BIT_*).  Prints one JSON line per arm and one summary line with the GPU name and power limit, read in the
same call.  Usage: python tools/agg_kinds_bench.py [--rows N] [--blocks B] [--steps K] [--warmup W]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def specs():
    import bench
    from first_bit_ref import Spec
    from tikv_b200 import ffi
    from tikv_b200.plan import ColumnDef, col, const_int, lt
    cols = [ColumnDef(100, pk_handle=True), ColumnDef(1, tp=ffi.TP_LONG), ColumnDef(2)]
    sel = [lt(col(2), const_int(0))]
    key = [(1, {"tp": ffi.TP_LONG})]
    S = lambda aggs, by: Spec(bench.TABLE_ID, cols, aggs, by, sel)
    return {"c3": S([("sum", 2, {})], key), "c3_first": S([("sum", 2, {}), ("first", 2, {})], key),
            "c3_bit_xor": S([("sum", 2, {}), ("bit_xor", 2, {})], key),
            # the same width with the older kinds: COUNT adds one CTA-table atomic per row, as BIT_XOR does; MAX adds two
            "c3_count": S([("sum", 2, {}), ("count", 2, {})], key), "c3_max": S([("sum", 2, {}), ("max", 2, {})], key),
            "bit_or_nokey": S([("bit_or", 2, {})], []), "first_nokey": S([("first", 2, {})], [])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500_000_000)
    ap.add_argument("--blocks", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--parity-rows", type=int, default=1_000_000)
    args = ap.parse_args()
    if not os.environ.get("B2_JIT_CACHE_DIR"):  # kernels compiled here go to a temporary directory, as in bench.py
        import atexit
        import shutil
        import tempfile
        jit_tmp = tempfile.mkdtemp(prefix="b2_jit_cache_")
        atexit.register(shutil.rmtree, jit_tmp, True)
        os.environ["B2_JIT_CACHE_DIR"] = jit_tmp
    import ctypes as C
    import threading
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    import bench
    from tikv_b200 import ffi
    from tikv_b200.executor import DagHandler
    L = ffi.lib()
    arms = specs()
    plans = {n: s.plan() for n, s in arms.items()}
    # every arm runs its plan-specialised kernels from the first timed step on (prepared like bench.py's plans)
    prep = {}
    ths = [threading.Thread(target=lambda n=n: prep.__setitem__(n, L.b2_plan_prepare(C.byref(plans[n].c), 0))) for n in plans]
    [t.start() for t in ths]
    [t.join() for t in ths]
    assert not any(prep.values()), prep
    gens, blks = bench.gen_blocks(ffi, 0, "c3", args.rows, args.blocks)
    src = bench.Source(ffi, [b.block for b in blks], ffi.LOC_DEVICE, 0)
    try:
        # parity on a prefix: the oracle over host-generated rows of the same handles
        arm = bench.CpuArm("c3", args.parity_rows, 1, 1, first_handle=0)
        rng = bench.table_range(0, args.parity_rows)
        parity = {}
        for n, s in arms.items():
            got = DagHandler(plans[n], rng, src).handle_request()
            s.check(got, rng, bench._Src(arm.source()), n)
            parity[n] = got.n_rows
        arm.close()
        whole = bench.table_range()
        times = {n: [] for n in arms}
        launches = {}
        for step in range(args.warmup + args.steps):
            for n in arms:  # alternating arms
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                _, st = bench.run_dag(ffi, plans[n], whole, src, ffi.LOC_DEVICE, 1 << 24)
                torch.cuda.synchronize()
                if step >= args.warmup:
                    times[n].append(time.perf_counter() - t0)
                    launches[n] = (st.jit_launches, st.kernel_launches)
        info = gpu_info()
        med = {n: sorted(t)[len(t) // 2] for n, t in times.items()}
        for n in arms:
            print(json.dumps({"arm": n, "rows": args.rows, "median_ms": round(med[n] * 1e3, 3), "rows_per_s": args.rows / med[n],
                              "min_ms": round(min(times[n]) * 1e3, 3), "max_ms": round(max(times[n]) * 1e3, 3),
                              "vs_c3": round(med["c3"] / med[n], 4), "parity_groups": parity[n],
                              "specialised_launches": launches[n][0], "kernel_launches": launches[n][1], "gpu": info}))
        print(json.dumps({"gpu": info, "steps": args.steps, "c3_first_vs_c3": round(med["c3"] / med["c3_first"], 4)}))
    finally:
        for g in gens:
            ffi.lib().b2_gen_destroy(g)


if __name__ == "__main__":
    main()
