"""GPU measurement: the C3 request end to end from RocksDB data blocks laid out as a compacted region (one sorted run)
against the same visible state laid out as a live LSM store (several sorted runs with shadowed versions, tombstones and
entries above the snapshot) merged on the device.

Setup (untimed): the C3 table generated as `--regions` regions.  Per region:
  compacted  the region's block as one run (b2_sst_encode, bench.sst_e2e's block sizing: ~32 KiB blocks, restart
             interval 16, 'z' prefix, internal-key footer, trailer), in pinned host memory
  lsm        the same rows split on the device (tests/sstmerge.device_lsm) into four small L0 runs (new keys, puts over
             older versions, puts / deletions above the snapshot), an L5 run (about a tenth of the keys at higher seqs,
             and tombstones over extra keys whose puts sit below them) and a bottom run at seq 0 holding the rest;
             every run encoded the same way with the footers it carries, in pinned host memory
  lsm_dev    the lsm runs already in HBM (B2_LOC_DEVICE)
The merging read of each lsm region at its snapshot is exactly the compacted region.  Timed, alternating arms within
each round: one step = every region decoded (b2_sst_decode) or merged (b2_sst_merge), two threads as bench.py overlaps
them, + the C3 request over the resulting blocks, result to the host.  Then, in a separate profiled pass
(torch.profiler, CUDA activities), the device time of each kernel per step.  Prints one JSON object (and writes it to
--out when given).

  python tools/sst_merge_bench.py [--rows 70000000] [--regions 7] [--rounds 3] [--steps 3] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import sstmerge  # noqa: E402
from tikv_b200 import ffi  # noqa: E402
from tikv_b200.executor import DagHandler, SstDecoder  # noqa: E402

KERNELS = ("sst_blocks", "sst_inflate", "sst_zstd", "sst_count", "sst_expand", "sst_stage", "sst_iota", "sst_visible", "sst_gather", "merge")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or "unknown (nvidia-smi: %s)" % q.stderr.strip()[:200]


def encode(L, dev, flat, per, suffix, keep):
    """flat device block -> (pinned host data, offsets, device copy of the data)"""
    import torch
    h, enc = C.c_void_p(), ffi.SstEncoded()
    assert L.b2_sst_encode(dev, C.byref(flat), per, 16, 1, ord("z"), suffix, 5, C.byref(h), C.byref(enc)) == 0, L.b2_last_error_message()
    p = L.b2_host_alloc_pinned_near(dev, enc.data_len + 64)
    offs = np.zeros(enc.n_blocks + 1, dtype=np.uint64)
    assert p and L.b2_copy_to_host(dev, p, enc.data, enc.data_len) == 0 and L.b2_copy_to_host(dev, offs.ctypes.data, enc.block_offs, 8 * len(offs)) == 0
    L.b2_sst_free(h)
    keep.append(p)
    t = torch.from_numpy(np.frombuffer(C.string_at(p, enc.data_len) + b"\0" * 16, dtype=np.uint8).copy()).to(dev)
    return p, offs, t, enc.data_len


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=70_000_000)
    ap.add_argument("--regions", type=int, default=7)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs cuda:0"
    L = ffi.lib()
    dev = 0
    info = gpu_info()
    plan = bench.build_plan("c3")
    gens, blks = bench.gen_blocks(ffi, dev, "c3", args.rows, args.regions)
    rows = sum(b.n_user_keys for b in blks)
    keep, compacted, lsm, lsm_dev, snaps = [], [], [], [], []
    compacted_bytes = lsm_bytes = lsm_entries = 0
    t0 = time.time()
    for b in blks:
        per = max(16, 32768 // max(8, int((b.key_bytes + b.val_bytes) / max(1, b.block.n)) - 9))  # (bench.sst_e2e's sizing)
        p, offs, _, n = encode(L, dev, b.block, per, 8, keep)
        compacted.append((p, offs))
        compacted_bytes += n
        runs, snap = sstmerge.device_lsm(b, n_l0=4)
        host_runs, dev_runs = [], []
        for keys, koff, vals, voff, cnt in runs:
            flat = ffi.CfBlock()
            flat.keys, flat.key_offs, flat.vals, flat.val_offs, flat.n = keys.data_ptr(), koff.data_ptr(), vals.data_ptr(), voff.data_ptr(), cnt
            p, offs, t, n = encode(L, dev, flat, per, 0, keep)
            host_runs.append((p, offs))
            dev_runs.append((t, offs))
            lsm_bytes += n
            lsm_entries += cnt
        del runs
        torch.cuda.empty_cache()
        lsm.append(host_runs)
        lsm_dev.append(dev_runs)
        snaps.append(snap)
    setup_s = time.time() - t0
    decs = [SstDecoder(dev) for _ in blks]
    arms = ("compacted", "lsm", "lsm_dev")
    src_keep = []
    with ThreadPoolExecutor(max_workers=2) as pool:  # two regions in flight, as bench.py's data-block record
        def one(arm, r):
            if arm == "compacted":
                return decs[r].decode(*compacted[r])
            runs = lsm[r] if arm == "lsm" else [(t.data_ptr(), o) for t, o in lsm_dev[r]]
            return decs[r].merge(runs, snaps[r], location=ffi.LOC_HOST if arm == "lsm" else ffi.LOC_DEVICE)

        def decode_all(arm):
            res = list(pool.map(lambda r: one(arm, r), range(len(blks))))
            src = bench.Source(ffi, [blk for blk, _ in res], ffi.LOC_DEVICE, dev)
            src_keep.append(src)
            return src, res

        def step(arm):
            src, res = decode_all(arm)
            bench.run_dag(ffi, plan, bench.table_range(), src, ffi.LOC_HOST, 1 << 20)
            return res

        results = {}
        for arm in arms:  # warm-up, and each arm's C3 result (rows sorted: the group order of a hash table is not fixed)
            step(arm)
            src, res = decode_all(arm)
            r = DagHandler(plan, bench.table_range(), src).handle_request()
            assert r.status == 0, r.message
            results[arm] = (sorted(zip(*r.columns)), sum(st.h2d_bytes for _, st in res), res)
        identical = all(results[a][0] == results["compacted"][0] for a in arms)
        merge_stats = {k: sum(getattr(st, k) for _, st in results["lsm"][2]) for k in ("n_in", "n_out", "n_invisible", "n_hidden", "n_deletions")}
        assert merge_stats["n_out"] == sum(b.block.n for b in blks)
        times = {a: [] for a in arms}
        for _ in range(args.rounds):
            for arm in arms:
                torch.cuda.synchronize()
                t = time.perf_counter()
                for _ in range(args.steps):
                    step(arm)
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t) * 1e3 / args.steps)
        events = {a: {"decode_ms": round(sum(st.decode_ms for _, st in decode_all(a)[1]), 2)} for a in arms}
        for a in ("lsm", "lsm_dev"):
            events[a]["merge_ms"] = round(sum(st.merge_ms for _, st in decode_all(a)[1]), 2)

        from torch.profiler import ProfilerActivity, profile
        kern = {}
        for arm in ("compacted", "lsm_dev"):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    decode_all(arm)
                torch.cuda.synchronize()
            k = {}
            for e in prof.key_averages():
                if e.device_time_total <= 0:
                    continue
                name = next((n for n in KERNELS if n in e.key), "cub_scan" if "DeviceScan" in e.key or "scan" in e.key.lower() else None)
                if name is None and "Memcpy" in e.key:
                    name = "memcpy " + ("DtoD" if "DtoD" in e.key else ("HtoD" if "HtoD" in e.key else "DtoH"))
                if name:
                    k[name] = k.get(name, 0.0) + e.device_time_total / 1e3 / args.steps
            kern[arm] = {n: round(v, 3) for n, v in sorted(k.items())}
    for d in decs:
        d.close()
    for p in keep:
        L.b2_host_free_pinned(p)
    for g in gens:
        L.b2_gen_destroy(g)
    compacted_decode = sum(v for n, v in kern["compacted"].items() if n.startswith(("sst_", "cub")))
    lsm_dev_total = sum(v for n, v in kern["lsm_dev"].items() if not n.startswith("memcpy"))
    out = {"gpu": info, "rows": rows, "regions": args.regions, "rounds": args.rounds, "steps_per_round": args.steps, "setup_s": round(setup_s, 1),
           "compacted_run_bytes": compacted_bytes, "lsm_run_bytes": lsm_bytes, "lsm_entries": lsm_entries, "runs_per_region": 6, "merge_stats_per_step": merge_stats,
           "arms": {a: {"ms_per_step_median": round(statistics.median(v), 2), "ms_per_step_range": [round(min(v), 2), round(max(v), 2)],
                        "rows_per_s_median": rows / (statistics.median(v) / 1e3), "h2d_bytes_per_step": results[a][1], **events[a]} for a, v in times.items()},
           "kernel_ms_per_step": kern, "compacted_decode_kernel_ms": round(compacted_decode, 3), "lsm_dev_decode_and_merge_kernel_ms": round(lsm_dev_total, 3),
           "lsm_dev_over_compacted": round(lsm_dev_total / compacted_decode, 2) if compacted_decode else None,
           "c3_results_bit_identical": identical, "c3_groups": len(results["compacted"][0])}
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
