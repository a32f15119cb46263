#!/usr/bin/env python
"""Where a bench step's time goes outside the kernels: a few C3 (or C5) steps at bench size under torch.profiler.

Same generator, plan and request shape as bench.py (run_dag over the HBM-resident table, result left in HBM, the torch
merge inside the step).  Per step it prints one JSON line:
  step_ms             host time of the step (it ends in a device synchronise)
  gpu_busy_ms / gpu_idle_ms   union of kernel, memcpy and memset intervals on the device inside the step, and the rest
  unit_kernel_ms      kernels that stream the table (lean + general scan kernels)
  syncs               per phase (open / next_batch / merge / close): synchronous copies and host waits, by API name
  launches            per phase: kernel launches (runtime + driver API)
  open_to_first_unit_ms       start of b2_exec_open to the start of the first unit kernel on the device
  last_unit_to_batch_end_ms   end of the last unit kernel on the device to the return of next_batch
  other_kernels       the device work that is not a unit kernel, by name: total ms and count
Usage: python tools/request_trace.py [--workload c3|c5] [--steps 3] [--rows 500000000] [--blocks 16] [--out DIR]
"""
import argparse
import collections
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SYNC_APIS = ("cudaMemcpy", "cudaStreamSynchronize", "cudaEventSynchronize", "cudaDeviceSynchronize", "cuMemcpyDtoH_v2", "cuMemcpyHtoD_v2",
             "cuStreamSynchronize", "cuCtxSynchronize")
LAUNCH_APIS = ("cudaLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernel", "cuLaunchKernelEx")
DEVICE_CATS = ("kernel", "gpu_memcpy", "gpu_memset")
PHASES = ("open", "next_batch", "merge", "close")


def is_unit_kernel(name):
    return any(k in name for k in ("b2_fast_jit", "b2_scan_jit", "fast_kernel", "scan_kernel"))


def union_ms(intervals):
    tot, end = 0.0, None
    for a, b in sorted(intervals):
        if end is None or a > end:
            tot += b - a
            end = b
        elif b > end:
            tot += b - end
            end = b
    return tot / 1e3


def analyse(events):
    """Chrome-trace events -> one dict per step (timestamps in microseconds)."""
    ann = [e for e in events if e.get("cat") == "user_annotation"]
    steps = sorted((e for e in ann if e["name"].startswith("step")), key=lambda e: e["ts"])
    phases = [e for e in ann if e["name"] in PHASES]
    dev = [e for e in events if e.get("cat") in DEVICE_CATS and "dur" in e]
    api = [e for e in events if e.get("cat") in ("cuda_runtime", "cuda_driver")]
    out = []
    for s in steps:
        t0, t1 = s["ts"], s["ts"] + s["dur"]
        inside = lambda e: t0 <= e["ts"] < t1  # noqa: E731
        d = [e for e in dev if inside(e)]
        units = [e for e in d if e.get("cat") == "kernel" and is_unit_kernel(e["name"])]
        ph = [p for p in phases if inside(p)]

        def phase_of(e):
            for p in ph:
                if p["ts"] <= e["ts"] < p["ts"] + p["dur"]:
                    return p["name"]
            return "other"
        syncs = collections.defaultdict(collections.Counter)
        launches = collections.Counter()
        for e in api:
            if not inside(e):
                continue
            if e["name"] in SYNC_APIS:
                syncs[phase_of(e)][e["name"]] += 1
            elif e["name"] in LAUNCH_APIS:
                launches[phase_of(e)] += 1
        other = collections.defaultdict(lambda: [0.0, 0])
        for e in d:
            if e in units:
                continue
            k = e["name"] if e.get("cat") == "kernel" else e.get("cat") + ":" + e["name"]
            other[k[:80]][0] += e["dur"] / 1e3
            other[k[:80]][1] += 1
        opens = [p for p in ph if p["name"] == "open"]
        batches = [p for p in ph if p["name"] == "next_batch"]
        rec = {
            "step": s["name"], "step_ms": s["dur"] / 1e3,
            "gpu_busy_ms": union_ms([(e["ts"], e["ts"] + e["dur"]) for e in d]),
            "unit_kernel_ms": sum(e["dur"] for e in units) / 1e3, "unit_kernels": len(units),
            "syncs": {k: dict(v) for k, v in syncs.items()}, "sync_total": sum(sum(v.values()) for v in syncs.values()),
            "launches": dict(launches),
            "phase_ms": {p["name"]: p["dur"] / 1e3 for p in ph},
            "open_to_first_unit_ms": (min(e["ts"] for e in units) - opens[0]["ts"]) / 1e3 if units and opens else None,
            "last_unit_to_batch_end_ms": (batches[-1]["ts"] + batches[-1]["dur"] - max(e["ts"] + e["dur"] for e in units)) / 1e3 if units and batches else None,
            "other_kernels": {k: [round(v[0], 4), v[1]] for k, v in sorted(other.items(), key=lambda kv: -kv[1][0])},
        }
        rec["gpu_idle_ms"] = rec["step_ms"] - rec["gpu_busy_ms"]
        out.append(rec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c3", choices=["c3", "c5"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=500_000_000)
    ap.add_argument("--blocks", type=int, default=16)
    ap.add_argument("--out", default="", help="directory for the chrome trace (default: a temporary one, removed)")
    args = ap.parse_args()
    if not os.environ.get("B2_JIT_CACHE_DIR"):
        os.environ["B2_JIT_CACHE_DIR"] = tempfile.mkdtemp(prefix="b2_jit_cache_")
    import ctypes as C
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    import bench
    from tikv_b200 import dist as b2dist
    from tikv_b200 import ffi
    from tikv_b200.executor import BatchExecutor
    from tikv_b200.executor import checksum as b2_checksum
    L = ffi.lib()
    device = 0
    torch.cuda.set_device(device)
    table = "c3" if args.workload == "c3" else "c2"
    plan = bench.build_plan("c3") if args.workload == "c3" else None
    if plan is not None:
        L.b2_plan_prepare(C.byref(plan.c), device)
    gens, blks = bench.gen_blocks(ffi, device, table, args.rows, args.blocks)
    src = bench.Source(ffi, [b.block for b in blks], ffi.LOC_DEVICE, device)
    stream = torch.cuda.Stream(device=device)
    dev = torch.device("cuda", device)

    def step():  # bench.run_workload's one(): request, then the final merge on the same stream, waited for
        if args.workload == "c5":
            with record_function("next_batch"):
                rc, res, msg = b2_checksum(bench.table_range(), src, stream=stream.cuda_stream, want_stats=True)
            assert rc == 0, msg
            with record_function("merge"), torch.cuda.stream(stream):
                b2dist.merge_checksum(res[0], res[1], res[2], device=dev)
                stream.synchronize()
            return
        with record_function("open"):
            ex = BatchExecutor(plan, bench.table_range(), src, output=ffi.LOC_DEVICE, stream=stream.cuda_stream)
        while True:
            with record_function("next_batch"):
                rc, b = ex.next_batch_raw(1 << 24)
            assert rc == 0, ex.last_error().message
            with record_function("merge"), torch.cuda.stream(stream):
                keys, nul, acc = b2dist.agg_partials_as_tensors(ex, device)
                b2dist.merge_agg_partials(keys, nul, acc)
                stream.synchronize()
            if b.is_drained != ffi.DRAIN_REMAIN:
                break
        with record_function("close"):
            ex.close()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            with record_function(f"step{i}"):
                step()
        torch.cuda.synchronize()
    out_dir = args.out or tempfile.mkdtemp(prefix="b2_trace_")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, f"request_trace_{args.workload}.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    if not args.out:
        os.remove(path)
        os.rmdir(out_dir)
    for g in gens:
        L.b2_gen_destroy(g)
    for rec in analyse(events):
        rec["workload"], rec["gpu"] = args.workload, torch.cuda.get_device_name(device)
        print(json.dumps(rec))


if __name__ == "__main__":
    main()
