"""GPU measurement: the C3 request end to end from RocksDB data blocks stored plain against the same blocks stored
LZ4-compressed, as TiKV's LZ4 levels hold them on disk, and ZSTD-compressed, as its bottommost levels do.

Setup (untimed): the C3 table generated as `--regions` regions, each encoded on the device (b2_sst_encode, bench.sst_e2e's
block sizing: ~32 KiB blocks, restart interval 16, 'z' prefix, internal-key footer, trailer) and copied to pinned host
memory; an LZ4 copy of every run made by the oracle's compressor (tests/lz4_oracle.cpp, RocksDB's 12.5 % rule) and a
ZSTD copy made by libzstd at level 3 (RocksDB's default level, the same rule), on all host cores.  Timed, alternating arms within each round: one step = b2_sst_decode of every region (two decoder threads, as
bench.py overlaps them) + the C3 request over the decoded blocks, result to the host.
  plain    plain blocks from pinned host memory
  lz4      LZ4 blocks from pinned host memory
  lz4_dev  the LZ4 runs already in HBM (B2_LOC_DEVICE): inflate + expansion + request, nothing crosses PCIe
  zstd     ZSTD blocks from pinned host memory
  zstd_dev the ZSTD runs already in HBM
  zstd_host every ZSTD block inflated by libzstd on all host cores inside the step (ctypes calls from a thread pool),
           then the run decoded as plain blocks from host memory: the path a caller without device ZSTD takes
Then, in a separate profiled pass (torch.profiler, CUDA activities), the device time of each b2_sst_decode kernel per step.
Prints one JSON object (and writes it to --out when given).

  python tools/sst_lz4_bench.py [--rows 70000000] [--regions 7] [--rounds 3] [--steps 3] [--out FILE]"""
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
import sstlz4  # noqa: E402
import sstzstd  # noqa: E402
from tikv_b200 import ffi  # noqa: E402
from tikv_b200.executor import DagHandler, SstDecoder  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or "unknown (nvidia-smi: %s)" % q.stderr.strip()[:200]


def compress_parallel(pool, data, offs, chunk=512, fn=sstlz4.compress_run):
    """the run fn makes of (data, offs) (default: the oracle's LZ4 run), block ranges processed on all cores"""
    parts = list(pool.map(lambda a: fn(data[offs[a]:offs[min(a + chunk, len(offs) - 1)]], [o - offs[a] for o in offs[a:min(a + chunk, len(offs) - 1) + 1]]),
                          range(0, len(offs) - 1, chunk)))
    out, noffs = [], [0]
    for d, o in parts:
        base = noffs[-1]
        out.append(d)
        noffs += [base + x for x in o[1:]]
    return b"".join(out), noffs


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
    plain, lz4, lz4_dev, keep = [], [], [], []
    zstd, zstd_dev, zstd_bytes_host = [], [], []
    n_blocks = n_lz4 = plain_bytes = lz4_bytes = inflated_bytes = 0
    n_zstd = zstd_bytes = zstd_inflated_bytes = 0
    assert sstzstd.libzstd() is not None, "needs libzstd.so.1"
    t0 = time.time()
    with ThreadPoolExecutor(max_workers=os.cpu_count()) as pool:
        for b in blks:
            per = max(16, 32768 // max(8, int((b.key_bytes + b.val_bytes) / max(1, b.block.n)) - 9))  # (bench.sst_e2e's sizing)
            h, enc = C.c_void_p(), ffi.SstEncoded()
            assert L.b2_sst_encode(dev, C.byref(b.block), per, 16, 1, ord("z"), 8, 5, C.byref(h), C.byref(enc)) == 0, L.b2_last_error_message()
            p = L.b2_host_alloc_pinned_near(dev, enc.data_len + 64)
            offs = np.zeros(enc.n_blocks + 1, dtype=np.uint64)
            assert p and L.b2_copy_to_host(dev, p, enc.data, enc.data_len) == 0 and L.b2_copy_to_host(dev, offs.ctypes.data, enc.block_offs, 8 * len(offs)) == 0
            L.b2_sst_free(h)
            keep.append(p)
            plain.append((p, offs))
            data, coffs = compress_parallel(pool, C.string_at(p, enc.data_len), [int(x) for x in offs])
            types = sstlz4.block_types(data, coffs)
            q = L.b2_host_alloc_pinned_near(dev, len(data) + 64)
            assert q
            C.memmove(q, data, len(data))
            keep.append(q)
            co = np.asarray(coffs, dtype=np.uint64)
            lz4.append((q, co))
            t = torch.from_numpy(np.frombuffer(data + b"\0" * 16, dtype=np.uint8).copy()).to(dev)
            lz4_dev.append((t, co))
            n_blocks += len(types)
            n_lz4 += types.count(4)
            plain_bytes += enc.data_len
            lz4_bytes += len(data)
            inflated_bytes += sum(offs[i + 1] - offs[i] - 5 for i, ty in enumerate(types) if ty == 4)
            data, coffs = compress_parallel(pool, C.string_at(p, enc.data_len), [int(x) for x in offs], fn=sstzstd.compress_run)
            types = sstzstd.block_types(data, coffs)
            q = L.b2_host_alloc_pinned_near(dev, len(data) + 64)
            assert q
            C.memmove(q, data, len(data))
            keep.append(q)
            co = np.asarray(coffs, dtype=np.uint64)
            zstd.append((q, co))
            zstd_bytes_host.append((data, coffs))
            zstd_dev.append((torch.from_numpy(np.frombuffer(data + b"\0" * 16, dtype=np.uint8).copy()).to(dev), co))
            n_zstd += types.count(sstzstd.ZSTD)
            zstd_bytes += len(data)
            zstd_inflated_bytes += sum(offs[i + 1] - offs[i] - 5 for i, ty in enumerate(types) if ty == sstzstd.ZSTD)
    setup_s = time.time() - t0
    decs = [SstDecoder(dev) for _ in blks]
    arms = {"plain": (plain, ffi.LOC_HOST), "lz4": (lz4, ffi.LOC_HOST), "lz4_dev": ([(t.data_ptr(), o) for t, o in lz4_dev], ffi.LOC_DEVICE),
            "zstd": (zstd, ffi.LOC_HOST), "zstd_dev": ([(t.data_ptr(), o) for t, o in zstd_dev], ffi.LOC_DEVICE), "zstd_host": (zstd_bytes_host, ffi.LOC_HOST)}
    src_keep = []
    hpool = ThreadPoolExecutor(max_workers=os.cpu_count())

    zlib = sstzstd.libzstd()

    def host_inflate(run):  # libzstd on all host cores (ZSTD_decompress releases the GIL): the run with every block plain
        def chunk(d, o):
            out, noffs = bytearray(), [0]
            for a, b in zip(o, o[1:]):
                if d[b - 5] == sstzstd.ZSTD:
                    size, i = 0, 0
                    while True:
                        size |= (d[a + i] & 0x7F) << (7 * i)
                        i += 1
                        if not d[a + i - 1] & 0x80:
                            break
                    dst = C.create_string_buffer(size + 5)
                    assert zlib.ZSTD_decompress(dst, size, d[a + i:b - 5], b - 5 - a - i) == size
                    out += dst.raw
                else:
                    out += d[a:b]
                noffs.append(len(out))
            return bytes(out), noffs
        return compress_parallel(hpool, run[0], run[1], chunk=256, fn=chunk)

    with ThreadPoolExecutor(max_workers=2) as pool:  # two regions in flight, as bench.py's data-block record
        def decode_all(arm):
            runs, loc = arms[arm]
            if arm == "zstd_host":
                res = list(pool.map(lambda a: a[0].decode(*host_inflate(a[1]), location=loc), zip(decs, runs)))
            else:
                res = list(pool.map(lambda a: a[0].decode(a[1][0], a[1][1], location=loc), zip(decs, runs)))
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
            results[arm] = (sorted(zip(*r.columns)), sum(st.h2d_bytes for _, st in res), sum(st.n_lz4_blocks for _, st in res))
        identical = all(results[a][0] == results["plain"][0] for a in arms)
        times = {a: [] for a in arms}
        for _ in range(args.rounds):
            for arm in arms:
                torch.cuda.synchronize()
                t = time.perf_counter()
                for _ in range(args.steps):
                    step(arm)
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t) * 1e3 / args.steps)

        # device time per kernel, in a profiled pass of its own
        from torch.profiler import ProfilerActivity, profile
        kern = {}
        for arm in ("plain", "lz4_dev", "zstd_dev"):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    decode_all(arm)
                torch.cuda.synchronize()
            k = {}
            for e in prof.key_averages():
                if e.key.find("sst_") >= 0 or e.key.find("DeviceScan") >= 0:
                    name = next((n for n in ("sst_blocks", "sst_inflate", "sst_zstd", "sst_count", "sst_expand") if n in e.key), "cub_scan")
                    k[name] = k.get(name, 0.0) + e.device_time_total / 1e3 / args.steps
            kern[arm] = {n: round(v, 3) for n, v in sorted(k.items())}
    hpool.shutdown()
    for d in decs:
        d.close()
    for p in keep:
        L.b2_host_free_pinned(p)
    for g in gens:
        L.b2_gen_destroy(g)
    inflate_ms = kern["lz4_dev"].get("sst_inflate", 0.0)
    zstd_ms = kern["zstd_dev"].get("sst_zstd", 0.0)
    out = {"gpu": info, "rows": rows, "regions": args.regions, "rounds": args.rounds, "steps_per_round": args.steps, "setup_s": round(setup_s, 1),
           "blocks": n_blocks, "lz4_blocks": n_lz4, "plain_block_bytes": plain_bytes, "lz4_run_bytes": lz4_bytes, "ratio": round(lz4_bytes / plain_bytes, 4),
           "arms": {a: {"ms_per_step_median": round(statistics.median(v), 2), "ms_per_step_range": [round(min(v), 2), round(max(v), 2)],
                        "rows_per_s_median": rows / (statistics.median(v) / 1e3), "h2d_bytes_per_step": results[a][1],
                        "lz4_blocks_per_step": results[a][2]} for a, v in times.items()},
           "kernel_ms_per_step": kern, "inflate_ms_per_step": inflate_ms,
           "inflated_GB_per_s": round(inflated_bytes / (inflate_ms / 1e3) / 1e9, 1) if inflate_ms else None,
           "zstd_blocks": n_zstd, "zstd_run_bytes": zstd_bytes, "zstd_ratio": round(zstd_bytes / plain_bytes, 4), "sst_zstd_ms_per_step": zstd_ms,
           "zstd_inflated_GB_per_s": round(zstd_inflated_bytes / (zstd_ms / 1e3) / 1e9, 1) if zstd_ms else None,
           "c3_results_bit_identical": identical, "c3_groups": len(results["plain"][0])}
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
