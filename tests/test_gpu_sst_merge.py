"""`-m gpu`: b2_sst_merge, the sorted runs of one LSM snapshot merged on the device.  Known answers (runs derived from a
dirty region's write block plus noise that must not change it) through the device, the CPU oracle and the Python model;
runs of plain, LZ4 and ZSTD blocks with and without trailers, long keys, from host and device memory; exact stats;
one-run equivalence with b2_sst_decode; rejections; requests over merged regions; concurrent handles; a 3 M-row LSM
split on the device."""
import ctypes as C
import random
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import orc
import scenarios as sc
import sstfmt
import sstlz4
import sstmerge as m
import sstzstd as z
from compare import assert_same_rows
from test_gpu_sst import SOME, device_block_kvs
from tikv_b200 import ffi
from tikv_b200.executor import B2Error, DagHandler, SstDecoder, SstRegion, checksum

pytestmark = pytest.mark.gpu
STATS = ("n_in", "n_out", "n_invisible", "n_hidden", "n_deletions")


def stored(runs, seed, compress=True):
    """each run as data blocks: plain with or without trailers, LZ4 or ZSTD (when libzstd is there), chosen per run"""
    rng = random.Random(seed)
    out = []
    for r in runs:
        kind = rng.choice(["plain0", "plain5", "lz4", "zstd"] if compress else ["plain0", "plain5"])
        tl = 0 if kind == "plain0" else 5
        data, offs = m.build_run(r, trailer_len=tl, block_size=rng.choice([512, 4096]), restart_interval=rng.choice([1, 16]))
        if kind == "lz4":
            data, offs = sstlz4.compress_run(data, offs, force=True)
        elif kind == "zstd" and z.libzstd() is not None:
            data, offs = z.compress_run(data, offs, force=True)
        out.append((data, offs, tl))
    return out


def merge(dec, built, snap, gs, location=ffi.LOC_HOST):
    import torch
    keep = []
    runs = []
    for data, offs, tl in built:
        if location == ffi.LOC_DEVICE:
            t = torch.from_numpy(np.frombuffer(bytes(data) + b"\0" * 16, dtype=np.uint8).copy()).cuda()
            keep.append(t)
            data = t.data_ptr()
        runs.append(dict(data=data, block_offs=offs, trailer_len=tl))
    blk, st = dec.merge(runs, snap, global_seqs=gs, location=location)
    return device_block_kvs(blk), st


def region_kvs(seed, n_keys=500):
    host = sc.dirty_region(seed, n_keys=n_keys).build(read_ts=sc.READ_TS, n_write_blocks=1)
    return host, list(host.wblocks[0].kvs)


@pytest.mark.parametrize("n_runs", [1, 2, 3, 5, 12])
def test_known_answer_device_oracle_and_model(n_runs):
    _, kvs = region_kvs(n_runs)
    runs, gs, snap = m.derive_runs(kvs, 100 + n_runs, n_runs, long_noise=True)
    assert any(len(u) > 128 for run in runs for u, _, _, _ in run)
    built = stored(runs, n_runs)
    exp, counts = m.model(runs, snap, gs)
    assert exp == kvs
    plain = [m.build_run(r) for r in runs]  # (the oracle's block iterator reads plain blocks)
    rc, okvs, ocounts = m.oracle_merge(plain, snap, gs)
    assert rc == 0 and okvs == kvs and ocounts == counts
    with SstDecoder() as dec:
        for loc in (ffi.LOC_HOST, ffi.LOC_DEVICE):
            got, st = merge(dec, built, snap, gs, loc)
            assert got == kvs
            assert {k: getattr(st, k) for k in STATS} == counts
            assert st.n_in == st.n_out + st.n_invisible + st.n_hidden + st.n_deletions
            assert st.key_bytes == sum(len(k) for k, _ in kvs) and st.val_bytes == sum(len(v) for _, v in kvs) and st.n_runs == n_runs
            data_bytes = sum(len(d) for d, _, _ in built) if loc == ffi.LOC_HOST else 0
            assert st.h2d_bytes == data_bytes + sum(8 * len(o) for _, o, _ in built)
            assert st.n_lz4_blocks == sum(sstlz4.block_types(d, o).count(sstlz4.LZ4) for d, o, tl in built if tl == 5)
        for s in (0, snap // 2, snap + 100_000, m.MAX_SEQ):  # other snapshots: device = model = oracle
            exp, counts = m.model(runs, s, gs)
            got, st = merge(dec, built, s, gs)
            assert got == exp and {k: getattr(st, k) for k in STATS} == counts
            assert m.oracle_merge(plain, s, gs)[1:] == (exp, counts)


@pytest.mark.parametrize("seed", range(6))
def test_generated_shapes(seed):
    rng = random.Random(seed)
    kvs = [(bytes(rng.choice(b"ab\x02\xff") for _ in range(rng.randrange(1, 200))) + b"\x02", b"v%d" % i) for i in range(300)]
    kvs = sorted(dict(kvs).items())
    n_runs = 1 + seed * 2
    runs, gs, snap = m.derive_runs(kvs, seed, n_runs, long_noise=True)
    built = stored(runs, seed)
    with SstDecoder() as dec:
        got, st = merge(dec, built, snap, gs)
    assert got == kvs and {k: getattr(st, k) for k in STATS} == m.model(runs, snap, gs)[1]


def test_one_run_equals_decode():
    """one run of kTypeValue entries at or below the snapshot: byte-identical to b2_sst_decode, offsets included"""
    _, kvs = region_kvs(7, 800)
    entries = [(k, rng_seq, m.VALUE, v) for (k, v), rng_seq in zip(kvs, range(1, len(kvs) + 1))]
    data, offs = m.build_run(entries, block_size=2048)
    L = ffi.lib()
    with SstDecoder() as a, SstDecoder() as b:
        d, _ = a.decode(data, offs)
        g, st = b.merge([(data, offs)], len(kvs))
        assert g.n == d.n == len(kvs) and st.n_out == len(kvs) and st.n_hidden == st.n_invisible == st.n_deletions == 0

        def host(p, n):
            h = np.zeros(n, dtype=np.uint8)
            assert L.b2_copy_to_host(0, h.ctypes.data, p, n) == 0
            return h.tobytes()
        kb, vb = sum(len(k) for k, _ in kvs), sum(len(v) for _, v in kvs)
        for x, y, n in ((g.keys, d.keys, ((kb + 47) & ~15)), (g.vals, d.vals, ((vb + 47) & ~15)), (g.key_offs, d.key_offs, 4 * (d.n + 1)),
                        (g.val_offs, d.val_offs, 4 * (d.n + 1))):
            assert host(x, n) == host(y, n)


def test_rejections_and_the_handle_keeps_working():
    ok = [(b"a", 5, m.VALUE, b"x"), (b"b", 5, m.VALUE, b"y")]
    good = m.build_run(ok)
    short = sstfmt.build(m.FlatBlock([(b"a" * 7, b"v")]), key_suffix_len=0)
    cases = [
        ([good, m.build_run([(b"a", 3, m.MERGE, b"m")])], None, ffi.B2_ERR_UNSUPPORTED),
        ([good, m.build_run([(b"a", 3, m.BLOB_INDEX, b"m")])], None, ffi.B2_ERR_UNSUPPORTED),
        ([good, m.build_run([(b"b", 5, 1, b""), (b"a", 5, 1, b"")], sort=False)], None, ffi.B2_ERR_STORAGE),
        ([good, m.build_run([(b"a", 3, 1, b""), (b"a", 5, 1, b"")], sort=False)], None, ffi.B2_ERR_STORAGE),
        ([good, m.build_run([(b"a", 5, 1, b""), (b"a", 5, 1, b"")], sort=False)], None, ffi.B2_ERR_STORAGE),
        ([good, m.build_run([(b"a", 1, 1, b"")])], [0, 9], ffi.B2_ERR_STORAGE),
        ([good, short], None, ffi.B2_ERR_STORAGE),
        ([(good[0][:-3], good[1][:-1] + [good[1][-1] - 3])], None, ffi.B2_ERR_STORAGE),  # a damaged block
    ]
    with SstDecoder() as dec:
        for runs, gs, status in cases:
            with pytest.raises(B2Error) as ei:
                dec.merge(runs, 10, global_seqs=gs)
            assert ei.value.status == status, (runs, ei.value.message)
            got, st = dec.merge([good], 10)
            assert device_block_kvs(got) == [(b"a", b"x"), (b"b", b"y")]
        L = ffi.lib()
        arr = (ffi.SstBlocks * 2)()
        for i in range(2):
            arr[i].data, arr[i].n_blocks, arr[i].trailer_len, arr[i].key_prefix_len, arr[i].key_suffix_len = None, 0, 5, 1, 8
        blk, st = ffi.CfBlock(), ffi.SstMergeStats()
        args = lambda n=2, snap=10, gs=None: (0, ffi.LOC_HOST, arr, n, gs, snap, C.byref(dec.h), C.byref(blk), C.byref(st))  # noqa: E731
        assert L.b2_sst_merge(*args()) == 0 and blk.n == 0 and st.n_runs == 2
        assert L.b2_sst_merge(*args(n=0)) == 0 and blk.n == 0
        assert L.b2_sst_merge(*args(n=1025)) == ffi.B2_ERR_INVALID_ARG
        assert L.b2_sst_merge(*args(snap=1 << 56)) == ffi.B2_ERR_INVALID_ARG
        assert L.b2_sst_merge(*args(gs=(C.c_uint64 * 2)(0, 1 << 56))) == ffi.B2_ERR_INVALID_ARG
        arr[1].key_suffix_len = 0
        assert L.b2_sst_merge(*args()) == ffi.B2_ERR_INVALID_ARG
        arr[1].key_suffix_len, arr[1].key_prefix_len = 8, 0
        assert L.b2_sst_merge(*args()) == ffi.B2_ERR_INVALID_ARG
        arr[1].key_prefix_len, arr[1].trailer_len = 1, 0  # trailer_len may differ per run
        assert L.b2_sst_merge(*args()) == 0
        assert device_block_kvs(dec.merge([good], 10)[0]) == [(b"a", b"x"), (b"b", b"y")]


@pytest.mark.parametrize("name,plan", SOME, ids=[n for n, _ in SOME])
def test_requests_over_merged_regions_match_oracle(name, plan):
    host = sc.dirty_region(3, n_keys=900).build(read_ts=sc.READ_TS, n_write_blocks=2)
    kvs = [kv for b in host.wblocks for kv in b.kvs]
    runs, gs, snap = m.derive_runs(kvs, 3, 6)
    reg = SstRegion(host, [(d, o, g) for (d, o, _), g in zip(stored_with_trailer(runs, 3), gs)], snapshot_seq=snap)
    try:
        assert reg.stats[0].n_out == len(kvs)
        for ranges in (sc.WHOLE, sc.split_ranges()):
            exp = orc.dag_handle(plan, ranges, host)
            got = DagHandler(plan, ranges, reg).handle_request()
            assert_same_rows(got, exp, ordered=not sc.is_agg(name), ctx=name)
            assert got.stats.write_processed_keys == exp.stats["processed_keys"] and got.stats.processed_size == exp.stats["processed_size"]
        assert checksum(sc.WHOLE, reg) == checksum(sc.WHOLE, host)
        assert checksum(sc.WHOLE, reg)[:2] == orc.checksum(sc.WHOLE, host)[:2]
    finally:
        reg.close()


def stored_with_trailer(runs, seed):
    """as stored(), every run with the 5-byte trailer (SstRegion passes one trailer_len for all runs)"""
    return [(d, o, 5) if tl == 5 else m.build_run(r, trailer_len=5) + (5,) for (d, o, tl), r in zip(stored(runs, seed), runs)]


def test_four_threads_on_four_handles():
    _, kvs = region_kvs(11)
    runs, gs, snap = m.derive_runs(kvs, 11, 7, long_noise=True)
    built = stored(runs, 11)
    decs = [SstDecoder() for _ in range(4)]
    try:
        with ThreadPoolExecutor(max_workers=4) as pool:
            for _ in range(3):
                outs = list(pool.map(lambda d: merge(d, built, snap, gs)[0], decs))
                assert all(o == kvs for o in outs)
    finally:
        for d in decs:
            d.close()


def test_bench_sized_lsm_split_on_the_device():
    """3 M generated rows split on the device into 5 runs (sstmerge.device_lsm) with tombstones over extra keys, shadowed
    versions, new keys and entries above the snapshot (footers appended with torch, blocks encoded by b2_sst_encode with key_suffix_len 0), merged from
    host memory: keys, values and both offset arrays bit-identical to the generator's block"""
    import torch
    L = ffi.lib()
    n = 3_000_000
    spec = ffi.GenSpec()
    spec.table_id, spec.first_handle, spec.n_rows, spec.n_cols, spec.row_format, spec.seed = 1000, 0, n, 2, 2, 0x525C682A2F7CE3DB
    spec.commit_ts, spec.newer_ts = 20, 1 << 62
    spec.extra_versions_per_million, spec.delete_per_million, spec.lock_rec_per_million = 30000, 20000, 10000
    g, blk = C.c_void_p(), ffi.GenBlock()
    assert L.b2_gen_create(0, C.byref(spec), C.byref(g), C.byref(blk)) == 0
    try:
        runs, snap = m.device_lsm(blk, n_l0=3)
        built = []
        for keys, koff, vals, voff, cnt in runs:
            flat = ffi.CfBlock()
            flat.keys, flat.key_offs, flat.vals, flat.val_offs, flat.n = keys.data_ptr(), koff.data_ptr(), vals.data_ptr(), voff.data_ptr(), cnt
            h, enc = C.c_void_p(), ffi.SstEncoded()
            assert L.b2_sst_encode(0, C.byref(flat), 600, 16, 1, ord("z"), 0, 5, C.byref(h), C.byref(enc)) == 0
            data, offs = np.zeros(enc.data_len + 16, dtype=np.uint8), np.zeros(enc.n_blocks + 1, dtype=np.uint64)
            assert L.b2_copy_to_host(0, data.ctypes.data, enc.data, enc.data_len) == 0
            assert L.b2_copy_to_host(0, offs.ctypes.data, enc.block_offs, 8 * len(offs)) == 0
            L.b2_sst_free(h)
            built.append((data, offs))
        del runs
        torch.cuda.empty_cache()
        with SstDecoder() as dec:
            got, st = dec.merge(built, snap)
            assert got.n == blk.block.n and st.key_bytes == blk.key_bytes and st.val_bytes == blk.val_bytes
            assert st.n_in == st.n_out + st.n_invisible + st.n_hidden + st.n_deletions and st.n_deletions > 0 and st.n_hidden > 0 and st.n_invisible > 0

            def same(a, b, nbytes):
                ha, hb = np.zeros(nbytes, dtype=np.uint8), np.zeros(nbytes, dtype=np.uint8)
                assert L.b2_copy_to_host(0, ha.ctypes.data, a, nbytes) == 0 and L.b2_copy_to_host(0, hb.ctypes.data, b, nbytes) == 0
                return np.array_equal(ha, hb)
            assert same(got.keys, blk.block.keys, blk.key_bytes) and same(got.vals, blk.block.vals, blk.val_bytes)
            assert same(got.key_offs, blk.block.key_offs, 4 * (got.n + 1)) and same(got.val_offs, blk.block.val_offs, 4 * (got.n + 1))
    finally:
        L.b2_gen_destroy(g)
