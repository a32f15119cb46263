"""`-m gpu`: ZSTD data blocks (RocksDB compression types 7 / 0x40) inflated by b2_sst_decode: libzstd's golden frames in
runs that mix plain, LZ4 and ZSTD blocks, from host and device location; the damaged corpus with libzstd's verdicts;
concurrent handles; requests over ZSTD runs; a bench-sized round trip."""
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import orc
import scenarios as sc
import sstfmt
import sstlz4
import sstzstd as z
from compare import assert_same_rows
from test_gpu_sst import SOME, device_block_kvs
from test_sst_zstd_cpu import DEVICE_STRICTER, hand_frames
from tikv_b200 import ffi
from tikv_b200.executor import B2Error, DagHandler, SstDecoder, SstRegion, checksum

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import gen_zstd_blocks  # noqa: E402

pytestmark = pytest.mark.gpu
NEEDS_LIB = pytest.mark.skipif(z.libzstd() is None, reason="needs libzstd.so.1 to compress at run time")
tail = lambda t: bytes([t]) + b"\0" * 4  # noqa: E731


def decode_both(dec, data, offs, exp, n_lz4):
    import torch
    got, st = dec.decode(data, offs)
    assert device_block_kvs(got) == exp
    assert st.n_entries == len(exp) and st.h2d_bytes == len(data) + 8 * len(offs) and st.n_lz4_blocks == n_lz4
    t = torch.from_numpy(np.frombuffer(bytes(data) + b"\0" * 16, dtype=np.uint8).copy()).cuda()
    got, st = dec.decode(t.data_ptr(), offs, location=ffi.LOC_DEVICE)
    assert device_block_kvs(got) == exp and st.h2d_bytes == 8 * len(offs) and st.n_lz4_blocks == n_lz4


def golden_run():
    """every golden and hand-assembled frame as a data block, each beside the same block plain and LZ4-compressed"""
    blks, _ = gen_zstd_blocks.load()
    data, offs, exp, n_lz4 = b"", [0], [], 0
    items = [(raw, p) for _, raw, frames in blks for _, p in frames]
    items += [(raw, p) for _, p, raw in hand_frames() if sstfmt.decode(raw + b"\0" * 5, [0, len(raw) + 5])[0] == 0]
    for i, (raw, p) in enumerate(items):
        kvs = sstfmt.decode(raw + b"\0" * 5, [0, len(raw) + 5])[1]
        parts = [z.var32(len(raw)) + p + tail(z.ZSTD if i % 2 else z.ZSTD_NOT_FINAL)]
        if i % 5 == 0:
            parts += [raw + tail(0), sstlz4.frame(raw) + tail(4)]
            kvs = kvs * 3
            n_lz4 += 1
        for c in parts:
            data += c
            offs.append(len(data))
        exp += kvs
    return data, offs, exp, n_lz4


def test_golden_frames_in_mixed_runs():
    data, offs, exp, n_lz4 = golden_run()
    with SstDecoder() as dec:
        decode_both(dec, data, offs, exp, n_lz4)


def test_damaged_corpus_matches_libzstds_verdicts():
    """alone and as the second block of a run: decoded, B2_ERR_STORAGE or B2_ERR_UNSUPPORTED exactly as committed; a frame
    libzstd decodes is then read as a data block (which a damaged one may not be), as the oracle reads the same bytes"""
    _, dam = gen_zstd_blocks.load()
    good = [c for label, c, _, _ in dam if label == "good_0"][0]
    plain = gen_zstd_blocks.tiny_block() + tail(0)
    inflated = z.emul([c for _, c, _, _ in dam])
    with SstDecoder() as dec:
        for (label, c, verdict, _), (_, out) in zip(dam, inflated):
            want = z.CORRUPT if label in DEVICE_STRICTER else verdict
            for data, offs in ((c + tail(z.ZSTD), [0, len(c) + 5]), (plain + c + tail(z.ZSTD), [0, len(plain), len(plain) + len(c) + 5])):
                # (a slice shorter than 4 bytes plus the trailer is a corrupted block whatever its type byte says)
                rc, exp = (1, None) if want == z.CORRUPT or len(c) < 4 else ((2, None) if want == z.UNSUPPORTED else
                                                                sstfmt.decode(plain[:len(data) - len(c) - 5] + out + tail(0), offs[:-1] + [offs[-2] + len(out) + 5]))
                try:
                    got = device_block_kvs(dec.decode(data, offs)[0])
                    assert rc == 0 and got == exp, label
                except B2Error as e:
                    assert rc != 0 and e.status == (ffi.B2_ERR_UNSUPPORTED if rc == 2 else ffi.B2_ERR_STORAGE), (label, rc, e.status)
        assert device_block_kvs(dec.decode(good + tail(z.ZSTD), [0, len(good) + 5])[0]) == sstfmt.decode(plain, [0, len(plain)])[1]


def test_four_threads_on_four_handles():
    data, offs, exp, n_lz4 = golden_run()
    decs = [SstDecoder() for _ in range(4)]
    try:
        with ThreadPoolExecutor(max_workers=4) as pool:
            for _ in range(3):
                outs = list(pool.map(lambda d: device_block_kvs(d.decode(data, offs)[0]), decs))
                assert all(o == exp for o in outs)
    finally:
        for d in decs:
            d.close()


@NEEDS_LIB
@pytest.mark.parametrize("name,plan", SOME, ids=[n for n, _ in SOME])
def test_requests_over_zstd_runs_match_oracle(name, plan):
    host = sc.dirty_region(1, n_keys=900).build(read_ts=sc.READ_TS, n_write_blocks=2)
    runs = [z.build(b, block_size=2048) for b in host.wblocks]
    assert all(z.ZSTD in z.block_types(*r) for r in runs)
    reg = SstRegion(host, runs)
    try:
        assert all(st.n_lz4_blocks == 0 for st in reg.stats)
        for ranges in (sc.WHOLE, sc.split_ranges()):
            exp = orc.dag_handle(plan, ranges, host)
            got = DagHandler(plan, ranges, reg).handle_request()
            assert_same_rows(got, exp, ordered=not sc.is_agg(name), ctx=name)
            assert got.stats.write_processed_keys == exp.stats["processed_keys"] and got.stats.processed_size == exp.stats["processed_size"]
        assert checksum(sc.WHOLE, reg) == checksum(sc.WHOLE, host)
        assert checksum(sc.WHOLE, reg)[:2] == orc.checksum(sc.WHOLE, host)[:2]
    finally:
        reg.close()


@NEEDS_LIB
def test_bench_sized_round_trip():
    """3 M generated rows: encode on the device, copy to the host, compress with libzstd level 3, decode from host
    memory: keys, values and both offset arrays byte-identical to the generator's block"""
    import ctypes as C
    L = ffi.lib()
    n = 3_000_000
    spec = ffi.GenSpec()
    spec.table_id, spec.first_handle, spec.n_rows, spec.n_cols, spec.row_format, spec.seed = 1000, 0, n, 2, 2, 0x525C682A2F7CE3DB
    spec.commit_ts, spec.newer_ts = 20, 1 << 62
    spec.extra_versions_per_million, spec.delete_per_million, spec.lock_rec_per_million = 30000, 20000, 10000
    g, blk = C.c_void_p(), ffi.GenBlock()
    assert L.b2_gen_create(0, C.byref(spec), C.byref(g), C.byref(blk)) == 0
    h, enc = C.c_void_p(), ffi.SstEncoded()
    assert L.b2_sst_encode(0, C.byref(blk.block), 600, 16, 1, ord("z"), 8, 5, C.byref(h), C.byref(enc)) == 0
    plain = np.zeros(enc.data_len, dtype=np.uint8)
    offs = np.zeros(enc.n_blocks + 1, dtype=np.uint64)
    assert L.b2_copy_to_host(0, plain.ctypes.data, enc.data, enc.data_len) == 0
    assert L.b2_copy_to_host(0, offs.ctypes.data, enc.block_offs, 8 * len(offs)) == 0
    L.b2_sst_free(h)
    pb, po = plain.tobytes(), [int(x) for x in offs]
    chunk = 256
    with ThreadPoolExecutor(max_workers=os.cpu_count()) as pool:
        parts = list(pool.map(lambda a: z.compress_run(pb[po[a]:po[min(a + chunk, len(po) - 1)]], [o - po[a] for o in po[a:min(a + chunk, len(po) - 1) + 1]]),
                              range(0, len(po) - 1, chunk)))
    data, coffs = b"".join(d for d, _ in parts), [0]
    for d, o in parts:
        coffs += [coffs[-1] + x for x in o[1:]]
    assert len(data) < 0.6 * len(plain)
    assert z.block_types(data, coffs).count(z.ZSTD) > 0.9 * enc.n_blocks
    with SstDecoder() as dec:
        got, st = dec.decode(data, coffs)
        assert got.n == blk.block.n and st.key_bytes == blk.key_bytes and st.val_bytes == blk.val_bytes and st.n_lz4_blocks == 0

        def same(a, b, nbytes):
            ha, hb = np.zeros(nbytes, dtype=np.uint8), np.zeros(nbytes, dtype=np.uint8)
            assert L.b2_copy_to_host(0, ha.ctypes.data, a, nbytes) == 0 and L.b2_copy_to_host(0, hb.ctypes.data, b, nbytes) == 0
            return np.array_equal(ha, hb)
        assert same(got.keys, blk.block.keys, blk.key_bytes) and same(got.vals, blk.block.vals, blk.val_bytes)
        assert same(got.key_offs, blk.block.key_offs, 4 * (got.n + 1)) and same(got.val_offs, blk.block.val_offs, 4 * (got.n + 1))
    L.b2_gen_destroy(g)
