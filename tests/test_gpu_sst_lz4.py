"""`-m gpu`: LZ4 / LZ4HC data blocks (RocksDB compression types 4 / 5) inflated by b2_sst_decode, against the oracle's
block reader (tests/lz4_oracle.cpp + oracle/orc_sst.h) and against the decode of the same entries stored plain: runs of
the oracle's compressor, liblz4's golden blocks, runs mixing plain and LZ4 blocks, host and device location, rejected
blocks, requests over LZ4 runs and a bench-sized round trip."""
import os
import random
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import kvfmt
import orc
import scenarios as sc
import sstfmt
import sstlz4 as z
from compare import assert_same_rows
from test_gpu_sst import OPTS, SOME, device_block_kvs
from test_sst_lz4_cpu import damaged_corpus, small_compressed
from tikv_b200 import ffi
from tikv_b200.executor import B2Error, DagHandler, SstDecoder, SstRegion, checksum

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import gen_lz4_blocks  # noqa: E402

pytestmark = pytest.mark.gpu

LZ4_OPTS = [o for o in OPTS if o.get("trailer_len", 5) == 5]  # (the compression type lives in the trailer)


def decode_both(dec, data, offs, fmt, n_lz4):
    """host and device location: the decoded block, checked against the oracle's reader; returns the entries"""
    import torch
    rc, exp = z.decode(data, offs, **fmt)
    assert rc == 0
    got, st = dec.decode(data, offs, **fmt)
    assert device_block_kvs(got) == exp
    assert st.n_entries == len(exp) and st.key_bytes == sum(len(k) for k, _ in exp) and st.val_bytes == sum(len(v) for _, v in exp)
    assert st.h2d_bytes == len(data) + 8 * len(offs) and st.n_lz4_blocks == n_lz4
    t = torch.from_numpy(np.frombuffer(bytes(data) + b"\0" * 16, dtype=np.uint8).copy()).cuda()
    got, st = dec.decode(t.data_ptr(), offs, location=ffi.LOC_DEVICE, **fmt)
    assert device_block_kvs(got) == exp and st.h2d_bytes == 8 * len(offs) and st.n_lz4_blocks == n_lz4
    return exp


@pytest.mark.parametrize("opts", LZ4_OPTS)
def test_lz4_runs_match_the_oracle_and_the_plain_decode(opts):
    host = sc.dirty_region(7, n_keys=900).build(read_ts=sc.READ_TS)
    fmt = {k: opts[k] for k in ("key_prefix_len", "key_suffix_len") if k in opts}
    with SstDecoder() as dec:
        for blk in host.wblocks + [host.dblock]:
            plain, poffs = sstfmt.build(blk, **opts)
            data, offs = z.build(blk, **opts)
            types = z.block_types(data, offs)  # (small blocks with few shared prefixes may all stay plain)
            exp = decode_both(dec, data, offs, fmt, types.count(4))
            assert exp == blk.kvs == device_block_kvs(dec.decode(plain, poffs, **fmt)[0])
            # every block compressed, as LZ4HC (type 5: the same stream format)
            data, offs = z.compress_run(plain, poffs, type_byte=z.LZ4HC, force=True)
            assert decode_both(dec, data, offs, fmt, len(offs) - 1) == blk.kvs


def test_golden_liblz4_blocks():
    """liblz4's LZ4 and LZ4HC output for scenario blocks (dirty region, default CF, v1 rows, long keys), in one run that
    also holds the same blocks plain"""
    data, offs, types, exp = b"", [0], [], []
    for name, raw, lz4, hc in gen_lz4_blocks.load():
        fmt_kvs = sstfmt.decode(raw + b"\0" * 5, [0, len(raw) + 5])[1]
        for contents, t in ((raw, 0), (z.frame(raw, lz4), 4), (z.frame(raw, hc), 5)):
            data += contents + bytes([t]) + b"\0" * 4
            offs.append(len(data))
            types.append(t)
            exp += fmt_kvs
    with SstDecoder() as dec:
        assert decode_both(dec, data, offs, {}, types.count(4) + types.count(5)) == exp


def test_mixed_runs_long_keys_and_concurrent_handles():
    """incompressible blocks stay plain between LZ4 blocks; keys beyond 128 bytes (the sequential path) inside LZ4 blocks;
    four threads decode LZ4 runs at once"""
    rng = random.Random(6)
    kvs = []
    for i in range(3000):
        k = b"k%06d" % i + (bytes(rng.randrange(97, 99) for _ in range(rng.choice((0, 60, 121, 130, 200, 400)))) if rng.random() < 0.3 else b"")
        v = bytes(rng.randrange(256) for _ in range(200)) if (i // 100) % 3 == 1 else b"v%d " % (i % 7) * rng.choice((1, 10, 40))
        kvs.append((k, v))
    blk = kvfmt.HostBlock(kvs)
    runs = [z.build(blk, restart_interval=r, block_size=bs) for r, bs in ((16, 32768), (5, 3000), (16, 100000), (1, 4096))]
    assert any(0 in z.block_types(*r) and 4 in z.block_types(*r) for r in runs)
    decs = [SstDecoder() for _ in runs]
    try:
        for d, (data, offs) in zip(decs, runs):
            assert decode_both(d, data, offs, {}, z.block_types(data, offs).count(4)) == blk.kvs
        with ThreadPoolExecutor(max_workers=4) as pool:
            for _ in range(3):
                outs = list(pool.map(lambda a: device_block_kvs(a[0].decode(a[1][0], a[1][1])[0]), zip(decs, runs)))
                assert all(o == blk.kvs for o in outs)
    finally:
        for d in decs:
            d.close()


def test_rejected_blocks():
    blk, raw, good = small_compressed()
    tail = lambda t: bytes([t]) + b"\0" * 4  # noqa: E731
    with SstDecoder() as dec:
        for t in (1, 2, 3, 6, 7, 0x40, 0x80, 200, 0xFE):
            with pytest.raises(B2Error) as e:
                dec.decode(good + tail(t), [0, len(good) + 5])
            assert e.value.status == ffi.B2_ERR_UNSUPPORTED
            assert z.decode(good + tail(t), [0, len(good) + 5])[0] == 2
        for t in (8, 0x7F, 0xFF):
            with pytest.raises(B2Error) as e:
                dec.decode(good + tail(t), [0, len(good) + 5])
            assert e.value.status == ffi.B2_ERR_STORAGE
            assert z.decode(good + tail(t), [0, len(good) + 5])[0] == 1
        # a valid run whose second block is in a compressor the device does not have: the host keeps it
        with pytest.raises(B2Error) as e:
            dec.decode(good + tail(4) + good + tail(7), [0, len(good) + 5, 2 * len(good) + 10])
        assert e.value.status == ffi.B2_ERR_UNSUPPORTED
        # the damaged-contents corpus of the CPU test, alone and as the second block of a run: corrupt exactly where
        # the oracle says so, and a good run decodes on the same handle afterwards
        plain = raw + tail(0)
        _, corpus = damaged_corpus()
        n_bad = 0
        for label, c in corpus:
            for data, offs in ((c + tail(4), [0, len(c) + 5]), (plain + c + tail(4), [0, len(plain), len(plain) + len(c) + 5])):
                rc, exp = z.decode(data, offs)
                try:
                    got = device_block_kvs(dec.decode(data, offs)[0])
                    assert rc == 0 and got == exp, label
                except B2Error as e:
                    assert rc != 0 and e.status == (ffi.B2_ERR_UNSUPPORTED if rc == 2 else ffi.B2_ERR_STORAGE), (label, rc, e.status)
                    n_bad += 1
        assert n_bad > 500
        assert device_block_kvs(dec.decode(good + tail(4), [0, len(good) + 5])[0]) == blk.kvs


@pytest.mark.parametrize("name,plan", SOME, ids=[n for n, _ in SOME])
def test_requests_over_lz4_runs_match_oracle(name, plan):
    host = sc.dirty_region(1, n_keys=900).build(read_ts=sc.READ_TS, n_write_blocks=2)
    runs = [z.build(b, block_size=2048) for b in host.wblocks]
    assert all(4 in z.block_types(*r) for r in runs)
    reg = SstRegion(host, runs)
    try:
        assert [st.n_lz4_blocks for st in reg.stats] == [z.block_types(*r).count(4) for r in runs]
        for ranges in (sc.WHOLE, sc.split_ranges()):
            exp = orc.dag_handle(plan, ranges, host)
            got = DagHandler(plan, ranges, reg).handle_request()
            assert_same_rows(got, exp, ordered=not sc.is_agg(name), ctx=name)
            assert got.stats.write_processed_keys == exp.stats["processed_keys"] and got.stats.processed_size == exp.stats["processed_size"]
        assert checksum(sc.WHOLE, reg) == checksum(sc.WHOLE, host)
        assert checksum(sc.WHOLE, reg)[:2] == orc.checksum(sc.WHOLE, host)[:2]
    finally:
        reg.close()


def test_bench_sized_round_trip():
    """3 M generated rows: encode on the device, copy to the host, compress with the oracle, decode from host memory:
    keys, values and both offset arrays byte-identical to the generator's block, and fewer bytes than the plain run"""
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
    data, coffs = z.compress_run(plain.tobytes(), [int(x) for x in offs])
    assert len(data) < 0.6 * len(plain)
    with SstDecoder() as dec:
        got, st = dec.decode(data, coffs)
        assert got.n == blk.block.n and st.key_bytes == blk.key_bytes and st.val_bytes == blk.val_bytes
        assert st.n_lz4_blocks == z.block_types(data, coffs).count(4) > 0.9 * enc.n_blocks

        def same(a, b, nbytes):
            ha, hb = np.zeros(nbytes, dtype=np.uint8), np.zeros(nbytes, dtype=np.uint8)
            assert L.b2_copy_to_host(0, ha.ctypes.data, a, nbytes) == 0 and L.b2_copy_to_host(0, hb.ctypes.data, b, nbytes) == 0
            return np.array_equal(ha, hb)
        assert same(got.keys, blk.block.keys, blk.key_bytes) and same(got.vals, blk.block.vals, blk.val_bytes)
        assert same(got.key_offs, blk.block.key_offs, 4 * (got.n + 1)) and same(got.val_offs, blk.block.val_offs, 4 * (got.n + 1))
    L.b2_gen_destroy(g)
