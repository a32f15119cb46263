"""`-m "not gpu"`: LZ4 / LZ4HC data blocks (RocksDB compression types 4 / 5) in four readings that must agree: the pure
Python decoder, the oracle (tests/lz4_oracle.cpp), the device's inflate routine built for the CPU under AddressSanitizer
(tikv_b200/csrc/lz4_block.h through tests/lz4_block_emul.cpp) and, when the machine has it, liblz4 itself.  Golden
blocks compressed by liblz4 pin all of them on machines without it."""
import os
import random
import sys

import pytest

import kvfmt
import scenarios as sc
import sstfmt
import sstlz4 as z

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import gen_lz4_blocks  # noqa: E402

LIB = z.liblz4()


def seq(lit, offset=None, match=None):
    """one LZ4 sequence: literals, then (unless last) a match of `match` bytes at `offset`"""
    n, m = len(lit), (match - 4 if match is not None else 0)
    out = bytes([(min(n, 15) << 4) | min(m, 15)])
    if n >= 15:
        r = n - 15
        out += b"\xff" * (r // 255) + bytes([r % 255])
    out += lit
    if match is not None:
        out += bytes([offset & 0xFF, offset >> 8])
        if m >= 15:
            r = m - 15
            out += b"\xff" * (r // 255) + bytes([r % 255])
    return out


def expand(parts):
    """the bytes a stream of (literals, offset, match) sequences stands for, the slow obvious way"""
    out = bytearray()
    for lit, off, ml in parts:
        out += lit
        for _ in range(ml or 0):
            out.append(out[-off])
    return bytes(out)


def stream(parts):
    return b"".join(seq(lit, off, ml) for lit, off, ml in parts)


TAIL = (b"end of block", None, None)  # the last match starts 12 bytes or more before the end (the format's rule): liblz4 reads it too


def hand_streams():
    rng = random.Random(4)
    pre = bytes(rng.randrange(256) for _ in range(70000))
    out = {"literals_only": [(b"hello, world", None, None)],
           "rle_offset1_4+15+255+7": [(b"a", 1, 4 + 15 + 255 + 7), TAIL],
           "literal_run_15+255+0": [(bytes(range(256)) + bytes(14), 1, 4), TAIL],
           "offset_65535": [(pre[:65535], 65535, 9), TAIL],
           "match_back_to_byte_0": [(b"abcdefgh", 8, 8), (b"x", 17, 30), TAIL]}
    for d in range(1, 41):
        out["offset_%d" % d] = [(pre[:d] if d > 4 else pre[:d] * 2, d, 4 + d * 3 + 1), TAIL]
    return out


def all_decoders(contents, exp_raw):
    """every reading of one block's stored contents (varint size | LZ4 block) -> assert each gives exp_raw (None: corrupt)"""
    assert z.inflate_contents(contents) == exp_raw
    assert z.py_inflate_contents(contents) == exp_raw


@pytest.mark.parametrize("name", sorted(hand_streams()))
def test_hand_assembled_streams(name):
    parts = hand_streams()[name]
    s, exp = stream(parts), expand(parts)
    assert z.py_decompress(s, len(exp)) == exp
    assert z.decompress(s, len(exp)) == exp
    if LIB is not None:
        assert z.lz4_decompress_safe(LIB, s, len(exp)) == exp
    contents = z.frame(exp, s)
    all_decoders(contents, exp)
    assert z.emul([contents]) == [exp]
    # and one byte short / long of the declared size is corrupt in every reading
    for size in (len(exp) - 1, len(exp) + 1):
        bad = z.var32(size) + s
        all_decoders(bad, None)
        assert z.emul([bad]) == [None]


def test_golden_blocks_from_liblz4():
    blocks = gen_lz4_blocks.load()
    assert len(blocks) >= 8
    contents, exps = [], []
    for name, raw, lz4, hc in blocks:
        for payload in (lz4, hc):
            assert z.py_decompress(payload, len(raw)) == raw, name
            assert z.decompress(payload, len(raw)) == raw, name
            if LIB is not None:
                assert z.lz4_decompress_safe(LIB, payload, len(raw)) == raw
            contents.append(z.frame(raw, payload))
            exps.append(raw)
        # the blocks themselves are RocksDB data blocks: the iterator reads them
        rc, kvs = sstfmt.decode(raw + b"\0" * 5, [0, len(raw) + 5])
        assert rc == 0 and kvs, name
    assert z.emul(contents) == exps


OPTS = [dict(), dict(restart_interval=1), dict(restart_interval=3, block_size=700), dict(block_size=0, entries_per_block=37),
        dict(key_prefix_len=3, key_prefix_byte=0x7a)]


@pytest.mark.parametrize("opts", OPTS)
def test_oracle_compressor_round_trips(opts):
    host = sc.dirty_region(5, n_keys=700).build(read_ts=sc.READ_TS)
    fmt = {k: opts[k] for k in ("key_prefix_len", "key_suffix_len") if k in opts}
    for blk in host.wblocks + [host.dblock]:
        plain, poffs = sstfmt.build(blk, **opts)
        data, offs = z.build(blk, **opts)
        assert len(offs) == len(poffs)
        types = z.block_types(data, offs)
        assert set(types) <= {0, 4}
        assert z.decode(data, offs, **fmt) == (0, blk.kvs)
        st, inflated, ioffs = z.inflate_run(data, offs)
        assert st == 0 and inflated == plain and ioffs == poffs
        contents = [data[a:b - 5] for a, b, t in zip(offs, offs[1:], types) if t == 4]
        raws = [plain[a:b - 5] for a, b, t in zip(poffs, poffs[1:], types) if t == 4]
        for c, r in zip(contents, raws):
            assert len(c) < len(r) - len(r) // 8  # RocksDB's rule for storing a block compressed
            assert z.py_inflate_contents(c) == r
            if LIB is not None:
                at = len(z.var32(len(r)))
                assert z.lz4_decompress_safe(LIB, c[at:], len(r)) == r
        assert z.emul(contents) == raws


def test_incompressible_blocks_stay_plain_and_runs_mix():
    rng = random.Random(8)
    kvs = []
    for i in range(600):
        v = bytes(rng.randrange(256) for _ in range(200)) if (i // 40) % 2 else b"row %d " % i * 20
        kvs.append((b"t%06d" % i, v))
    blk = kvfmt.HostBlock(kvs)
    data, offs = z.build(blk, block_size=4096)
    types = z.block_types(data, offs)
    assert 0 in types and 4 in types, types
    assert z.decode(data, offs) == (0, blk.kvs)


def small_compressed():
    blk = kvfmt.HostBlock([(b"key%03d" % i, b"value value %d" % (i % 3)) for i in range(12)])
    plain, poffs = sstfmt.build(blk, restart_interval=4)
    data, offs = z.compress_run(plain, poffs, force=True)
    assert len(offs) == 2
    return blk, plain[:-5], data[:-5]


def damaged_corpus():
    """compressed contents of one small block, damaged every way the format allows: (label, contents)"""
    _, raw, good = small_compressed()
    at = len(z.var32(len(raw)))
    payload = good[at:]
    out = [("good", good)]
    out += [("truncated_%d" % n, good[:n]) for n in range(len(good))]
    out += [("size%+d" % d, z.var32(len(raw) + d) + payload) for d in (-1, 1)]
    out += [("size_zero", b"\0" + payload), ("size_huge", z.var32(1 << 31) + payload), ("size_unterminated", b"\xff" * 5 + payload)]
    # a stream whose first match has offset 0, then one past the bytes produced so far
    lit = raw[:20]
    for name, off in (("offset_0", 0), ("offset_past_output", 21)):
        s = seq(lit, off, 8) + seq(raw[28:])
        out.append((name, z.var32(len(raw)) + s))
    out.append(("literals_past_payload", z.var32(len(raw)) + bytes([0xF0, 200]) + raw[:50]))
    out.append(("match_past_size", z.var32(40) + seq(raw[:20], 1, 30) + seq(b"12345")))
    out.append(("trailing_bytes", good + b"\0"))
    out.append(("trailing_sequence", good + seq(b"x")))
    rng = random.Random(12)
    for i in range(300):
        bad = bytearray(good)
        for _ in range(1 + i % 3):
            bad[rng.randrange(len(bad))] ^= 1 << rng.randrange(8)
        out.append(("flip_%d" % i, bytes(bad)))
    return raw, out


def test_damaged_blocks_same_verdict_in_every_reading():
    raw, corpus = damaged_corpus()
    got = z.emul([c for _, c in corpus])
    n_bad = 0
    for (label, c), dev in zip(corpus, got):
        exp = z.inflate_contents(c)
        assert dev == exp, label
        assert z.py_inflate_contents(c) == exp, label
        n_bad += exp is None
        if label == "good":
            assert exp == raw
        elif not label.startswith("flip_"):
            assert exp is None, label
    assert n_bad > 300


def test_damaged_blocks_in_a_run():
    """the oracle's block reader: corrupt LZ4 contents are a corrupted block (status 1) inside a run"""
    _, corpus = damaged_corpus()
    for label, c in corpus[:40]:
        st, kvs = z.decode(c + b"\x04" + b"\0" * 4, [0, len(c) + 5])
        exp = z.inflate_contents(c)
        assert st == (0 if exp is not None else 1), label


def test_unsupported_and_unknown_compression_types():
    blk, raw, good = small_compressed()
    assert z.decode(good + b"\x04" + b"\0" * 4, [0, len(good) + 5]) == (0, blk.kvs)
    assert z.decode(good + b"\x05" + b"\0" * 4, [0, len(good) + 5]) == (0, blk.kvs)  # LZ4HC: the same stream format
    # Snappy, zlib, BZip2, Xpress, ZSTD, ZSTD (not final) and RocksDB's custom-compressor range: the host may inflate them
    for t in (1, 2, 3, 6, 7, 0x40, 0x80, 200, 0xFE):
        assert z.decode(good + bytes([t]) + b"\0" * 4, [0, len(good) + 5])[0] == 2
    for t in (8, 0x3F, 0x41, 0x7F, 0xFF):  # values no RocksDB writer stores: a damaged block
        assert z.decode(good + bytes([t]) + b"\0" * 4, [0, len(good) + 5])[0] == 1
    # without a trailer there is no type byte: the contents are plain
    assert z.decode(raw, [0, len(raw)], trailer_len=0) == (0, blk.kvs)
