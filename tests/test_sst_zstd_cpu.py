"""`-m "not gpu"`: ZSTD data blocks (RocksDB compression types 7 / 0x40) through the device's routine built for the CPU
under AddressSanitizer (tikv_b200/csrc/zstd_block.h through tests/zstd_block_emul.cpp), against libzstd's output and
verdicts committed in tests/golden/zstd_blocks.json and, when the machine has it, libzstd itself."""
import hashlib
import os
import sys

import pytest

import kvfmt
import scenarios as sc
import sstfmt
import sstzstd as z
from sstzstd import BitWriter, block_header

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import gen_zstd_blocks  # noqa: E402

LIB = z.libzstd()

# Damaged entries libzstd 1.5.5 decodes and the device rejects (B2_ERR_STORAGE).  No RocksDB writer produces them:
# - window_desc_00 / 07 / 08: a window shrunk below the frame's 4 KiB block.  The device keeps RFC 8878's
#   Block_Maximum_Size = min(Window_Size, 128 KiB); libzstd's one-shot decoder only bounds a block by 128 KiB.
# - the flips below: a Huffman literals stream that does not end exactly on its last code (bits left over, or read past
#   its start).  The device requires every bitstream to be consumed exactly; libzstd's double-symbol and fast Huffman
#   decoders let the last code overrun or stop short.  An encoder writes exactly the bits of its codes.
DEVICE_STRICTER = {"window_desc_00", "window_desc_07", "window_desc_08"} | {"flip_%d" % i for i in (
    29, 46, 52, 53, 56, 59, 61, 62, 65, 71, 77, 89, 104, 118, 121, 124, 131, 134, 140, 148, 151, 166, 173, 176, 178, 179, 191, 194,
    197, 202, 209, 226, 232, 233, 235, 244, 245, 251, 257, 271, 274, 280, 283, 292, 296)}


def hand_frames():
    """(name, payload, expected bytes): frames libzstd does not emit on its own"""
    out = []
    # RLE literals; LL, OF and ML all in RLE mode (no state bits: the stream holds the offsets' extra bits only);
    # an 8-byte Frame_Content_Size in a single-segment frame
    bw = BitWriter().read(3, 2).read(0, 2)  # offsets 1 + 3 = 4, then 1 + 0 = 1 (OF code 2: 4 + two bits - 3)
    blk = bytes([10 << 3 | 1]) + b"a" + bytes([2, 1 << 6 | 1 << 4 | 1 << 2, 4, 2, 2]) + bw.bytes()
    out.append(("rle_literals_rle_tables_fcs8", b"\x28\xb5\x2f\xfd" + bytes([3 << 6 | 1 << 5]) + (20).to_bytes(8, "little") + block_header(1, 2, len(blk)) + blk, b"a" * 20))
    # Raw literals then the same RLE tables with a new offset and a repeat offset (code 0, literal length 4: rep0)
    lit = b"abcdefghij"
    bw = BitWriter().read(1, 2)
    blk1 = z.raw_literals(lit) + bytes([1, 1 << 6 | 1 << 4 | 1 << 2, 4, 2, 2]) + bw.bytes()  # "abcd" + 5 bytes at offset 2
    bw = BitWriter()
    blk2 = z.raw_literals(b"XY") + bytes([1, 1 << 6 | 1 << 4 | 1 << 2, 2, 0, 3]) + bw.bytes()  # "XY" + 6 bytes at rep0 = 2
    exp = bytearray(b"abcd")
    for _ in range(5):
        exp.append(exp[-2])
    exp += b"efghij" + b"XY"
    for _ in range(6):
        exp.append(exp[-2])
    out.append(("repeat_offset_across_blocks", z.frame_header(len(exp), window_desc=0) + block_header(0, 2, len(blk1)) + blk1 + block_header(1, 2, len(blk2)) + blk2,
                bytes(exp)))
    # Huffman literals over {0, 1} with direct 4-bit weights (symbol 0: weight 1, symbol 1 implied), four streams; then
    # Treeless literals with one stream and with four (the last one empty); a 1-byte Frame_Content_Size
    lits = [bytes([0, 1, 1, 0, 1, 1, 1, 0]), bytes([1, 0, 0, 1, 1]), bytes([1, 1, 0, 1, 0, 0])]

    def stream(bits):
        w = BitWriter()
        for b in bits:
            w.read(b, 1)
        return w.bytes()

    def four(lit):
        seg = (len(lit) + 3) // 4
        ss = [stream(lit[i * seg:(i + 1) * seg]) for i in range(3)] + [stream(lit[3 * seg:])]
        return b"".join(len(s).to_bytes(2, "little") for s in ss[:3]) + b"".join(ss)

    def lit_header(lt, sf, n, c):
        return (lt | sf << 2 | n << 4 | c << 14).to_bytes(3, "little")
    tree = bytes([128, 0x10])
    body0 = tree + four(lits[0])
    body1 = stream(lits[1])
    body2 = four(lits[2])
    blocks = [lit_header(2, 1, 8, len(body0)) + body0 + b"\0", lit_header(3, 0, 5, len(body1)) + body1 + b"\0", lit_header(3, 1, 6, len(body2)) + body2 + b"\0"]
    exp = b"".join(lits)
    out.append(("direct_weights_treeless", z.frame_header(len(exp)) + b"".join(block_header(i == 2, 2, len(b)) + b for i, b in enumerate(blocks)), exp))
    return out


def golden_cases():
    blks, _ = gen_zstd_blocks.load()
    return [(name, p, raw) for name, raw, frames in blks for _, p in frames]


def test_golden_and_hand_frames_decode():
    cases = golden_cases() + hand_frames()
    assert len(cases) > 20
    got = z.emul([z.var32(len(raw)) + p for _, p, raw in cases])
    for (name, p, raw), g in zip(cases, got):
        assert g == (z.OK, raw), name
        if LIB is not None:
            assert z.decompress(p, len(raw)) == raw, name


def test_corpus_covers_the_format():
    feats = set()
    for _, p, _ in golden_cases() + hand_frames():
        feats |= z.features(p)
    need = {"raw_block", "rle_block", "compressed_block", "multi_block", "raw_literals", "rle_literals", "huffman_literals_1_streams",
            "huffman_literals_4_streams", "treeless_literals_1_streams", "treeless_literals_4_streams", "huffman_weights_fse",
            "huffman_weights_direct", "zero_sequences", "checksum", "no_checksum", "single_segment", "windowed",
            "fcs_0", "fcs_1", "fcs_2", "fcs_4", "fcs_8"}
    need |= {"%s_%s" % (t, m) for t in ("ll", "of", "ml") for m in ("predefined", "rle", "fse", "repeat")}
    assert need <= feats, sorted(need - feats)


def test_damaged_corpus_gets_libzstds_verdict():
    _, dam = gen_zstd_blocks.load()
    assert len(dam) > 400
    got = z.emul([c for _, c, _, _ in dam])
    seen = set()
    for (label, c, verdict, sha), (v, out) in zip(dam, got):
        if label in DEVICE_STRICTER:
            assert verdict == z.OK and v == z.CORRUPT, label
            seen.add(label)
            continue
        assert v == verdict, label
        assert (hashlib.sha256(out).hexdigest() if out is not None else None) == sha, label
        if LIB is not None:
            rv, rout = z.reference_verdict(c)
            assert rv == verdict and (rout is None or hashlib.sha256(rout).hexdigest() == sha), label
    assert seen == DEVICE_STRICTER
    labels = {d[0]: d[2] for d in dam}
    for name in ("magic_missing", "skippable_frame", "dictionary_id"):
        assert labels[name] == z.UNSUPPORTED, name
    for name in ("size-1", "size+1", "size_zero", "size_huge", "size_unterminated", "checksum_wrong", "fcs_wrong", "reserved_bit",
                 "trailing_byte", "trailing_frame", "window_desc_b0", "window_desc_ff"):
        assert labels[name] == z.CORRUPT, name


def small_block():
    blk = kvfmt.HostBlock([(b"key%03d" % i, b"value value %d" % (i % 3)) for i in range(12)])
    plain, poffs = sstfmt.build(blk, restart_interval=4)
    return blk, plain[:-5]


def test_type_classification():
    """7 and 0x40 decode; a payload without the magic (LZ4 contents under a ZSTD type) and a dictionary are unsupported"""
    blk, raw = small_block()
    _, dam = gen_zstd_blocks.load()
    good = [c for label, c, _, _ in dam if label == "good_0"][0]
    for t in (z.ZSTD, z.ZSTD_NOT_FINAL):
        assert z.decode(good + bytes([t]) + b"\0" * 4, [0, len(good) + 5]) == (0, blk.kvs)
    import sstlz4
    lz4_contents = sstlz4.frame(raw)
    assert z.emul([lz4_contents])[0][0] == z.UNSUPPORTED
    assert z.reference_verdict(lz4_contents)[0] == z.UNSUPPORTED
    dict_frame = [c for label, c, _, _ in dam if label == "dictionary_id"][0]
    assert z.emul([dict_frame])[0][0] == z.UNSUPPORTED


@pytest.mark.skipif(LIB is None, reason="needs libzstd.so.1 to compress at run time")
@pytest.mark.parametrize("level", [-5, 1, 3, 19])
def test_compress_run_round_trips(level):
    host = sc.dirty_region(5, n_keys=700).build(read_ts=sc.READ_TS)
    for blk in host.wblocks + [host.dblock]:
        plain, poffs = sstfmt.build(blk)
        data, offs = z.build(blk, level=level)
        types = z.block_types(data, offs)
        assert set(types) <= {0, z.ZSTD} and len(offs) == len(poffs)
        assert z.decode(data, offs) == (0, blk.kvs)
        st, inflated, ioffs = z.inflate_run(data, offs)
        assert st == 0 and inflated == plain and ioffs == poffs
        contents = [data[a:b - 5] for a, b, t in zip(offs, offs[1:], types) if t == z.ZSTD]
        raws = [plain[a:b - 5] for a, b, t in zip(poffs, poffs[1:], types) if t == z.ZSTD]
        for c, r in zip(contents, raws):
            assert len(c) < len(r) - len(r) // 8  # RocksDB's rule for storing a block compressed
        assert z.emul(contents) == [(z.OK, r) for r in raws]
