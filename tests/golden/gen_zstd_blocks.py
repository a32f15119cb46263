"""Regenerates tests/golden/zstd_blocks.json: RocksDB data blocks compressed by libzstd (the library RocksDB links for
kZSTD) at several levels and parameters, and a damaged corpus stored as edits of a few base frames, each with
libzstd's verdict.  The file pins the device's ZSTD routine to the library on machines that do not have it.  Needs
libzstd.so.1 (written with 1.5.5).  Run from the repo root:  python tests/golden/gen_zstd_blocks.py

Blocks:  [name, raw_sha256, [[params, base64 frame], ...]]; the raw block is rebuilt by blocks() from the
         scenario generators (deterministic) and checked against its SHA-256
Damaged: [label, base (index into "bases": block contents, varint | frame), edits, verdict (0 decoded, 1 corrupted,
         2 unsupported), SHA-256 of the output when decoded]
Edits, applied in order: ["cut", n] keep n bytes; ["xor", at, mask]; ["set", at, hex] overwrite; ["ins", at, hex];
         ["del", at, n]."""
import base64
import hashlib
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import gen_lz4_blocks  # noqa: E402
import kvfmt  # noqa: E402
import sstfmt  # noqa: E402
import sstzstd as z  # noqa: E402

LEVELS = (-5, 1, 3, 9, 19, 22)
VARIANTS = [dict(checksum=1), dict(contentSize=0), dict(windowLog=10), dict(targetCBlockSize=1300), dict(literalCompressionMode=2),
            dict(targetCBlockSize=1300, checksum=1, level=19)]


def one_block(kvs, **opts):
    data, offs = sstfmt.build(kvfmt.HostBlock(kvs), block_size=0, entries_per_block=len(kvs), **opts)
    assert len(offs) == 2
    return data[:-5]


def big_block(recipe):
    """a 300 KB zero value (RLE blocks, a multi-block frame) and a 2 KB random value (a Raw block)"""
    if recipe == "zero_value_300k":
        return one_block([(b"k%04d" % i, bytes(300_000) if i == 3 else b"v%d" % i) for i in range(8)])
    assert recipe == "random_value_2k"
    return one_block([(b"k%04d" % i, random.Random(5).randbytes(2000) if i == 1 else b"v%d" % i) for i in range(4)])


def small_block():
    """a block of 3-4 KB"""
    rng = random.Random(9)
    return one_block([(b"key%05d" % i, b"value %d " % rng.randrange(50) * rng.randrange(1, 6)) for i in range(100)])


def tiny_block():
    return one_block([(b"key%03d" % i, b"value value %d" % (i % 3)) for i in range(12)], restart_interval=4)


def blocks():
    """(name, raw) of every block of the corpus"""
    out = []
    for name, data, offs, keep in gen_lz4_blocks.cases():
        for b in range(min(keep, len(offs) - 1)):
            out.append(("%s/%d" % (name, b), data[offs[b]:offs[b + 1] - 5]))
    out.append(("small_3k", small_block()))
    out.append(("tiny", tiny_block()))
    out += [(r, big_block(r)) for r in ("zero_value_300k", "random_value_2k")]
    return out


ALL = [dict(level=lv) for lv in LEVELS] + [dict(dict(level=3), **v) for v in VARIANTS]
# which frames each block keeps: every level and variant for one 4 KB block, a level or two for the others
FRAMES = {"long_keys/0": ALL, "dirty_region/0": [dict(level=3)], "dirty_region_default_cf/0": [dict(level=3)], "v1_rows/0": [dict(level=3)],
          "small_3k": [dict(level=3), dict(level=19)], "tiny": [dict(level=3), dict(level=19)],
          "zero_value_300k": [dict(level=3, checksum=1, contentSize=0)], "random_value_2k": [dict(level=3)]}


def damaged():
    """(bases, [(label, base index, edits)])"""
    tiny = tiny_block()
    b0 = z.frame(tiny, level=3, checksum=1)                       # single segment, checksum
    b1 = z.frame(blocks()[0][1], level=19)                        # Huffman + FSE tables
    b2 = z.frame(blocks()[0][1], level=3, windowLog=12)           # windowed
    bases = [b0, b1, b2]
    at0 = len(z.var32(len(tiny)))
    fhd0 = at0 + 4
    out = [("good_%d" % i, i, []) for i in range(len(bases))]
    out += [("truncated_%d" % n, 0, [["cut", n]]) for n in range(len(b0))]
    for d in (-1, 1):
        out.append(("size%+d" % d, 0, [["del", 0, at0], ["ins", 0, z.var32(len(tiny) + d).hex()]]))
    out.append(("size_zero", 0, [["del", 0, at0], ["ins", 0, "00"]]))
    out.append(("size_huge", 0, [["del", 0, at0], ["ins", 0, z.var32(1 << 31).hex()]]))
    out.append(("size_unterminated", 0, [["del", 0, at0], ["ins", 0, "ffffffffff"]]))
    out.append(("checksum_wrong", 0, [["xor", len(b0) - 1, 0x40]]))
    out.append(("fcs_wrong", 0, [["xor", fhd0 + 1, 0x01]]))
    out.append(("reserved_bit", 0, [["xor", fhd0, 0x08]]))
    out.append(("dictionary_id", 0, [["xor", fhd0, 0x01], ["ins", fhd0 + 1, "07"]]))
    out.append(("dictionary_id_zero", 0, [["xor", fhd0, 0x01], ["ins", fhd0 + 1, "00"]]))
    out.append(("magic_missing", 0, [["xor", at0, 0x01]]))
    out.append(("skippable_frame", 0, [["set", at0, "505d2a18"]]))
    out.append(("trailing_byte", 0, [["ins", len(b0), "00"]]))
    out.append(("trailing_frame", 0, [["ins", len(b0), b0[at0:].hex()]]))
    at2 = len(b2) - len(z.split(b2)[1])
    assert not z.header(z.split(b2)[1])["single"]
    for wd in (0x00, 0x07, 0x08, 0xA8, 0xAF, 0xB0, 0xFF):
        out.append(("window_desc_%02x" % wd, 2, [["set", at2 + 5, "%02x" % wd]]))
    rng = random.Random(12)
    for i in range(300):
        base = 1 if i % 3 else 0
        n = len(bases[base])
        out.append(("flip_%d" % i, base, [["xor", rng.randrange(n), 1 << rng.randrange(8)] for _ in range(1 + i % 3)]))
    return bases, out


def apply(contents, edits):
    c = bytearray(contents)
    for e in edits:
        if e[0] == "cut":
            del c[e[1]:]
        elif e[0] == "xor":
            c[e[1]] ^= e[2]
        elif e[0] == "set":
            b = bytes.fromhex(e[2])
            c[e[1]:e[1] + len(b)] = b
        elif e[0] == "ins":
            c[e[1]:e[1]] = bytes.fromhex(e[2])
        else:
            assert e[0] == "del"
            del c[e[1]:e[1] + e[2]]
    return bytes(c)


def main():
    L = z.libzstd()
    assert L is not None, "needs libzstd.so.1"
    b64 = lambda b: base64.b64encode(b).decode()  # noqa: E731
    out = []
    for name, raw in blocks():
        if name in FRAMES:
            fr = [(c, z.compress(raw, **c)) for c in FRAMES[name]]
            assert all(z.decompress(p, len(raw)) == raw for _, p in fr)
            out.append([name, hashlib.sha256(raw).hexdigest(), [[c, b64(p)] for c, p in fr]])
    bases, muts = damaged()
    dam = []
    for label, base, edits in muts:
        v, got = z.reference_verdict(apply(bases[base], edits))
        dam.append([label, base, edits, v, hashlib.sha256(got).hexdigest() if v == z.OK else None])
    lines = lambda xs: ",\n".join(json.dumps(x) for x in xs)  # noqa: E731  (one entry per line)
    with open(os.path.join(HERE, "zstd_blocks.json"), "w") as f:
        f.write('{"generator": %s,\n"format": %s,\n"blocks": [\n%s],\n"bases": [\n%s],\n"damaged": [\n%s]}\n' % (
            json.dumps("libzstd %d ZSTD_compress2; verdicts: ZSTD_decompress into exactly the declared size" % L.ZSTD_versionNumber()),
            json.dumps(__doc__.split("\n\n", 1)[1]), lines(out), lines(b64(b) for b in bases), lines(dam)))


def load():
    """(blocks: [(name, raw, [(params, payload)])], damaged: [(label, contents, verdict, sha256)]) from the committed file"""
    with open(os.path.join(HERE, "zstd_blocks.json")) as f:
        j = json.load(f)
    raws = dict(blocks())
    blks = []
    for name, sha, frames in j["blocks"]:
        raw = raws[name]
        assert hashlib.sha256(raw).hexdigest() == sha, name
        blks.append((name, raw, [(c, base64.b64decode(p)) for c, p in frames]))
    bases = [base64.b64decode(b) for b in j["bases"]]
    dam = [(label, apply(bases[base], edits), v, sha) for label, base, edits, v, sha in j["damaged"]]
    return blks, dam


if __name__ == "__main__":
    main()
