"""Regenerates tests/golden/lz4_blocks.json: RocksDB data blocks of a few scenario regions, compressed by the LZ4 library
RocksDB links (liblz4: LZ4_compress_default, and LZ4_compress_HC at level 12 for kLZ4HCCompression), with their
uncompressed bytes.  The file pins every LZ4 decoder of the project (the device's, the oracle's, the Python one) to
the library's output on machines that do not have it.  Needs liblz4.so.1.  Run from the repo root:
python tests/golden/gen_lz4_blocks.py"""
import base64
import ctypes as C
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import kvfmt  # noqa: E402
import scenarios as sc  # noqa: E402
import sstfmt  # noqa: E402
import sstlz4  # noqa: E402

HC_LEVEL = 12


def long_key_block():
    rng = random.Random(17)
    kvs = []
    for i in range(400):
        stem = b"k%06d" % i
        kvs.append((stem + bytes(rng.randrange(97, 100) for _ in range(rng.choice((130, 200, 400)))), bytes(rng.randrange(4) for _ in range(rng.choice((0, 8, 60))))))
    return kvfmt.HostBlock(kvs)


def cases():
    """(name, plain data blocks with trailers, their offsets, max blocks kept)"""
    dirty = sc.dirty_region(21, n_keys=300).build(read_ts=sc.READ_TS)
    v1 = sc.dirty_region(22, n_keys=300, only_fmt=1).build(read_ts=sc.READ_TS)
    return [("dirty_region", *sstfmt.build(dirty.wblocks[0], block_size=4096), 3),
            ("dirty_region_default_cf", *sstfmt.build(dirty.dblock, block_size=4096), 1),
            ("v1_rows", *sstfmt.build(v1.wblocks[0], block_size=4096), 2),
            ("long_keys", *sstfmt.build(long_key_block(), block_size=4096, restart_interval=4), 2)]


def main():
    L = sstlz4.liblz4()
    assert L is not None, "needs liblz4.so.1"
    out = []
    for name, data, offs, keep in cases():
        for b in range(min(keep, len(offs) - 1)):
            raw = data[offs[b]:offs[b + 1] - 5]
            cap = len(raw) + len(raw) // 255 + 64
            dst = C.create_string_buffer(cap)
            n = L.LZ4_compress_default(raw, dst, len(raw), cap)
            lz4 = dst.raw[:n]
            n = L.LZ4_compress_HC(raw, dst, len(raw), cap, HC_LEVEL)
            hc = dst.raw[:n]
            assert lz4 and hc and sstlz4.lz4_decompress_safe(L, lz4, len(raw)) == raw == sstlz4.lz4_decompress_safe(L, hc, len(raw))
            out.append({"name": "%s/%d" % (name, b), "raw": base64.b64encode(raw).decode(), "lz4": base64.b64encode(lz4).decode(),
                        "lz4hc": base64.b64encode(hc).decode()})
    with open(os.path.join(HERE, "lz4_blocks.json"), "w") as f:
        json.dump({"generator": "liblz4 LZ4_compress_default / LZ4_compress_HC level %d" % HC_LEVEL,
                   "format": "raw: data block contents without the trailer (key prefix 'z', internal-key footer); lz4 / lz4hc: the raw LZ4 block of raw, base64",
                   "blocks": out}, f, indent=0)
        f.write("\n")


def load():
    """[(name, raw, lz4 payload, lz4hc payload)] from the committed file"""
    with open(os.path.join(HERE, "lz4_blocks.json")) as f:
        return [(b["name"], base64.b64decode(b["raw"]), base64.b64decode(b["lz4"]), base64.b64decode(b["lz4hc"])) for b in json.load(f)["blocks"]]


if __name__ == "__main__":
    main()
