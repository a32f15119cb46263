"""ZSTD-compressed RocksDB data blocks (compression types 7 kZSTD / 0x40 kZSTDNotFinalCompression, format_version >= 2
framing: varint32 uncompressed size | ZSTD frame).  TEST INFRASTRUCTURE, two readings of the format:
- libzstd (ZSTD_compress2 / ZSTD_decompress), when the machine has libzstd.so.1; the golden corpus
  (tests/golden/zstd_blocks.json) pins its output and its verdicts for machines that do not;
- the device's routine (tikv_b200/csrc/zstd_block.h) built for the CPU under AddressSanitizer (emul).
Also: RocksDB's table-builder step with ZSTD (the 12.5 % rule), a walker over frame and block headers that tallies the
features a frame uses, and a bit writer for frames assembled by hand."""
import ctypes as C
import os
import struct
import subprocess
import tempfile

import sstfmt
from sstlz4 import BUILD, ROOT, _built, block_types, var32  # noqa: F401  (block_types: re-exported for the tests)

EMUL_SRC = os.path.join(ROOT, "tests", "zstd_block_emul.cpp")
DEVICE_HDR = os.path.join(ROOT, "tikv_b200", "csrc", "zstd_block.h")
ZSTD, ZSTD_NOT_FINAL = 7, 0x40
MAGIC = b"\x28\xb5\x2f\xfd"
OK, CORRUPT, UNSUPPORTED = 0, 1, 2

# ZSTD_cParameter ids of libzstd 1.5.5 (zstd.h; the last two are experimental)
PARAMS = {"level": 100, "windowLog": 101, "checksum": 201, "contentSize": 200, "dictID": 202,
          "literalCompressionMode": 1002, "targetCBlockSize": 1003}
_zstd = False


def libzstd():
    """the system's libzstd, or None"""
    global _zstd
    if _zstd is False:
        try:
            L = C.CDLL("libzstd.so.1")
            L.ZSTD_createCCtx.restype = C.c_void_p
            L.ZSTD_freeCCtx.argtypes = [C.c_void_p]
            L.ZSTD_CCtx_setParameter.argtypes, L.ZSTD_CCtx_setParameter.restype = [C.c_void_p, C.c_int, C.c_int], C.c_size_t
            L.ZSTD_compress2.argtypes, L.ZSTD_compress2.restype = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t], C.c_size_t
            L.ZSTD_decompress.argtypes, L.ZSTD_decompress.restype = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t], C.c_size_t
            L.ZSTD_isError.argtypes, L.ZSTD_isError.restype = [C.c_size_t], C.c_uint
            L.ZSTD_compressBound.argtypes, L.ZSTD_compressBound.restype = [C.c_size_t], C.c_size_t
            L.ZSTD_versionNumber.restype = C.c_uint
            _zstd = L
        except OSError:
            _zstd = None
    return _zstd


def compress(raw, level=3, **params):
    """raw bytes -> one ZSTD frame by libzstd's ZSTD_compress2 (params: PARAMS names)"""
    L = libzstd()
    assert L is not None, "needs libzstd.so.1"
    cc = L.ZSTD_createCCtx()
    try:
        for k, v in dict(params, level=level).items():
            assert not L.ZSTD_isError(L.ZSTD_CCtx_setParameter(cc, PARAMS[k], int(v))), k
        cap = L.ZSTD_compressBound(len(raw))
        dst = C.create_string_buffer(cap)
        n = L.ZSTD_compress2(cc, dst, cap, bytes(raw), len(raw))
        assert not L.ZSTD_isError(n)
        return dst.raw[:n]
    finally:
        L.ZSTD_freeCCtx(cc)


def decompress(payload, size):
    """libzstd's reading of a block's frame as RocksDB's reader does it (ZSTD_decompress into exactly the declared size):
    the bytes, or None when it fails or produces another size"""
    L = libzstd()
    dst = C.create_string_buffer(max(size, 1))
    r = L.ZSTD_decompress(dst, size, bytes(payload), len(payload))
    return dst.raw[:size] if not L.ZSTD_isError(r) and r == size else None


def frame(raw, payload=None, **kw):
    """the stored contents of a compressed block: varint32 len(raw) | ZSTD frame (libzstd's unless `payload` is given)"""
    return var32(len(raw)) + (compress(raw, **kw) if payload is None else payload)


def split(contents):
    """(declared size, payload) of block contents, or None when the varint is malformed"""
    v = 0
    for i in range(min(5, len(contents))):
        v |= (contents[i] & 0x7F) << (7 * i)
        if not contents[i] & 0x80:
            return v & 0xFFFFFFFF, bytes(contents[i + 1:])
    return None


def reference_verdict(contents):
    """libzstd's verdict on block contents, under the contract's framing rules: (OK, bytes) / (CORRUPT, None) /
    (UNSUPPORTED, None)"""
    s = split(contents)
    if s is None:
        return CORRUPT, None
    size, payload = s
    if payload[:4] != MAGIC:
        return UNSUPPORTED, None
    if size < 4 or size > 1 << 30:
        return CORRUPT, None
    h = header(payload)
    if h is not None and h["dict_id"]:
        return UNSUPPORTED, None
    out = decompress(payload, size)
    return (OK, out) if out is not None else (CORRUPT, None)


def compress_run(data, offs, level=3, type_byte=ZSTD, force=False, **params):
    """a run of plain blocks with 5-byte trailers -> the run RocksDB's table builder stores with ZSTD: each block compressed
    when that saves at least 1/8 of it (force: always), else kept plain"""
    out, noffs = bytearray(), [0]
    for a, b in zip(offs, offs[1:]):
        raw = bytes(data[a:b - 5])
        c = frame(raw, level=level, **params)
        if force or len(c) < len(raw) - len(raw) // 8:
            out += c + bytes([type_byte]) + b"\0" * 4
        else:
            out += data[a:b]
        noffs.append(len(out))
    return bytes(out), noffs


def build(host_block, level=3, **opts):
    """sstfmt.build with the blocks stored as RocksDB stores them under ZSTD at `level`"""
    params = {k: opts.pop(k) for k in list(opts) if k in PARAMS}
    assert opts.get("trailer_len", 5) == 5, "compressed blocks carry their type in the trailer"
    data, offs = sstfmt.build(host_block, **opts)
    return compress_run(data, offs, level=level, **params)


def inflate_run(data, offs):
    """(status, data, offs) of the same run with every ZSTD block inflated by libzstd: 0 ok, 1 corrupted, 2 unsupported"""
    out, noffs = bytearray(), [0]
    for a, b in zip(offs, offs[1:]):
        t = data[b - 5]
        if t in (ZSTD, ZSTD_NOT_FINAL):
            st, raw = reference_verdict(data[a:b - 5])
            if st:
                return st, b"", []
            out += raw + b"\0" * 5
        else:
            out += data[a:b]
        noffs.append(len(out))
    return 0, bytes(out), noffs


def decode(data, offs, key_prefix_len=1, key_suffix_len=8):
    """(status, [(key, value)]): every ZSTD block inflated by libzstd, then the oracle's block iterator"""
    st, d, o = inflate_run(data, offs)
    if st:
        return st, []
    return sstfmt.decode(d, o, trailer_len=5, key_prefix_len=key_prefix_len, key_suffix_len=key_suffix_len)


def emul(contents_list):
    """Every compressed block contents through the device's frame() + inflate() built for the CPU (one lane) under
    AddressSanitizer: [(verdict, bytes or None)].  A read or write out of bounds fails the harness, and this."""
    exe = _built(os.path.join(BUILD, "zstd_block_emul"), [EMUL_SRC, DEVICE_HDR],
                 ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", EMUL_SRC])
    with tempfile.TemporaryDirectory() as td:
        cin, cout = os.path.join(td, "corpus"), os.path.join(td, "verdicts")
        with open(cin, "wb") as f:
            for c in contents_list:
                f.write(struct.pack("<I", len(c)) + bytes(c))
        r = subprocess.run([exe, cin, cout], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
        out, raw, p = [], open(cout, "rb").read(), 0
        while p < len(raw):
            v, size = raw[p], struct.unpack_from("<I", raw, p + 1)[0]
            p += 5
            out.append((v, raw[p:p + size] if v == OK else None))
            p += size
    assert len(out) == len(contents_list)
    return out


# ---- frame and block headers ----

def header(payload):
    """the frame header fields of a payload starting with the magic, or None when it is cut short"""
    if len(payload) < 5:
        return None
    fhd, q = payload[4], 5
    single, did_len = fhd >> 5 & 1, (0, 1, 2, 4)[fhd & 3]
    fcs_len = (single, 2, 4, 8)[fhd >> 6]
    if len(payload) < q + (not single) + did_len + fcs_len:
        return None
    wd = None
    if not single:
        wd = payload[q]
        q += 1
    did = int.from_bytes(payload[q:q + did_len], "little")
    q += did_len
    fcs = int.from_bytes(payload[q:q + fcs_len], "little") + (256 if fcs_len == 2 else 0) if fcs_len else None
    q += fcs_len
    return dict(single=single, checksum=fhd >> 2 & 1, dict_id=did, fcs_len=fcs_len, fcs=fcs, window_desc=wd, reserved=fhd >> 3 & 1, at=q)


def features(payload):
    """the set of format features a well-formed frame uses (for the corpus coverage check)"""
    h = header(payload)
    f = {"single_segment" if h["single"] else "windowed", "checksum" if h["checksum"] else "no_checksum", "fcs_%d" % h["fcs_len"]}
    q, n_blocks = h["at"], 0
    while True:
        bh = int.from_bytes(payload[q:q + 3], "little")
        q += 3
        t, size = bh >> 1 & 3, bh >> 3
        n_blocks += 1
        f.add(("raw", "rle", "compressed")[t] + "_block")
        if t == 2:
            blk = payload[q:q + size]
            lt, sf = blk[0] & 3, blk[0] >> 2 & 3
            if lt <= 1:
                lh = (1, 2, 1, 3)[sf]
                f.add(("raw", "rle")[lt] + "_literals")
            else:
                lh = (3, 3, 4, 5)[sf]
                v = int.from_bytes(blk[:lh], "little")
                w = {3: 10, 4: 14, 5: 18}[lh]
                csize = v >> (4 + w) & ((1 << w) - 1)
                f.add("%s_literals_%d_streams" % (("huffman", "treeless")[lt - 2], 1 if sf == 0 else 4))
                if lt == 2:
                    f.add("huffman_weights_" + ("direct" if blk[lh] >= 128 else "fse"))
                lh += csize
            if lt == 0:
                lh += (v := blk[0] >> 3 if sf in (0, 2) else (blk[0] >> 4) + (blk[1] << 4) + ((blk[2] << 12) if sf == 3 else 0))
            elif lt == 1:
                lh += 1
            s0 = blk[lh]
            if s0 == 0:
                f.add("zero_sequences")
            else:
                m = blk[lh + (1 if s0 < 128 else (2 if s0 < 255 else 3))]
                for name, mode in (("ll", m >> 6), ("of", m >> 4 & 3), ("ml", m >> 2 & 3)):
                    f.add("%s_%s" % (name, ("predefined", "rle", "fse", "repeat")[mode]))
            q += size
        else:
            q += 1 if t == 1 else size
        if bh & 1:
            break
    if n_blocks > 1:
        f.add("multi_block")
    return f


class BitWriter:
    """a backward bitstream assembled from the reads a decoder makes, in the order it makes them"""
    def __init__(self):
        self.reads = []

    def read(self, value, nbits):
        assert 0 <= value < 1 << nbits or nbits == 0 and value == 0
        self.reads.append((value, nbits))
        return self

    def bytes(self):
        acc, n = 0, 0
        for v, k in reversed(self.reads):  # the first read takes the highest bits
            acc |= v << n
            n += k
        acc |= 1 << n  # the end mark
        return (acc).to_bytes((n + 8) // 8, "little")


def block_header(last, btype, size):
    return (last | btype << 1 | size << 3).to_bytes(3, "little")


def frame_header(content_size=None, checksum=False, window_desc=None, dict_id=0):
    """magic | descriptor | window | dictionary id | content size: single segment when window_desc is None"""
    single = window_desc is None
    if content_size is None:
        fcs_flag, fcs = 0, b""
        assert not single
    elif single and content_size < 256:
        fcs_flag, fcs = 0, bytes([content_size])
    elif 256 <= content_size < 65536 + 256:
        fcs_flag, fcs = 1, (content_size - 256).to_bytes(2, "little")
    elif content_size < 1 << 32:
        fcs_flag, fcs = 2, content_size.to_bytes(4, "little")
    else:
        fcs_flag, fcs = 3, content_size.to_bytes(8, "little")
    did_flag, did = (0, b"") if not dict_id else (3, dict_id.to_bytes(4, "little"))
    fhd = fcs_flag << 6 | single << 5 | checksum << 2 | did_flag
    return MAGIC + bytes([fhd]) + (b"" if single else bytes([window_desc])) + did + fcs


def raw_literals(lit):
    n = len(lit)
    assert n < 1 << 20
    if n < 32:
        return bytes([n << 3]) + lit
    if n < 4096:
        return bytes([0b0100 | (n & 15) << 4, n >> 4]) + lit
    return bytes([0b1100 | (n & 15) << 4, n >> 4 & 0xFF, n >> 12]) + lit
