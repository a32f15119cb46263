"""LZ4-compressed RocksDB data blocks (compression types 4 kLZ4Compression / 5 kLZ4HCCompression, format_version >= 2
framing: varint32 uncompressed size | raw LZ4 block).  TEST INFRASTRUCTURE, four readings of the format:
- the oracle (tests/lz4_oracle.cpp): an LZ4 compressor and decoder of its own, the table builder's per-block step
  (RocksDB's 12.5 % rule) and the block reader's (inflate, then oracle/orc_sst.h's iterator through sstfmt);
- a pure-Python LZ4 block decoder (py_decompress);
- liblz4 (LZ4_decompress_safe), when the machine has liblz4.so.1;
- the device's routine (tikv_b200/csrc/lz4_block.h) built for the CPU under AddressSanitizer (emul)."""
import ctypes as C
import os
import struct
import subprocess
import tempfile

import numpy as np

import sstfmt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
ORACLE_SRC = os.path.join(ROOT, "tests", "lz4_oracle.cpp")
EMUL_SRC = os.path.join(ROOT, "tests", "lz4_block_emul.cpp")
DEVICE_HDR = os.path.join(ROOT, "tikv_b200", "csrc", "lz4_block.h")
LZ4, LZ4HC = 4, 5
_lib = None


def _built(out, deps, cmd):
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        os.makedirs(BUILD, exist_ok=True)
        tmp = out + ".%d" % os.getpid()
        subprocess.check_call(cmd + ["-o", tmp])
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        so = _built(os.path.join(BUILD, "liblz4oracle.so"), [ORACLE_SRC], ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", ORACLE_SRC])
        L = C.CDLL(so)
        vp, u8p, u64p = C.c_void_p, C.c_char_p, C.POINTER(C.c_uint64)
        L.lz4o_compress.argtypes, L.lz4o_compress.restype = [u8p, C.c_uint32, vp], C.c_size_t
        L.lz4o_decompress.argtypes, L.lz4o_decompress.restype = [u8p, C.c_size_t, vp, C.c_size_t], C.c_int
        L.lz4o_inflate_contents.argtypes = [u8p, C.c_size_t, vp, C.c_size_t, C.POINTER(C.c_uint32)]
        L.lz4o_compress_run.argtypes, L.lz4o_compress_run.restype = [u8p, vp, C.c_uint32, C.c_uint8, C.c_int], vp
        L.lz4o_inflate_run.argtypes, L.lz4o_inflate_run.restype = [u8p, vp, C.c_uint32, C.c_uint32, C.POINTER(C.c_int)], vp
        L.lz4o_run_data.argtypes, L.lz4o_run_data.restype = [vp, u64p, C.POINTER(u64p), C.POINTER(C.c_uint32)], vp
        L.lz4o_run_free.argtypes = [vp]
        _lib = L
    return _lib


def compress(raw):
    """raw bytes -> an LZ4 block (no framing), by the oracle's compressor"""
    dst = C.create_string_buffer(len(raw) + len(raw) // 255 + 16)
    n = lib().lz4o_compress(bytes(raw), len(raw), dst)
    return dst.raw[:n]


def decompress(payload, size):
    """an LZ4 block that must inflate to exactly `size` bytes -> the bytes, or None when it is corrupt (oracle)"""
    dst = C.create_string_buffer(max(size, 1))
    return dst.raw[:size] if lib().lz4o_decompress(bytes(payload), len(payload), dst, size) == 0 else None


def inflate_contents(contents):
    """compressed block contents (varint32 size | LZ4 block) -> the block, or None (oracle)"""
    cap = 255 * len(contents) + 16
    dst, size = C.create_string_buffer(cap), C.c_uint32()
    return dst.raw[:size.value] if lib().lz4o_inflate_contents(bytes(contents), len(contents), dst, cap, C.byref(size)) == 0 else None


def var32(v):
    out = b""
    while v >= 0x80:
        out += bytes([(v & 0x7F) | 0x80])
        v >>= 7
    return out + bytes([v])


def frame(raw, payload=None):
    """the stored contents of a compressed block: varint32 len(raw) | LZ4 block (the oracle's unless `payload` is given)"""
    return var32(len(raw)) + (compress(raw) if payload is None else payload)


def _run(h):
    L = lib()
    ln, offs, nb = C.c_uint64(), C.POINTER(C.c_uint64)(), C.c_uint32()
    p = L.lz4o_run_data(h, C.byref(ln), C.byref(offs), C.byref(nb))
    out = (C.string_at(p, ln.value) if ln.value else b"", [offs[i] for i in range(nb.value + 1)])
    L.lz4o_run_free(h)
    return out


def compress_run(data, offs, type_byte=LZ4, force=False):
    """a run of plain blocks with 5-byte trailers -> the run RocksDB's table builder stores with LZ4: each block compressed
    when that saves at least 1/8 of it (force: always), else kept plain"""
    o = np.ascontiguousarray(np.asarray(offs, dtype=np.uint64))
    return _run(lib().lz4o_compress_run(bytes(data), o.ctypes.data, len(offs) - 1, type_byte, int(force)))


def build(host_block, compression="lz4", **opts):
    """sstfmt.build with the blocks stored as RocksDB stores them under `compression` (None or "lz4")"""
    data, offs = sstfmt.build(host_block, **opts)
    if compression is None:
        return data, offs
    assert compression == "lz4" and opts.get("trailer_len", 5) == 5, "compressed blocks carry their type in the trailer"
    return compress_run(data, offs)


def inflate_run(data, offs, trailer_len=5):
    """(status, data, offs) of the same run with every block plain, as the block reader sees it: 0 ok, 1 corrupted,
    2 unsupported compression"""
    st = C.c_int()
    o = np.ascontiguousarray(np.asarray(offs, dtype=np.uint64))
    d, no = _run(lib().lz4o_inflate_run(bytes(data) + b"\0" * 8, o.ctypes.data, len(offs) - 1, trailer_len, C.byref(st)))
    return st.value, d, no


def decode(data, offs, trailer_len=5, key_prefix_len=1, key_suffix_len=8):
    """(status, [(key, value)]) by the oracle's block reader: inflate, then the block iterator"""
    st, d, o = inflate_run(data, offs, trailer_len)
    if st:
        return st, []
    return sstfmt.decode(d, o, trailer_len=trailer_len, key_prefix_len=key_prefix_len, key_suffix_len=key_suffix_len)


def block_types(data, offs):
    return [data[b - 5] for b in offs[1:]]


def py_decompress(payload, size):
    """A third reading of the LZ4 block format, in plain Python: the bytes, or None when the stream is corrupt."""
    src, out, ip, n = bytes(payload), bytearray(), 0, len(payload)

    def length(v):
        nonlocal ip
        while True:
            if ip >= n:
                return None
            b = src[ip]
            ip += 1
            v += b
            if b != 255 or v > size:
                return v
    while True:
        if ip >= n:
            return None
        tok = src[ip]
        ip += 1
        lit = tok >> 4
        if lit == 15 and (lit := length(lit)) is None:
            return None
        if ip + lit > n or len(out) + lit > size:
            return None
        out += src[ip:ip + lit]
        ip += lit
        if ip == n:
            return bytes(out) if len(out) == size else None
        if ip + 2 > n:
            return None
        off = src[ip] | src[ip + 1] << 8
        ip += 2
        ml = tok & 15
        if ml == 15 and (ml := length(ml)) is None:
            return None
        ml += 4
        if off == 0 or off > len(out) or len(out) + ml > size:
            return None
        for _ in range(ml):
            out.append(out[-off])


def py_inflate_contents(contents):
    c, v, i = bytes(contents), 0, 0
    while True:
        if i == len(c) or i == 5:
            return None
        v |= (c[i] & 0x7F) << (7 * i)
        i += 1
        if not c[i - 1] & 0x80:
            break
    v &= 0xFFFFFFFF
    if v < 4 or v > 1 << 30 or v > 255 * (len(c) - i):
        return None
    return py_decompress(c[i:], v)


def liblz4():
    """the system's liblz4, or None"""
    try:
        L = C.CDLL("liblz4.so.1")
    except OSError:
        return None
    L.LZ4_decompress_safe.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    L.LZ4_compress_default.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    L.LZ4_compress_HC.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int]
    return L


def lz4_decompress_safe(L, payload, size):
    dst = C.create_string_buffer(max(size, 1))
    r = L.LZ4_decompress_safe(bytes(payload), dst, len(payload), size)
    return dst.raw[:size] if r == size else None


def emul(contents_list):
    """Every compressed block contents through the device's frame() + inflate() built for the CPU (one lane) under
    AddressSanitizer: [bytes, or None when rejected].  A read or write out of bounds fails the harness, and this."""
    exe = _built(os.path.join(BUILD, "lz4_block_emul"), [EMUL_SRC, DEVICE_HDR],
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
            ok, size = raw[p], struct.unpack_from("<I", raw, p + 1)[0]
            p += 5
            out.append(raw[p:p + size] if ok else None)
            p += size if ok else 0
    assert len(out) == len(contents_list)
    return out
