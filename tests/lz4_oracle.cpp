// TEST INFRASTRUCTURE — CPU oracle for LZ4-compressed RocksDB data blocks, not product code.
//
// An LZ4 block compressor and a scalar decoder of our own, written from the LZ4 project's published block format
// (lz4_Block_format.md), with no liblz4 behind them; and the two run-level steps RocksDB's BlockBasedTable takes around
// them: the table builder's (compress each finished block, keep it only under the 12.5 % rule) and the block reader's
// (inflate type 4 / 5 blocks before the block iterator, oracle/orc_sst.h, reads them).
//
//   compressed contents := varint32 uncompressed_size | LZ4 block             (format_version >= 2 framing)
//   LZ4 block           := sequence*;  sequence := token | literal length bytes | literals | offset u16 LE | match length bytes
//   trailer             := compression type (0 none, 4 LZ4, 5 LZ4HC) | fixed32 checksum (left zero, as the builder does)
//
// The decoder here is deliberately not tikv_b200/csrc/lz4_block.h: the tests compare the two.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace {

const uint32_t kMinMatch = 4, kLastLiterals = 5, kMatchStartLimit = 12, kMaxOffset = 65535, kHashLog = 14;

uint32_t read32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

void put_len(std::string* o, uint32_t extra) {  // length bytes after a nibble of 15
  while (extra >= 255) { o->push_back((char)255); extra -= 255; }
  o->push_back((char)extra);
}

void put_sequence(std::string* o, const uint8_t* lit, uint32_t n_lit, uint32_t offset, uint32_t match_len /* 0: last sequence */) {
  const uint32_t ml = match_len ? match_len - kMinMatch : 0;
  o->push_back((char)(((n_lit < 15 ? n_lit : 15) << 4) | (ml < 15 ? ml : 15)));
  if (n_lit >= 15) put_len(o, n_lit - 15);
  o->append((const char*)lit, n_lit);
  if (!match_len) return;
  o->push_back((char)(offset & 0xff));
  o->push_back((char)(offset >> 8));
  if (ml >= 15) put_len(o, ml - 15);
}

// Greedy: the last position of every hashed 4-byte sequence; a match starts no later than 12 bytes before the end and
// ends no later than 5 bytes before it (the format's end-of-block rules).
std::string compress(const uint8_t* src, uint32_t n) {
  std::string o;
  std::vector<int64_t> table(1u << kHashLog, -1);
  uint32_t anchor = 0, i = 0;
  if (n >= kMatchStartLimit + 1) {
    const uint32_t start_end = n - kMatchStartLimit, match_end = n - kLastLiterals;
    while (i <= start_end) {
      const uint32_t h = (read32(src + i) * 2654435761u) >> (32 - kHashLog);
      const int64_t c = table[h];
      table[h] = i;
      if (c < 0 || i - c > kMaxOffset || read32(src + c) != read32(src + i)) { ++i; continue; }
      uint32_t ml = kMinMatch;
      while (i + ml < match_end && src[c + ml] == src[i + ml]) ++ml;
      put_sequence(&o, src + anchor, i - anchor, i - (uint32_t)c, ml);
      i += ml;
      anchor = i;
    }
  }
  put_sequence(&o, src + anchor, n - anchor, 0, 0);
  return o;
}

// 0 ok: exactly `size` bytes from exactly src[0, n); 1 corrupt.  Never reads or writes outside those.
int decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t size) {
  size_t ip = 0, op = 0;
  auto more = [&](size_t* len) {  // length bytes: false when they run past the input or the output
    for (;;) {
      if (ip == n) return false;
      const uint8_t b = src[ip++];
      *len += b;
      if (*len > size) return false;
      if (b != 255) return true;
    }
  };
  while (true) {
    if (ip == n) return 1;
    const uint8_t token = src[ip++];
    size_t lit = token >> 4;
    if (lit == 15 && !more(&lit)) return 1;
    if (lit > n - ip || lit > size - op) return 1;
    memcpy(dst + op, src + ip, lit);
    ip += lit; op += lit;
    if (ip == n) return op == size ? 0 : 1;
    if (n - ip < 2) return 1;
    const size_t offset = src[ip] | (size_t)src[ip + 1] << 8;
    ip += 2;
    size_t ml = token & 15;
    if (ml == 15 && !more(&ml)) return 1;
    ml += kMinMatch;
    if (offset == 0 || offset > op || ml > size - op) return 1;
    for (size_t j = 0; j < ml; ++j, ++op) dst[op] = dst[op - offset];  // byte by byte: an overlapping match repeats
  }
}

void put_var32(std::string* o, uint32_t v) {
  while (v >= 0x80) { o->push_back((char)(v | 0x80)); v >>= 7; }
  o->push_back((char)v);
}

// the varint32 size prefix of compressed contents and the bounds a block reader can check before allocating
bool frame(const uint8_t* p, size_t len, uint32_t* size, size_t* at) {
  uint64_t v = 0;
  for (size_t i = 0; i < 5; ++i) {
    if (i == len) return false;
    v |= (uint64_t)(p[i] & 0x7f) << (7 * i);
    if (p[i] & 0x80) continue;
    v &= 0xffffffffu;  // (a varint32 keeps 32 bits)
    if (v < 4 || v > (1u << 30) || v > 255ull * (len - i - 1)) return false;
    *size = (uint32_t)v; *at = i + 1;
    return true;
  }
  return false;
}

struct Run {
  std::string data;
  std::vector<uint64_t> offs{0};
};

}  // namespace

extern "C" {

// raw LZ4 block of src; returns its length (dst has room for n + n / 255 + 16)
size_t lz4o_compress(const uint8_t* src, uint32_t n, uint8_t* dst) {
  const std::string o = compress(src, n);
  memcpy(dst, o.data(), o.size());
  return o.size();
}

int lz4o_decompress(const uint8_t* src, size_t n, uint8_t* dst, size_t size) { return decompress(src, n, dst, size); }

// contents of one block as RocksDB stores them (varint size | LZ4 block): 0 ok, 1 corrupt; *size the declared size
int lz4o_inflate_contents(const uint8_t* p, size_t len, uint8_t* dst, size_t cap, uint32_t* size) {
  size_t at;
  if (!frame(p, len, size, &at) || *size > cap) return 1;
  return decompress(p + at, len - at, dst, *size);
}

// The table builder's step: each block of a plain run (5-byte trailers) compressed with LZ4 and stored with compression
// type `type` when the compressed contents are below raw - raw / 8 (RocksDB's GoodCompressionRatio), else kept plain.
// force != 0 stores every block compressed.
void* lz4o_compress_run(const uint8_t* data, const uint64_t* offs, uint32_t n_blocks, uint8_t type, int force) {
  Run* r = new Run();
  for (uint32_t b = 0; b < n_blocks; ++b) {
    const uint8_t* blk = data + offs[b];
    const uint32_t raw = (uint32_t)(offs[b + 1] - offs[b]) - 5;
    std::string c;
    put_var32(&c, raw);
    c += compress(blk, raw);
    if (force || c.size() < raw - raw / 8) {
      r->data += c;
      r->data.push_back((char)type);
      r->data.append(4, '\0');
    } else {
      r->data.append((const char*)blk, raw + 5);
    }
    r->offs.push_back(r->data.size());
  }
  return r;
}

// The block reader's step: a run with LZ4 / LZ4HC blocks -> the same run with every block plain (type 0).  *status: 0 ok,
// 1 corrupted (a slice too short, a bad LZ4 block, a type byte no RocksDB writer stores: 8..0x3f, 0x41..0x7f, 0xff),
// 2 unsupported (Snappy, zlib, BZip2, Xpress, ZSTD, the older ZSTD 0x40 and the custom-compressor range 0x80..0xfe: a
// valid block the host's reader may inflate).  trailer_len 0: the contents are plain, copied as they are.
void* lz4o_inflate_run(const uint8_t* data, const uint64_t* offs, uint32_t n_blocks, uint32_t trailer_len, int* status) {
  Run* r = new Run();
  *status = 0;
  std::vector<uint8_t> buf;
  for (uint32_t b = 0; b < n_blocks && !*status; ++b) {
    const uint8_t* blk = data + offs[b];
    const uint64_t len = offs[b + 1] - offs[b];
    if (len < trailer_len + 4ull) { *status = 1; break; }
    const uint8_t type = trailer_len ? blk[len - trailer_len] : 0;
    if (type == 0) r->data.append((const char*)blk, len);
    else if (type == 4 || type == 5) {
      uint32_t size = 0;
      size_t at;
      if (!frame(blk, len - trailer_len, &size, &at)) { *status = 1; break; }
      buf.assign(size, 0);
      if (decompress(blk + at, len - trailer_len - at, buf.data(), size)) { *status = 1; break; }
      r->data.append((const char*)buf.data(), size);
      r->data.append(trailer_len, '\0');
    } else *status = ((type >= 1 && type <= 7) || type == 0x40 || (type >= 0x80 && type <= 0xfe)) ? 2 : 1;
    r->offs.push_back(r->data.size());
  }
  return r;
}

const uint8_t* lz4o_run_data(void* h, uint64_t* len, const uint64_t** offs, uint32_t* n_blocks) {
  Run* r = (Run*)h;
  *len = r->data.size(); *offs = r->offs.data(); *n_blocks = (uint32_t)r->offs.size() - 1;
  return (const uint8_t*)r->data.data();
}

void lz4o_run_free(void* h) { delete (Run*)h; }

}  // extern "C"
