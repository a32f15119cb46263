// ZSTD data blocks of a RocksDB BlockBasedTable (compression types 7 kZSTD and 0x40 kZSTDNotFinalCompression: one stream
// format), as b2_sst_decode inflates them.  One definition for nvcc and g++: the device kernel calls it with (lane, 32),
// one warp per block and one Workspace per warp in shared memory; the CPU harness (tests/zstd_block_emul.cpp) with (0, 1)
// and a heap Workspace, under AddressSanitizer.
//
// Framing (RocksDB format_version >= 2):  contents := varint32 uncompressed_size | one ZSTD frame (RFC 8878 §3.1.1)
// Restated from RFC 8878: frame header, Raw / RLE / Compressed blocks, literals (Raw, RLE, Huffman with 1 or 4 streams,
// Treeless), sequences (Predefined / RLE / FSE_Compressed / Repeat tables for LL, OF and ML, repeat offsets), XXH64
// content checksum.  Not read: dictionaries (Dictionary_ID != 0), skippable and legacy frames, and anything after the
// frame.  Every read stays inside the contents and every write inside the declared size; every bitstream must be
// consumed exactly.
//
// The work of one compressed block, on one warp:
//   1. lane 0 parses the literals and sequences headers and builds the Huffman and FSE tables in the workspace;
//   2. lanes 0-3 decode the four Huffman streams at once (one lane decodes all four when n_lanes == 1);
//   3. lane 0 decodes up to kBatch sequences into the workspace, resolving repeat offsets and checking every bound;
//   4. the warp copies each sequence's literals striped over the lanes, then (after a __syncwarp) its match, byte j of a
//      match of offset d being out[pos - d + j % d]; then the next batch.
// Decoded literals are not kept in a second buffer: they are written at the end of the frame's own output region,
// out[size - n_literals, size).  Writes never overtake an unread literal: after the block the frame has written
// out[0, op_end) with op_end <= size, and at any point the block still has to write the unread literals plus the
// remaining match bytes, so op + unread + remaining_match <= size - ... <= lit_pos, the position of the next unread
// literal (checked per sequence: op + unread + match_length <= size).  A match therefore ends at or below lit_pos, and a
// literal copy moves bytes down (dst <= src), which is safe when done in order: in the overlapping case the lanes load
// a round of bytes before any of them stores.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define ZSTDB_HD __host__ __device__ __forceinline__
#else
#define ZSTDB_HD inline
#endif

namespace b2zstd {

enum : uint32_t { kMinSize = 4, kMaxSize = 1u << 30, kBlockCap = 128u << 10, kMagic = 0xFD2FB528u, kBatch = 32, kHufLogMax = 11 };
enum : int { kOk = 0, kCorrupt = 1, kUnsupported = 2 };

struct Fse { uint16_t next; uint8_t sym, nb; };  // one decoding state: symbol, bits to read, base of the next state
struct Seq { uint32_t ll, ml, off; };

struct Workspace {
  uint16_t huf[1u << kHufLogMax];  // symbol << 8 | code length, indexed by the next huf_log bits
  Fse ll[512], ml[512], of[256];   // sequence tables (accuracy log <= 9 / 9 / 8)
  Fse hw[64];                      // the FSE table of a Huffman tree description (accuracy log <= 6)
  int16_t norm[256];               // normalized counts of the table being built, then its next-state counters
  uint8_t wt[256];                 // Huffman weights
  uint32_t llb[36], mlb[53];       // literal / match length code -> baseline << 5 | extra bits
  Seq seq[kBatch];
  uint32_t huf_log, have_huf, have_seq, ok, hok[4];
  uint32_t lit_type, lit_size, lit_at, lit_n, n_streams, nseq, seq_at;  // lane 0's parse of one block, for the warp
};

ZSTDB_HD void lane_sync() {
#if defined(__CUDA_ARCH__)
  __syncwarp();
#endif
}
ZSTDB_HD uint32_t highbit(uint32_t v) {  // index of the highest set bit, v > 0
#if defined(__CUDA_ARCH__)
  return 31 - __clz(v);
#else
  return 31 - __builtin_clz(v);
#endif
}
ZSTDB_HD uint32_t le32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

struct Frame {
  uint32_t size;      // declared size (varint32)
  uint32_t blocks;    // offset of the first block header in the contents
  uint32_t block_max; // Block_Maximum_Size = min(Window_Size, 128 KiB)
  uint32_t checksum;  // Content_Checksum_Flag
};

// The framing and the frame header of one block's contents (len bytes at p), and a walk over the block headers.
// kUnsupported: no ZSTD frame magic after the varint (a skippable or legacy frame, or not ZSTD at all), or a
// Dictionary_ID.  kCorrupt: a malformed varint, a declared size below 4 or above 1 GiB, a reserved bit, a window
// beyond 2^31, a Frame_Content_Size other than the declared size, a Reserved block or one above Block_Maximum_Size, a
// frame that does not end exactly at the end of the contents (plus 4 checksum bytes), or a declared size the blocks
// cannot produce: Raw and RLE blocks count exactly, a Compressed block at most Block_Maximum_Size.
ZSTDB_HD int frame(const uint8_t* p, uint32_t len, Frame* f) {
  uint32_t v = 0, q = 0;
  for (;;) {
    if (q == 5 || q >= len) return kCorrupt;
    const uint32_t b = p[q];
    v |= (b & 0x7fu) << (7 * q);
    ++q;
    if (!(b & 0x80u)) break;
  }
  if (len - q < 4 || le32(p + q) != kMagic) return kUnsupported;
  if (v < kMinSize || v > kMaxSize) return kCorrupt;
  q += 4;
  if (q >= len) return kCorrupt;
  const uint32_t fhd = p[q++];
  const uint32_t fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, did_flag = fhd & 3;
  const uint32_t did_len = did_flag == 3 ? 4 : did_flag, fcs_len = fcs_flag == 0 ? single : (1u << fcs_flag);
  if (fhd & 8) return kCorrupt;
  if ((uint64_t)q + !single + did_len + fcs_len > len) return kCorrupt;
  uint64_t window = 0;
  if (!single) {
    const uint32_t wd = p[q++];
    if ((wd >> 3) > 21) return kCorrupt;  // Window_Log above 31
    window = 1ull << (10 + (wd >> 3));
    window += (window >> 3) * (wd & 7);
  }
  uint32_t did = 0;
  for (uint32_t i = 0; i < did_len; ++i) did |= (uint32_t)p[q++] << (8 * i);
  if (did) return kUnsupported;
  if (fcs_len) {
    uint64_t fcs = 0;
    for (uint32_t i = 0; i < fcs_len; ++i) fcs |= (uint64_t)p[q++] << (8 * i);
    if (fcs_len == 2) fcs += 256;
    if (fcs != v) return kCorrupt;
    if (single) window = fcs;
  }
  const uint32_t bmax = window < kBlockCap ? (uint32_t)window : kBlockCap;
  f->size = v; f->blocks = q; f->block_max = bmax; f->checksum = (fhd >> 2) & 1;
  uint64_t exact = 0, upto = 0;
  for (;;) {
    if (len - q < 3) return kCorrupt;
    const uint32_t bh = (uint32_t)p[q] | ((uint32_t)p[q + 1] << 8) | ((uint32_t)p[q + 2] << 16);
    const uint32_t type = (bh >> 1) & 3, bsize = bh >> 3;
    q += 3;
    if (type == 3 || bsize > bmax) return kCorrupt;
    const uint32_t in = type == 1 ? 1 : bsize;
    if (len - q < in) return kCorrupt;
    q += in;
    if (type == 2) upto += bmax;
    else exact += bsize;
    if (bh & 1) break;
  }
  if (len - q != 4 * f->checksum) return kCorrupt;
  if (v < exact || v > exact + upto) return kCorrupt;
  return kOk;
}

// ---- bitstreams ----
// A backward bitstream (Huffman streams, FSE streams): bits are read from the end, the highest set bit of the last byte
// marks where they start.  pos = unread bits; a read past the start yields zeros and leaves pos negative (overflow).
struct BitR {
  const uint8_t* p;
  int32_t n, pos, wlo;
  uint64_t win;  // bytes [wlo / 8, wlo / 8 + 8), zeros outside [0, n)
};
ZSTDB_HD int32_t floor8(int32_t x) { return x >= 0 ? x >> 3 : -((-x + 7) >> 3); }
ZSTDB_HD bool br_init(BitR* r, const uint8_t* p, uint32_t n) {
  if (n == 0 || p[n - 1] == 0) return false;
  r->p = p; r->n = (int32_t)n; r->pos = 8 * ((int32_t)n - 1) + (int32_t)highbit(p[n - 1]); r->wlo = 0x7fffffff; r->win = 0;
  return true;
}
ZSTDB_HD void br_fill(BitR* r) {  // the 8 bytes ending with the byte of bit pos - 1
  const int32_t b = floor8(r->pos - 1) - 7;
  uint64_t w = 0;
  for (int32_t i = 0; i < 8; ++i) {
    const int32_t j = b + i;
    if (j >= 0 && j < r->n) w |= (uint64_t)r->p[j] << (8 * i);
  }
  r->win = w; r->wlo = 8 * b;
}
ZSTDB_HD uint32_t br_peek(BitR* r, uint32_t k) {  // the next k <= 32 bits, first bit read as the highest
  if (k == 0) return 0;
  const int32_t lo = r->pos - (int32_t)k;
  if (lo < r->wlo) br_fill(r);
  return (uint32_t)((r->win >> (lo - r->wlo)) & ((1ull << k) - 1));
}
ZSTDB_HD uint32_t br_read(BitR* r, uint32_t k) {
  const uint32_t v = br_peek(r, k);
  r->pos -= (int32_t)k;
  return v;
}

// A forward bitstream (FSE table descriptions): bits from bit 0 of the first byte up, zeros past the end.
ZSTDB_HD uint32_t fw_peek(const uint8_t* p, uint32_t n, uint32_t bit, uint32_t k) {
  uint64_t w = 0;
  const uint32_t b = bit >> 3;
  for (uint32_t i = 0; i < 5; ++i)
    if (b + i < n) w |= (uint64_t)p[b + i] << (8 * i);
  return (uint32_t)((w >> (bit & 7)) & ((1ull << k) - 1));
}

// ---- FSE ----
// An FSE table description (RFC 8878 §4.1.1) at p[0, n): normalized counts of symbols 0..max_sym into norm (0 beyond
// the last one read), accuracy log <= max_log.  Returns the bytes used, 0 when corrupt.
ZSTDB_HD uint32_t read_ncount(const uint8_t* p, uint32_t n, int16_t* norm, uint32_t max_sym, uint32_t max_log, uint32_t* log) {
  uint32_t bit = 0;
  const uint32_t al = fw_peek(p, n, 0, 4) + 5;
  bit = 4;
  if (al > max_log) return 0;
  int32_t remaining = (1 << al) + 1, threshold = 1 << al;
  uint32_t nbits = al + 1, sym = 0;
  bool prev0 = false;
  while (remaining > 1 && sym <= max_sym) {
    if (prev0) {
      uint32_t n0 = sym;
      while (fw_peek(p, n, bit, 2) == 3) { n0 += 3; bit += 2; if (n0 > max_sym) return 0; }
      n0 += fw_peek(p, n, bit, 2);
      bit += 2;
      if (n0 > max_sym) return 0;
      while (sym < n0) norm[sym++] = 0;
    }
    const int32_t mx = 2 * threshold - 1 - remaining;
    const uint32_t v = fw_peek(p, n, bit, nbits);
    int32_t count;
    if ((int32_t)(v & (threshold - 1)) < mx) { count = (int32_t)(v & (threshold - 1)); bit += nbits - 1; }
    else { count = (int32_t)(v & (2 * threshold - 1)); if (count >= threshold) count -= mx; bit += nbits; }
    --count;
    remaining -= count < 0 ? -count : count;
    norm[sym++] = (int16_t)count;
    prev0 = count == 0;
    if (remaining < threshold) {
      if (remaining <= 1) break;
      nbits = highbit((uint32_t)remaining) + 1;
      threshold = 1 << (nbits - 1);
    }
  }
  if (remaining != 1) return 0;
  const uint32_t used = (bit + 7) >> 3;
  if (used > n) return 0;
  for (; sym <= max_sym; ++sym) norm[sym] = 0;
  *log = al;
  return used;
}

// Decoding table of accuracy log `log` from norm[0..max_sym] (RFC 8878 §4.1.1: "less than 1" symbols at the top,
// the others spread with step 5/8 + 3 of the table); norm becomes the next-state counters.
ZSTDB_HD void build_fse(Fse* t, int16_t* norm, uint32_t max_sym, uint32_t log) {
  const uint32_t size = 1u << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
  uint32_t high = size - 1;
  for (uint32_t s = 0; s <= max_sym; ++s)
    if (norm[s] == -1) { t[high--].sym = (uint8_t)s; norm[s] = 0x4001; }  // (marked: not spread, one state)
  uint32_t pos = 0;
  for (uint32_t s = 0; s <= max_sym; ++s) {
    if (norm[s] <= 0 || (norm[s] & 0x4000)) continue;
    for (int32_t i = 0; i < norm[s]; ++i) {
      t[pos].sym = (uint8_t)s;
      do pos = (pos + step) & mask; while (pos > high);
    }
  }
  for (uint32_t s = 0; s <= max_sym; ++s) norm[s] &= 0x3fff;
  for (uint32_t u = 0; u < size; ++u) {
    const uint32_t s = t[u].sym, nx = (uint32_t)norm[s]++;
    const uint32_t nb = log - highbit(nx);
    t[u].nb = (uint8_t)nb;
    t[u].next = (uint16_t)((nx << nb) - size);
  }
}

ZSTDB_HD void rle_fse(Fse* t, uint32_t sym) { t[0].sym = (uint8_t)sym; t[0].nb = 0; t[0].next = 0; }

// the predefined distributions (RFC 8878 §3.1.1.3.2.2), 0xff = -1
ZSTDB_HD void predefined(int16_t* norm, uint32_t which) {
  const char* d = which == 0 ? "\4\3\2\2\2\2\2\2\2\2\2\2\2\1\1\1\2\2\2\2\2\2\2\2\2\3\2\1\1\1\1\1\377\377\377\377"
                  : which == 1 ? "\1\1\1\1\1\1\2\2\2\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\377\377\377\377\377"
                               : "\1\4\3\2\2\2\2\2\2\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\1\377\377\377\377\377\377\377";
  const uint32_t n = which == 0 ? 36 : (which == 1 ? 29 : 53);
  for (uint32_t s = 0; s < n; ++s) norm[s] = (int16_t)(int8_t)d[s];
}

// ---- Huffman ----
// A Huffman tree description (RFC 8878 §4.2.1) at p[0, n) -> ws->huf / huf_log.  Returns the bytes used, 0 when corrupt.
ZSTDB_HD uint32_t read_huf(const uint8_t* p, uint32_t n, Workspace* ws) {
  if (n < 1) return 0;
  const uint32_t hdr = p[0];
  uint32_t nw = 0, used;
  if (hdr >= 128) {
    nw = hdr - 127;
    const uint32_t bytes = (nw + 1) / 2;
    if (1 + bytes > n) return 0;
    for (uint32_t i = 0; i < nw; ++i) ws->wt[i] = (uint8_t)(i & 1 ? p[1 + i / 2] & 15 : p[1 + i / 2] >> 4);
    used = 1 + bytes;
  } else {
    const uint32_t cs = hdr;
    if (1 + cs > n) return 0;
    uint32_t al;
    const uint32_t h = read_ncount(p + 1, cs, ws->norm, 255, 6, &al);
    if (h == 0 || h >= cs) return 0;
    uint32_t last = 255;
    while (last > 0 && ws->norm[last] == 0) --last;
    build_fse(ws->hw, ws->norm, last, al);
    BitR r;
    if (!br_init(&r, p + 1 + h, cs - h)) return 0;
    uint32_t s1 = br_read(&r, al), s2 = br_read(&r, al);
    for (;;) {  // two interleaved states until the stream overflows, then the other state's symbol ends it
      if (nw > 253) return 0;
      ws->wt[nw++] = ws->hw[s1].sym;
      s1 = ws->hw[s1].next + br_read(&r, ws->hw[s1].nb);
      if (r.pos < 0) { ws->wt[nw++] = ws->hw[s2].sym; break; }
      if (nw > 253) return 0;
      ws->wt[nw++] = ws->hw[s2].sym;
      s2 = ws->hw[s2].next + br_read(&r, ws->hw[s2].nb);
      if (r.pos < 0) { ws->wt[nw++] = ws->hw[s1].sym; break; }
    }
    used = 1 + cs;
  }
  uint32_t total = 0, rank1 = 0;
  for (uint32_t i = 0; i < nw; ++i) {
    const uint32_t w = ws->wt[i];
    if (w > kHufLogMax) return 0;
    total += (1u << w) >> 1;
    rank1 += w == 1;
  }
  if (total == 0) return 0;
  const uint32_t log = highbit(total) + 1;
  if (log > kHufLogMax) return 0;
  const uint32_t rest = (1u << log) - total, lw = highbit(rest) + 1;
  if ((1u << highbit(rest)) != rest) return 0;
  ws->wt[nw] = (uint8_t)lw;
  rank1 += lw == 1;
  if (rank1 < 2 || (rank1 & 1)) return 0;
  uint32_t pos = 0;
  for (uint32_t w = 1; w <= log; ++w)
    for (uint32_t s = 0; s <= nw; ++s)
      if (ws->wt[s] == w) {
        const uint16_t e = (uint16_t)((s << 8) | (log + 1 - w));
        for (uint32_t i = 0; i < (1u << (w - 1)); ++i) ws->huf[pos++] = e;
      }
  ws->huf_log = log;
  return used;
}

// one Huffman stream: exactly cnt symbols, and exactly all of its bits
ZSTDB_HD bool huf_stream(const uint8_t* p, uint32_t n, uint8_t* dst, uint32_t cnt, const Workspace* ws) {
  BitR r;
  if (!br_init(&r, p, n)) return false;
  const uint32_t log = ws->huf_log;
  for (uint32_t k = 0; k < cnt; ++k) {
    const uint32_t e = ws->huf[br_peek(&r, log)];
    dst[k] = (uint8_t)(e >> 8);
    r.pos -= (int32_t)(e & 0xff);
  }
  return r.pos == 0;
}

// ---- XXH64 (seed 0) ----
ZSTDB_HD uint64_t rotl64(uint64_t x, uint32_t r) { return (x << r) | (x >> (64 - r)); }
ZSTDB_HD uint64_t le64(const uint8_t* p) { return (uint64_t)le32(p) | ((uint64_t)le32(p + 4) << 32); }
ZSTDB_HD uint64_t xxh64(const uint8_t* p, uint64_t len) {
  const uint64_t P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
  uint64_t h, i = 0;
  if (len >= 32) {
    uint64_t v[4] = {P1 + P2, P2, 0, 0 - P1};
    for (; i + 32 <= len; i += 32)
      for (int k = 0; k < 4; ++k) v[k] = rotl64(v[k] + le64(p + i + 8 * k) * P2, 31) * P1;
    h = rotl64(v[0], 1) + rotl64(v[1], 7) + rotl64(v[2], 12) + rotl64(v[3], 18);
    for (int k = 0; k < 4; ++k) { h ^= rotl64(v[k] * P2, 31) * P1; h = h * P1 + P4; }
  } else h = P5;
  h += len;
  for (; i + 8 <= len; i += 8) { h ^= rotl64(le64(p + i) * P2, 31) * P1; h = rotl64(h, 27) * P1 + P4; }
  if (i + 4 <= len) { h ^= (uint64_t)le32(p + i) * P1; h = rotl64(h, 23) * P2 + P3; i += 4; }
  for (; i < len; ++i) { h ^= p[i] * P5; h = rotl64(h, 11) * P1; }
  h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
  return h;
}

// ---- blocks ----
// Literal bytes src[0, n) to dst: in place when src lies n or more bytes above dst (or outside the output), else in
// rounds of n_lanes bytes, every lane loading its byte of the round before any lane stores (dst < src: in order).
ZSTDB_HD void copy_down(uint8_t* dst, const uint8_t* src, uint32_t n, bool apart, uint32_t lane, uint32_t n_lanes) {
  if (dst == src) return;
  if (apart) {
    for (uint32_t j = lane; j < n; j += n_lanes) dst[j] = src[j];
    return;
  }
  for (uint32_t b = 0; b < n; b += n_lanes) {
    const uint32_t j = b + lane;
    const uint8_t c = j < n ? src[j] : 0;
    lane_sync();
    if (j < n) dst[j] = c;
    lane_sync();
  }
}

ZSTDB_HD void init_codes(Workspace* ws) {
  for (uint32_t c = 0; c < 36; ++c) {  // literal lengths: 0..15 as is, then (baseline, extra bits) pairs
    uint32_t base = c, bits = 0;
    if (c >= 16) {
      bits = c < 25 ? (uint32_t)((0x433221111ull >> (4 * (c - 16))) & 15) : c - 19;
      base = c < 25 ? 16 : 1u << (c - 19);
      for (uint32_t k = 16; k < c && c < 25; ++k) base += 1u << ((0x433221111ull >> (4 * (k - 16))) & 15);
    }
    ws->llb[c] = base << 5 | bits;
  }
  for (uint32_t c = 0; c < 53; ++c) {  // match lengths: 3..34, then pairs
    uint32_t base = c + 3, bits = 0;
    if (c >= 32) {
      const uint64_t nib = 0x54433221111ull;
      bits = c < 43 ? (uint32_t)((nib >> (4 * (c - 32))) & 15) : c - 36;
      base = c < 43 ? 35 : (1u << (c - 36)) + 3;
      for (uint32_t k = 32; k < c && c < 43; ++k) base += 1u << ((nib >> (4 * (k - 32))) & 15);
    }
    ws->mlb[c] = base << 5 | bits;
  }
}

// One sequence table (mode 0 Predefined, 1 RLE, 2 FSE_Compressed, 3 Repeat) at p[0, n) -> the bytes used, or -1.
ZSTDB_HD int32_t seq_table(const uint8_t* p, uint32_t n, uint32_t mode, uint32_t which, Fse* t, uint32_t* log, Workspace* ws) {
  const uint32_t max_sym = which == 0 ? 35 : (which == 1 ? 31 : 52), max_log = which == 1 ? 8 : 9;
  if (mode == 0) {
    predefined(ws->norm, which);
    *log = which == 1 ? 5 : 6;
    build_fse(t, ws->norm, which == 0 ? 35 : (which == 1 ? 28 : 52), *log);
    return 0;
  }
  if (mode == 1) {
    if (n < 1 || p[0] > max_sym) return -1;
    rle_fse(t, p[0]);
    *log = 0;
    return 1;
  }
  if (mode == 2) {
    uint32_t al;
    const uint32_t h = read_ncount(p, n, ws->norm, max_sym, max_log, &al);
    if (h == 0) return -1;
    uint32_t last = max_sym;
    while (last > 0 && ws->norm[last] == 0) --last;
    build_fse(t, ws->norm, last, al);
    *log = al;
    return (int32_t)h;
  }
  return ws->have_seq ? 0 : -1;
}

// Lane 0's state across the blocks of a frame: the repeat offsets and the accuracy logs of the current tables.
struct Lane0 { uint32_t rep0, rep1, rep2, ll_log, of_log, ml_log; };

// Lane 0: literals and sequences headers of the compressed block src[0, n), tables built; results in ws->lit_* / nseq /
// seq_at.  False when corrupt.
ZSTDB_HD bool parse_block(const uint8_t* src, uint32_t n, uint32_t op, uint32_t size, uint32_t bmax, Workspace* ws, Lane0* z) {
  if (n < 1) return false;
  const uint32_t b0 = src[0], lt = b0 & 3, sf = (b0 >> 2) & 3;
  uint32_t lh, lsize, csize = 0, ns = 1;
  if (lt <= 1) {
    lh = sf == 1 ? 2 : (sf == 3 ? 3 : 1);
    if (n < lh) return false;
    lsize = lh == 1 ? b0 >> 3 : (lh == 2 ? (b0 >> 4) | ((uint32_t)src[1] << 4) : (b0 >> 4) | ((uint32_t)src[1] << 4) | ((uint32_t)src[2] << 12));
  } else {
    lh = sf <= 1 ? 3 : sf + 2;
    ns = sf == 0 ? 1 : 4;
    if (n < lh) return false;
    uint64_t v = 0;
    for (uint32_t i = 0; i < lh; ++i) v |= (uint64_t)src[i] << (8 * i);
    const uint32_t w = lh == 3 ? 10 : (lh == 4 ? 14 : 18);
    lsize = (uint32_t)((v >> 4) & ((1u << w) - 1));
    csize = (uint32_t)((v >> (4 + w)) & ((1u << w) - 1));
    if (ns == 4 && lsize < 6) return false;
  }
  if (lsize > bmax || lsize > size - op) return false;
  uint32_t pos = lh, lit_at = pos, lit_n = lsize;
  if (lt == 0) { if (n - pos < lsize) return false; pos += lsize; }
  else if (lt == 1) { if (n - pos < 1) return false; pos += 1; }
  else {
    if (n - pos < csize) return false;
    uint32_t t = 0;
    if (lt == 2) {
      if (!(t = read_huf(src + pos, csize, ws))) return false;
      ws->have_huf = 1;
    } else if (!ws->have_huf) return false;
    lit_at = pos + t; lit_n = csize - t;
    pos += csize;
    if (ns == 4 && lit_n < 10) return false;
  }
  ws->lit_type = lt; ws->lit_size = lsize; ws->lit_at = lit_at; ws->lit_n = lit_n; ws->n_streams = ns;
  // sequences section header
  if (pos >= n) return false;
  uint32_t nseq = src[pos++];
  if (nseq >= 128) {
    if (nseq == 255) { if (n - pos < 2) return false; nseq = (uint32_t)src[pos] + ((uint32_t)src[pos + 1] << 8) + 0x7f00; pos += 2; }
    else { if (n - pos < 1) return false; nseq = ((nseq - 128) << 8) + src[pos]; pos += 1; }
  }
  ws->nseq = nseq;
  if (nseq == 0) { ws->seq_at = pos; return pos == n; }
  if (pos >= n) return false;
  const uint32_t modes = src[pos++];
  if (modes & 3) return false;
  int32_t u;
  if ((u = seq_table(src + pos, n - pos, modes >> 6, 0, ws->ll, &z->ll_log, ws)) < 0) return false;
  pos += (uint32_t)u;
  if ((u = seq_table(src + pos, n - pos, (modes >> 4) & 3, 1, ws->of, &z->of_log, ws)) < 0) return false;
  pos += (uint32_t)u;
  if ((u = seq_table(src + pos, n - pos, (modes >> 2) & 3, 2, ws->ml, &z->ml_log, ws)) < 0) return false;
  pos += (uint32_t)u;
  ws->have_seq = 1;
  ws->seq_at = pos;
  return pos < n;
}

// One compressed block src[0, n) of the frame whose output is out[0, size), written from op on.
ZSTDB_HD bool compressed_block(const uint8_t* src, uint32_t n, uint8_t* out, uint32_t* opp, uint32_t size, uint32_t bmax, Workspace* ws, Lane0* z,
                               uint32_t lane, uint32_t n_lanes) {
  const uint32_t op0 = *opp;
  if (lane == 0) ws->ok = parse_block(src, n, op0, size, bmax, ws, z);
  lane_sync();
  if (!ws->ok) return false;
  const uint32_t lt = ws->lit_type, lsize = ws->lit_size, nseq = ws->nseq;
  const uint8_t* lit;
  uint8_t* const lit_out = out + (size - lsize);  // (the end of the frame's output region)
  if (lt == 0) lit = src + ws->lit_at;
  else {
    lit = lit_out;
    if (lt == 1) {
      const uint8_t c = src[ws->lit_at];
      for (uint32_t j = lane; j < lsize; j += n_lanes) lit_out[j] = c;
    } else {
      const uint8_t* hs = src + ws->lit_at;
      const uint32_t hn = ws->lit_n;
      if (ws->n_streams == 1) {
        if (lane == 0) ws->hok[0] = huf_stream(hs, hn, lit_out, lsize, ws);
        if (lane == 0) ws->hok[1] = ws->hok[2] = ws->hok[3] = 1;
      } else {
        const uint32_t l1 = hs[0] | (hs[1] << 8), l2 = hs[2] | (hs[3] << 8), l3 = hs[4] | (hs[5] << 8);
        const uint32_t seg = (lsize + 3) / 4;
        const bool fits = 6ull + l1 + l2 + l3 <= hn;
        for (uint32_t i = lane; i < 4; i += n_lanes) {
          if (!fits) { ws->hok[i] = 0; continue; }
          const uint32_t at = 6 + (i > 0 ? l1 : 0) + (i > 1 ? l2 : 0) + (i > 2 ? l3 : 0);
          const uint32_t len = i == 0 ? l1 : (i == 1 ? l2 : (i == 2 ? l3 : hn - 6 - l1 - l2 - l3));
          ws->hok[i] = huf_stream(hs + at, len, lit_out + i * seg, i < 3 ? seg : lsize - 3 * seg, ws);
        }
      }
    }
  }
  lane_sync();
  if (lt >= 2 && !(ws->hok[0] & ws->hok[1] & ws->hok[2] & ws->hok[3])) return false;
  const bool lit_in_out = lt != 0;
  uint32_t op = op0, lit_rd = 0;
  // lane 0's sequence decoder
  BitR r;
  uint32_t sll = 0, sof = 0, sml = 0, sim_op = op0, sim_lit = 0;
  if (lane == 0 && nseq) {
    ws->ok = br_init(&r, src + ws->seq_at, n - ws->seq_at);
    if (ws->ok) { sll = br_read(&r, z->ll_log); sof = br_read(&r, z->of_log); sml = br_read(&r, z->ml_log); }
  }
  lane_sync();
  if (nseq && !ws->ok) return false;
  lane_sync();  // (every lane has read ws->ok before lane 0 writes it again)
  for (uint32_t done = 0; done < nseq; done += kBatch) {
    const uint32_t cnt = nseq - done < kBatch ? nseq - done : kBatch;
    if (lane == 0) {
      bool ok = true;
      for (uint32_t i = 0; i < cnt && ok; ++i) {
        const uint32_t ofc = ws->of[sof].sym, mlc = ws->ml[sml].sym, llc = ws->ll[sll].sym;
        const uint32_t ofv = (1u << ofc) + br_read(&r, ofc);
        const uint32_t ml = (ws->mlb[mlc] >> 5) + br_read(&r, ws->mlb[mlc] & 31);
        const uint32_t ll = (ws->llb[llc] >> 5) + br_read(&r, ws->llb[llc] & 31);
        uint32_t off;
        if (ofv > 3) { off = ofv - 3; z->rep2 = z->rep1; z->rep1 = z->rep0; z->rep0 = off; }
        else {
          const uint32_t k = ofv - 1 + (ll == 0);  // 0 rep0, 1 rep1, 2 rep2, 3 rep0 - 1
          if (k == 0) off = z->rep0;
          else {
            off = k == 3 ? z->rep0 - 1 : (k == 1 ? z->rep1 : z->rep2);
            if (k != 1) z->rep2 = z->rep1;
            z->rep1 = z->rep0; z->rep0 = off;
          }
        }
        const uint32_t left = lsize - sim_lit;  // unread literals
        if (ll > left || off == 0 || off > sim_op + ll || (uint64_t)sim_op + left + ml > size || (uint64_t)(sim_op - op0) + left + ml > bmax) ok = false;
        ws->seq[i].ll = ll; ws->seq[i].ml = ml; ws->seq[i].off = off;
        sim_op += ll + ml; sim_lit += ll;
        if (done + i + 1 < nseq) {
          sll = ws->ll[sll].next + br_read(&r, ws->ll[sll].nb);
          sml = ws->ml[sml].next + br_read(&r, ws->ml[sml].nb);
          sof = ws->of[sof].next + br_read(&r, ws->of[sof].nb);
        }
        if (r.pos < 0) ok = false;
      }
      if (ok && done + cnt == nseq && r.pos != 0) ok = false;
      ws->ok = ok;
    }
    lane_sync();
    if (!ws->ok) return false;
    for (uint32_t i = 0; i < cnt; ++i) {
      const Seq s = ws->seq[i];
      const uint8_t* from = lit + lit_rd;
      copy_down(out + op, from, s.ll, !lit_in_out || (uint32_t)(from - (out + op)) >= s.ll, lane, n_lanes);
      op += s.ll; lit_rd += s.ll;
      lane_sync();
      const uint32_t d = s.off, ml = s.ml, at = op - d;
      if (d >= ml)
        for (uint32_t j = lane; j < ml; j += n_lanes) out[op + j] = out[at + j];
      else
        for (uint32_t j = lane; j < ml; j += n_lanes) out[op + j] = out[at + j % d];
      op += ml;
    }
    lane_sync();
  }
  // the last literals
  const uint32_t rest = lsize - lit_rd;
  const uint8_t* from = lit + lit_rd;
  copy_down(out + op, from, rest, !lit_in_out || (uint32_t)(from - (out + op)) >= rest, lane, n_lanes);
  op += rest;
  lane_sync();
  *opp = op;
  return true;
}

// Inflates the frame of the contents p[0, len) that frame() accepted into out[0, f.size).  True when it produces
// exactly f.size bytes (and the checksum matches when the frame carries one).
ZSTDB_HD bool inflate(const uint8_t* p, uint32_t len, const Frame& f, uint8_t* out, Workspace* ws, uint32_t lane, uint32_t n_lanes) {
  Lane0 z;
  z.rep0 = 1; z.rep1 = 4; z.rep2 = 8; z.ll_log = z.of_log = z.ml_log = 0;
  if (lane == 0) { init_codes(ws); ws->have_huf = ws->have_seq = 0; }
  lane_sync();
  uint32_t q = f.blocks, op = 0;
  const uint32_t size = f.size;
  for (;;) {
    const uint32_t bh = (uint32_t)p[q] | ((uint32_t)p[q + 1] << 8) | ((uint32_t)p[q + 2] << 16);
    const uint32_t type = (bh >> 1) & 3, bsize = bh >> 3;
    q += 3;
    if (type == 0) {
      if (bsize > size - op) return false;
      for (uint32_t j = lane; j < bsize; j += n_lanes) out[op + j] = p[q + j];
      op += bsize; q += bsize;
    } else if (type == 1) {
      if (bsize > size - op) return false;
      const uint8_t c = p[q];
      for (uint32_t j = lane; j < bsize; j += n_lanes) out[op + j] = c;
      op += bsize; q += 1;
    } else {
      if (!compressed_block(p + q, bsize, out, &op, size, f.block_max, ws, &z, lane, n_lanes)) return false;
      q += bsize;
    }
    if (bh & 1) break;
  }
  if (op != size) return false;
  if (f.checksum) {
    lane_sync();
    if (lane == 0) ws->ok = (uint32_t)xxh64(out, size) == le32(p + q);
    lane_sync();
    return ws->ok;
  }
  return true;
}

}  // namespace b2zstd
