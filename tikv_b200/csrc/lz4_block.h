// LZ4 data blocks of a RocksDB BlockBasedTable (compression types 4 kLZ4Compression and 5 kLZ4HCCompression: one stream
// format), as b2_sst_decode inflates them.  One definition for nvcc and g++: the device kernel calls it with
// (lane, 32), one warp per block; the CPU harness (tests/lz4_block_emul.cpp) with (0, 1), under AddressSanitizer.
//
// Framing (RocksDB format_version >= 2):  contents := varint32 uncompressed_size | LZ4 block (raw format, no frame header)
// LZ4 block format (published by the LZ4 project, lz4_Block_format.md):
//   sequence := token | [literal length bytes] | literals | offset (u16 LE) | [match length bytes]
//   token    := literal length (high nibble) | match length - 4 (low nibble); a nibble of 15 continues with bytes that
//               add up until one is not 255.  The last sequence ends after its literals (no offset, no match).
// Every read stays inside the payload and every write inside the declared size; anything else is corruption.  What the
// format's end-of-block rules forbid (a match in the last 12 bytes, fewer than 5 trailing literals) is not rejected:
// such a stream is still decoded within bounds.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define LZ4B_HD __host__ __device__ __forceinline__
#else
#define LZ4B_HD inline
#endif

namespace b2lz4 {

enum : uint32_t { kMinSize = 4, kMaxRatio = 255, kMaxSize = 1u << 30 };  // a block holds num_restarts; LZ4 expands at most 255x

// The framing of one block's contents (len bytes at p): declared size and where the LZ4 payload starts.  False when the
// varint is malformed or the size is impossible: below 4, above 255 x the payload, or above 1 GiB (this bounds what a
// damaged varint can make the caller allocate).
LZ4B_HD bool frame(const uint8_t* p, uint32_t len, uint32_t* size, uint32_t* payload_at) {
  uint32_t v = 0;
  for (uint32_t i = 0; i < 5 && i < len; ++i) {
    const uint32_t b = p[i];
    v |= (b & 0x7fu) << (7 * i);
    if (!(b & 0x80u)) {
      const uint32_t n = len - (i + 1);
      if (v < kMinSize || v > kMaxSize || (uint64_t)v > (uint64_t)kMaxRatio * n) return false;
      *size = v; *payload_at = i + 1;
      return true;
    }
  }
  return false;
}

LZ4B_HD void lane_sync() {
#if defined(__CUDA_ARCH__)
  __syncwarp();
#endif
}

// Inflates the LZ4 block src[0, n) into dst[0, out_len).  Every lane parses every sequence header from the same bytes
// (the control flow is the same on all lanes) and copies bytes lane, lane + n_lanes, ...  True when the stream ends
// exactly at src + n having produced exactly out_len bytes.
LZ4B_HD bool inflate(const uint8_t* src, uint32_t n, uint8_t* dst, uint32_t out_len, uint32_t lane, uint32_t n_lanes) {
  uint32_t ip = 0, op = 0;
  for (;;) {
    if (ip >= n) return false;
    const uint32_t token = src[ip++];
    uint32_t lit = token >> 4;
    if (lit == 15) {
      uint32_t b;
      do {
        if (ip >= n) return false;
        b = src[ip++];
        lit += b;
      } while (b == 255 && lit <= out_len);
    }
    if (lit > n - ip || lit > out_len - op) return false;
    for (uint32_t j = lane; j < lit; j += n_lanes) dst[op + j] = src[ip + j];
    ip += lit; op += lit;
    if (ip == n) return op == out_len;  // the last sequence: literals only
    if (n - ip < 2) return false;
    const uint32_t off = (uint32_t)src[ip] | ((uint32_t)src[ip + 1] << 8);
    ip += 2;
    if (off == 0 || off > op) return false;
    uint32_t ml = token & 15;
    if (ml == 15) {
      uint32_t b;
      do {
        if (ip >= n) return false;
        b = src[ip++];
        ml += b;
      } while (b == 255 && ml <= out_len);
    }
    ml += 4;
    if (ml > out_len - op) return false;
    // A match reads only bytes below op, written by earlier literal and match copies of other lanes: make them visible.
    // Byte j of the match is out[op - off + j % off], so an overlapping match (off < ml, RLE at off 1) repeats the
    // window without waiting on its own bytes.
    lane_sync();
    const uint32_t from = op - off;
    if (off >= ml)
      for (uint32_t j = lane; j < ml; j += n_lanes) dst[op + j] = dst[from + j];
    else
      for (uint32_t j = lane; j < ml; j += n_lanes) dst[op + j] = dst[from + j % off];
    op += ml;
  }
}

}  // namespace b2lz4
