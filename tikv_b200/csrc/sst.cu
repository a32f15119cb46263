// RocksDB BlockBasedTable data blocks -> the flat CF block layout of the scan kernels (SURVEY.md §8(f)4, b2_sst_decode),
// and the inverse as tooling (b2_sst_encode).  RocksDB is an external dependency of the reference (librocksdb behind
// components/engine_rocks); the block layout restated here is the published one:
//
//   data block := entry* restart[u32 LE x num_restarts] num_restarts[u32 LE]      (+ 5-byte trailer when stored)
//   entry      := varint32 shared | varint32 non_shared | varint32 value_len | key bytes [shared, shared + non_shared) | value
//   restart[j] := offset of an entry with shared == 0; one every block_restart_interval entries (16 by default)
//
// A restart interval is the unit of parallelism: one thread walks one interval (<= 16 entries in practice).  The passes,
// each bounded by HBM traffic that is a small multiple of the block bytes:
//   sst_blocks    one thread per data block: the trailer's compression type, the slice; a plain block (type 0) gets its
//                 contents view (the slice) and its footer read and validated   -> restart points per block; an LZ4 /
//                 LZ4HC block (type 4 / 5) its framing checked, a ZSTD block (type 7 / 0x40) its frame header and block
//                 headers walked                                                -> inflated size per block
//   sst_inflate   only when the run holds LZ4 blocks: one warp per LZ4 block (lz4_block.h) inflates it into the
//                 handle's inflate buffer at the exclusive sum of the inflated sizes; that is its contents view.
//   sst_zstd      only when the run holds ZSTD blocks, beside sst_inflate: one warp per ZSTD block (zstd_block.h, its
//                 workspace in shared memory) inflates it into the same buffer.  sst_blocks then reads the footers of the
//                 inflated blocks (the one extra host round trip, for compressed runs only)
//   sst_count     one thread per restart interval: entries, key bytes, value bytes   -> prefix sums give every
//                 interval its place in the flat block
//   sst_expand    one warp per restart interval: the current key lives in the warp's registers (byte j in lane j % 32),
//                 every entry overwrites the bytes past `shared` and streams the key, minus the data prefix and the
//                 internal-key footer (whose value type must be kTypeValue), and the value out as consecutive bytes
// sst_count and sst_expand read each block through its contents view, so plain and LZ4 blocks mix in one run (RocksDB
// stores a block plain when LZ4 saves less than 1/8 of it).  The expansion runs an order of magnitude above the PCIe
// link the compressed bytes arrive over, which is the point: fewer bytes cross the link (53 instead of 69 per C3 entry
// with prefix compression alone; LZ4 blocks of the same table hold about 0.31 of those bytes).
#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b2_copr.h"
#include "lz4_block.h"
#include "sst_merge.h"
#include "zstd_block.h"

namespace b2 {
void set_last_error(const std::string& m);  // engine.cu (thread-local message behind b2_last_error_message)
}

namespace {

enum { SST_OK = 0, SST_CORRUPT = 1, SST_UNSUPPORTED = 2 };

struct SstView {
  const uint8_t* data;
  const unsigned long long* boffs;  // n_blocks + 1
  const uint8_t* inflated;          // the inflated LZ4 blocks
  const unsigned long long* voff;   // n_blocks: contents view of each block: offset into data, or into inflated | kInflated
  const unsigned int* vlen;         // n_blocks: contents length (0: no view, the block failed its checks)
  unsigned int n_blocks, trailer, pl, sl;
};
constexpr unsigned long long kInflated = 1ull << 63;

// (an offset, not a pointer, in the view array: with a pointer loaded from memory ptxas spills in sst_expand_kernel)
__device__ __forceinline__ const uint8_t* view_of(const SstView& S, unsigned int b) {
  const unsigned long long v = S.voff[b];
  return (v & kInflated ? S.inflated : S.data) + (v & ~kInflated);
}

__device__ __forceinline__ unsigned int ld_le32(const uint8_t* p) { return (unsigned int)p[0] | ((unsigned int)p[1] << 8) | ((unsigned int)p[2] << 16) | ((unsigned int)p[3] << 24); }

// varint32 at p (limit lim): returns bytes used, 0 when malformed / truncated
__device__ __forceinline__ unsigned int get_var32(const uint8_t* p, const uint8_t* lim, unsigned int* v) {
  unsigned int r = 0;
#pragma unroll 1
  for (unsigned int i = 0; i < 5 && p + i < lim; ++i) {
    const unsigned int b = p[i];
    r |= (b & 0x7f) << (7 * i);
    if (!(b & 0x80)) { *v = r; return i + 1; }
  }
  return 0;
}

__device__ __forceinline__ void raise(unsigned int* err, unsigned int code) { atomicMax(err, code); }

// restart count of a block from its contents view (0 and an error when the footer is invalid)
__device__ __forceinline__ unsigned int block_restarts(const uint8_t* base, unsigned int len, unsigned int* err) {
  if (len < 4) { raise(err, SST_CORRUPT); return 0; }
  const unsigned int foot = ld_le32(base + len - 4);
  if (foot >> 31) { raise(err, SST_UNSUPPORTED); return 0; }  // data block hash index packed into the footer
  if (foot == 0 || (unsigned long long)foot * 4 + 4 > len) { raise(err, SST_CORRUPT); return 0; }
  return foot;
}

struct ViewOut { unsigned long long* off; unsigned int* len; };  // the writable side of SstView::voff / vlen

// RocksDB CompressionType values a valid block may carry that the device does not inflate: the built-in Snappy 1, zlib 2,
// BZip2 3 and Xpress 6, and the custom-compressor range 0x80..0xfe (LZ4 4 / 5 and ZSTD 7 / 0x40 are tested first).  The host's block reader may inflate them: B2_ERR_UNSUPPORTED.  No RocksDB writer stores any other value
// (8..0x3f, 0x41..0x7f, 0xff kDisableCompressionOption): a block carrying one is damaged.
__device__ __forceinline__ bool host_compression(unsigned int t) { return (t >= 1 && t <= 7) || t == 0x40 || (t >= 0x80 && t <= 0xfe); }

// Before inflation (inflated == 0): classify every block.  Plain blocks get their contents view and restart count, LZ4
// and ZSTD blocks their declared size in isz (0 for every other block) and a restart count of 0; their numbers and the
// sum of their sizes come back with the first round trip, so the inflate buffer is sized without another.  After inflation:
// the restart count of every block from its view.
__global__ void sst_blocks_kernel(SstView S, ViewOut V, unsigned int* nres /* n_blocks + 1, last = 0 */, unsigned long long* isz /* n_blocks + 1 */,
                                  unsigned int* n_lz4, unsigned long long* lz4_bytes, unsigned int* n_zstd, unsigned int inflated, unsigned int* err) {
  const unsigned int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > S.n_blocks) return;
  if (b == S.n_blocks) { nres[b] = 0; if (!inflated) isz[b] = 0; return; }
  if (inflated) { nres[b] = S.vlen[b] ? block_restarts(view_of(S, b), S.vlen[b], err) : 0; return; }
  const unsigned long long lo = S.boffs[b], hi = S.boffs[b + 1];
  unsigned int nr = 0;
  unsigned long long sz = 0;
  unsigned int len = 0, vlen = 0;
  if (hi < lo || hi - lo < (unsigned long long)S.trailer + 4 || hi - lo > 0xffffff00ull) raise(err, SST_CORRUPT);
  else {
    const uint8_t* base = S.data + lo;
    len = (unsigned int)(hi - lo) - S.trailer;
    const unsigned int type = S.trailer ? base[len] : 0;  // the trailer's first byte: RocksDB's compression type
    if (type == 0) { vlen = len; nr = block_restarts(base, len, err); }
    else if (type == 4 || type == 5) {
      unsigned int n, at;
      if (b2lz4::frame(base, len, &n, &at)) { sz = n; atomicAdd(n_lz4, 1u); atomicAdd(lz4_bytes, sz); }
      else raise(err, SST_CORRUPT);
    } else if (type == 7 || type == 0x40) {
      b2zstd::Frame f;
      const int v = b2zstd::frame(base, len, &f);
      if (v == b2zstd::kOk) { sz = f.size; atomicAdd(n_zstd, 1u); atomicAdd(lz4_bytes, sz); }
      else raise(err, v == b2zstd::kUnsupported ? SST_UNSUPPORTED : SST_CORRUPT);
    } else raise(err, host_compression(type) ? SST_UNSUPPORTED : SST_CORRUPT);
  }
  V.off[b] = lo; V.len[b] = vlen;
  nres[b] = nr; isz[b] = sz;
}

// One warp per block: LZ4 blocks (isz[b + 1] > isz[b]) inflate into inflated + isz[b] and get that as their view.
__global__ void __launch_bounds__(256) sst_inflate_kernel(SstView S, ViewOut V, const unsigned long long* isz /* exclusive sums */, unsigned int* err) {
  const unsigned int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (b >= S.n_blocks) return;
  const unsigned long long at = isz[b], size = isz[b + 1] - at;
  if (size == 0) return;
  const uint8_t* base = S.data + S.boffs[b];
  const unsigned int len = (unsigned int)(S.boffs[b + 1] - S.boffs[b]) - S.trailer;
  if (base[len] != 4 && base[len] != 5) return;  // a ZSTD block: sst_zstd_kernel's
  unsigned int n, p;
  b2lz4::frame(base, len, &n, &p);  // (validated by sst_blocks_kernel: n == size)
  uint8_t* out = (uint8_t*)S.inflated + at;
  const bool ok = b2lz4::inflate(base + p, len - p, out, n, lane, 32);
  if (lane == 0) {
    if (ok) { V.off[b] = kInflated | at; V.len[b] = n; }
    else raise(err, SST_CORRUPT);  // (no view: the footer pass must not read a half-written block and report its garbage)
  }
}

// One warp per block: ZSTD blocks inflate into inflated + isz[b] and get that as their view.  Four warps per CTA, each
// with its workspace (tables and a sequence batch, sizeof(b2zstd::Workspace)) in shared memory.
constexpr unsigned int kZstdWarps = 4;
__global__ void __launch_bounds__(32 * kZstdWarps) sst_zstd_kernel(SstView S, ViewOut V, const unsigned long long* isz, unsigned int* err) {
  __shared__ b2zstd::Workspace ws[kZstdWarps];
  const unsigned int w = threadIdx.x >> 5, b = blockIdx.x * kZstdWarps + w, lane = threadIdx.x & 31;
  if (b >= S.n_blocks) return;
  const unsigned long long at = isz[b];
  if (isz[b + 1] == at) return;
  const uint8_t* base = S.data + S.boffs[b];
  const unsigned int len = (unsigned int)(S.boffs[b + 1] - S.boffs[b]) - S.trailer;
  if (base[len] != 7 && base[len] != 0x40) return;  // an LZ4 block: sst_inflate_kernel's
  b2zstd::Frame f;
  b2zstd::frame(base, len, &f);  // (validated by sst_blocks_kernel: f.size == isz[b + 1] - at)
  uint8_t* out = (uint8_t*)S.inflated + at;
  const bool ok = b2zstd::inflate(base, len, f, out, &ws[w], lane, 32);
  if (lane == 0) {
    if (ok) { V.off[b] = kInflated | at; V.len[b] = f.size; }
    else raise(err, SST_CORRUPT);  // (no view, as in sst_inflate_kernel)
  }
}

struct Interval { const uint8_t *p, *end; };

// the entry bytes of restart interval t
__device__ __forceinline__ bool interval_of(const SstView& S, const unsigned int* ibase, unsigned int t, Interval* iv, unsigned int* err) {
  unsigned int lo = 0, hi = S.n_blocks;  // last block with ibase[b] <= t
  while (hi - lo > 1) { const unsigned int mid = (lo + hi) >> 1; if (ibase[mid] <= t) lo = mid; else hi = mid; }
  const unsigned int b = lo, j = t - ibase[b], nr = ibase[b + 1] - ibase[b];
  const uint8_t* base = view_of(S, b);
  const unsigned int len = S.vlen[b];
  const unsigned int ents_end = len - 4 - 4 * nr;
  const uint8_t* rs = base + ents_end;
  const unsigned int s = ld_le32(rs + 4 * j), e = j + 1 < nr ? ld_le32(rs + 4 * (j + 1)) : ents_end;
  if (s > e || e > ents_end || (j == 0 && s != 0)) { raise(err, SST_CORRUPT); return false; }
  iv->p = base + s; iv->end = base + e;
  return true;
}

__global__ void sst_count_kernel(SstView S, const unsigned int* ibase, unsigned int n_iv, unsigned int* cnt_n, unsigned long long* cnt_k, unsigned long long* cnt_v,
                                 unsigned int* err) {
  const unsigned int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > n_iv) return;
  if (t == n_iv) { cnt_n[t] = 0; cnt_k[t] = 0; cnt_v[t] = 0; return; }
  unsigned int n = 0;
  unsigned long long kb = 0, vb = 0;
  Interval iv;
  if (interval_of(S, ibase, t, &iv, err)) {
    const uint8_t* p = iv.p;
    unsigned int pfl = 0;
    bool first = true;
#pragma unroll 1
    while (p < iv.end) {
      unsigned int sh, ns, vl, u;
      if (!(u = get_var32(p, iv.end, &sh))) { raise(err, SST_CORRUPT); break; }
      p += u;
      if (!(u = get_var32(p, iv.end, &ns))) { raise(err, SST_CORRUPT); break; }
      p += u;
      if (!(u = get_var32(p, iv.end, &vl))) { raise(err, SST_CORRUPT); break; }
      p += u;
      const unsigned long long fl = (unsigned long long)sh + ns;
      if ((first && sh != 0) || sh > pfl || fl < (unsigned long long)S.pl + S.sl || fl > 0xffffffu || (unsigned long long)(iv.end - p) < (unsigned long long)ns + vl) {
        raise(err, SST_CORRUPT);
        break;
      }
      p += ns + vl;
      pfl = (unsigned int)fl;
      first = false;
      ++n; kb += fl - S.pl - S.sl; vb += vl;
    }
  }
  cnt_n[t] = n; cnt_k[t] = kb; cnt_v[t] = vb;
}

struct FlatOut { uint8_t* keys; unsigned int* koff; uint8_t* vals; unsigned int* voff; };

// One warp per restart interval.  The current full key lives in the warp's registers, byte j in lane j % 32, slot j / 32
// (four slots: keys up to 128 bytes), so "keep the first `shared` bytes, take the rest from the entry" is a predicated
// byte load per slot with consecutive lanes on consecutive addresses, and the key leaves as consecutive byte stores: the
// heaps are written in full sectors.  Headers are parsed by every lane alike (same addresses: one transaction).  A key
// longer than 128 bytes sends the rest of its interval down the sequential path on lane 0, which rebuilds keys from
// the previous key in the output heap.
__global__ void __launch_bounds__(256) sst_expand_kernel(SstView S, const unsigned int* ibase, unsigned int n_iv, const unsigned int* base_n,
                                                         const unsigned long long* base_k, const unsigned long long* base_v, FlatOut O, unsigned int* err) {
  const unsigned int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (t > n_iv) return;
  if (t == n_iv) { if (lane == 0) { O.koff[base_n[t]] = (unsigned int)base_k[t]; O.voff[base_n[t]] = (unsigned int)base_v[t]; } return; }
  Interval iv;
  if (!interval_of(S, ibase, t, &iv, err)) return;
  unsigned int e = base_n[t];
  const unsigned int e_end = base_n[t + 1];
  unsigned int ko = (unsigned int)base_k[t], vo = (unsigned int)base_v[t];
  const uint8_t* p = iv.p;
  const unsigned int PL = S.pl, SL = S.sl;
  unsigned int kb0 = 0, kb1 = 0, kb2 = 0, kb3 = 0;  // bytes lane, 32 + lane, 64 + lane, 96 + lane of the current full key
  unsigned int pfl = 0, pko = 0;
#pragma unroll 1
  while (e < e_end) {  // (validated by sst_count_kernel)
    unsigned int sh, ns, vl;
    p += get_var32(p, iv.end, &sh);
    p += get_var32(p, iv.end, &ns);
    p += get_var32(p, iv.end, &vl);
    const unsigned int fl = sh + ns;
    if (fl > 128) break;
    const unsigned int body_end = fl - SL;
    if (lane == 0) { O.koff[e] = ko; O.voff[e] = vo; }
#define SST_SLOT(kb, base)                                                          \
    if ((base) < fl) {                                                                \
      const unsigned int j = (base) + lane;                                           \
      if (j >= sh && j < fl) kb = p[j - sh];                                          \
      if (j >= PL && j < body_end) O.keys[ko + (j - PL)] = (uint8_t)kb;               \
      if (SL == 8 && j == body_end && kb != 1) raise(err, SST_UNSUPPORTED);           \
    }
    SST_SLOT(kb0, 0u) SST_SLOT(kb1, 32u) SST_SLOT(kb2, 64u) SST_SLOT(kb3, 96u)
#undef SST_SLOT
    p += ns;
#pragma unroll 1
    for (unsigned int i = lane; i < vl; i += 32) O.vals[vo + i] = p[i];
    p += vl;
    pko = ko; pfl = fl;
    ko += body_end - PL; vo += vl;
    ++e;
  }
  if (e >= e_end) return;
  // ---- sequential path (lane 0): the interval holds a key longer than 128 bytes ----
  // footer of the previous key (it is not in the output heap): gather its SL bytes from the lanes
  unsigned long long psuf = 0;
  if (SL == 8 && pfl) {
    for (unsigned int q = 0; q < 8; ++q) {
      const unsigned int j = pfl - 8 + q, slot = j >> 5;
      const unsigned int v = slot == 0 ? kb0 : (slot == 1 ? kb1 : (slot == 2 ? kb2 : kb3));
      psuf |= (unsigned long long)(__shfl_sync(0xffffffffu, v, j & 31) & 0xff) << (8 * q);
    }
  }
  __syncwarp();
  if (lane != 0) return;
  // (p was advanced past the three varints of entry e: walk again from its start)
  const uint8_t* q = iv.p;
  {  // re-find entry e's start: entries before it were consumed in order
    unsigned int skip = e - base_n[t];
    while (skip--) { unsigned int a, b, c; q += get_var32(q, iv.end, &a); q += get_var32(q, iv.end, &b); q += get_var32(q, iv.end, &c); q += b + c; }
  }
  const volatile uint8_t* okeys = O.keys;  // bytes other lanes stored: read them back from memory, not from a stale L1 line
#pragma unroll 1
  while (e < e_end) {
    unsigned int sh, ns, vl;
    q += get_var32(q, iv.end, &sh);
    q += get_var32(q, iv.end, &ns);
    q += get_var32(q, iv.end, &vl);
    const unsigned int fl = sh + ns, body_end = fl - SL, pbody_end = pfl - SL;
    unsigned long long suf = 0;
    O.koff[e] = ko; O.voff[e] = vo;
#pragma unroll 1
    for (unsigned int j = PL; j < fl; ++j) {
      uint8_t c;
      if (j < sh) c = j < pbody_end ? okeys[pko + (j - PL)] : (uint8_t)(psuf >> (8 * (j - pbody_end)));
      else c = q[j - sh];
      if (j < body_end) O.keys[ko + (j - PL)] = c;
      else suf |= (unsigned long long)c << (8 * (j - body_end));
    }
    if (SL == 8 && (suf & 0xff) != 1) raise(err, SST_UNSUPPORTED);  // kTypeDeletion / Merge / ...: the host's merging iterator must resolve them
    q += ns;
#pragma unroll 1
    for (unsigned int i = 0; i < vl; ++i) O.vals[vo + i] = q[i];
    q += vl;
    pko = ko; pfl = fl; psuf = suf;
    ko += body_end - PL; vo += vl;
    ++e;
  }
}

// ---- merge of sorted runs (b2_sst_merge; the per-entry rules in sst_merge.h) ----
struct Flat { const uint8_t* keys; const unsigned int* koff; const uint8_t* vals; const unsigned int* voff; };
struct Staged { uint8_t* keys; unsigned int* koff; };

// One thread per entry of one decoded run (keys with their footer, already copied to the staged heap at k0): the run's
// offsets join the staged block at entry n0, the entry is checked against the one before it, and its staged footer
// becomes the effective one (the global seqno of an ingested run).
__global__ void sst_stage_kernel(Flat R, unsigned int n, Staged T, unsigned int* tvoff, unsigned int n0, unsigned int k0, unsigned int v0,
                                 unsigned long long global_seq, unsigned int* err) {
  const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  T.koff[n0 + i] = k0 + R.koff[i]; tvoff[n0 + i] = v0 + R.voff[i];
  if (i == n) return;
  const unsigned int ks = R.koff[i], len = R.koff[i + 1] - ks;
  const unsigned int ps = i ? R.koff[i - 1] : 0;
  uint64_t eff;
  const unsigned int st = b2merge::stage_check(R.keys + ks, len, i ? R.keys + ps : nullptr, ks - ps, global_seq, &eff);
  if (st) { raise(err, st); return; }
  uint8_t* f = T.keys + k0 + ks + len - 8;
#pragma unroll
  for (int q = 0; q < 8; ++q) f[q] = (uint8_t)(eff >> (8 * q));
}

__global__ void sst_iota_kernel(unsigned int* ids, unsigned int n) {
  const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ids[i] = i;
}

// Internal-key order over staged entry ids; equal internal keys keep the order of their ids, i.e. of the runs as listed.
struct StagedLess {
  const uint8_t* keys;
  const unsigned int* koff;
  __device__ __forceinline__ bool operator()(unsigned int a, unsigned int b) const {
    const unsigned int sa = koff[a], sb = koff[b];
    const int c = b2merge::ikey_cmp(keys + sa, koff[a + 1] - sa, keys + sb, koff[b + 1] - sb);
    return c ? c < 0 : a < b;
  }
};

// One thread per merged position (and one past the end, which zeroes the scans' last element): its verdict, its kept
// lengths and the stats counters stat[0..2] = invisible, hidden, deleted.
__global__ void sst_visible_kernel(Staged T, const unsigned int* ids, unsigned int n, unsigned long long snapshot_seq, unsigned int* keep_n,
                                   unsigned int* keep_k, unsigned int* keep_v, const unsigned int* voff, unsigned long long* stat) {
  const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned int v = b2merge::kOut + 10;  // (no position: counts nothing)
  if (i < n) {
    const unsigned int id = ids[i], s = T.koff[id], len = T.koff[id + 1] - s, bl = b2merge::body_len(len);
    const uint64_t f = b2merge::footer_of(T.keys + s + bl, 8);
    bool same = false;
    uint64_t pf = 0;
    if (i) {
      const unsigned int pid = ids[i - 1], ps = T.koff[pid], pbl = b2merge::body_len(T.koff[pid + 1] - ps);
      same = b2merge::user_key_cmp(T.keys + ps, pbl, T.keys + s, bl) == 0;
      pf = b2merge::footer_of(T.keys + ps + pbl, 8);
    }
    v = b2merge::verdict(f, same, pf, snapshot_seq);
    const bool keep = v == b2merge::kOut;
    keep_n[i] = keep; keep_k[i] = keep ? bl : 0; keep_v[i] = keep ? voff[id + 1] - voff[id] : 0;
  } else if (i == n) {
    keep_n[i] = 0; keep_k[i] = 0; keep_v[i] = 0;
  }
  const unsigned int mask = __activemask();
  const unsigned int a = __reduce_add_sync(mask, v == b2merge::kInvisible), h = __reduce_add_sync(mask, v == b2merge::kHidden),
                     d = __reduce_add_sync(mask, v == b2merge::kDeleted);
  if ((threadIdx.x & 31) == __ffs(mask) - 1) {
    if (a) atomicAdd(stat + 0, (unsigned long long)a);
    if (h) atomicAdd(stat + 1, (unsigned long long)h);
    if (d) atomicAdd(stat + 2, (unsigned long long)d);
  }
}

// One warp per merged position: a kept entry's key body and value leave as consecutive byte stores, as in sst_expand.
__global__ void __launch_bounds__(256) sst_gather_kernel(Staged T, const unsigned int* tvoff, const uint8_t* tvals, const unsigned int* ids, unsigned int n,
                                                         const unsigned int* keep_n, const unsigned int* keep_k, const unsigned int* keep_v, FlatOut O) {
  const unsigned int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i > n) return;
  const unsigned int e = keep_n[i], ko = keep_k[i], vo = keep_v[i];
  if (i == n) { if (lane == 0) { O.koff[e] = ko; O.voff[e] = vo; } return; }
  if (keep_n[i + 1] == e) return;
  const unsigned int id = ids[i], kl = keep_k[i + 1] - ko, vl = keep_v[i + 1] - vo;
  if (lane == 0) { O.koff[e] = ko; O.voff[e] = vo; }
  const uint8_t* k = T.keys + T.koff[id];
  const uint8_t* v = tvals + tvoff[id];
#pragma unroll 1
  for (unsigned int j = lane; j < kl; j += 32) O.keys[ko + j] = k[j];
#pragma unroll 1
  for (unsigned int j = lane; j < vl; j += 32) O.vals[vo + j] = v[j];
}

// ---- encoder (tooling) ----
struct FlatIn { const uint8_t* keys; const unsigned int* koff; const uint8_t* vals; const unsigned int* voff; unsigned int n; };
struct EncOpt { unsigned int per_block, restart, pl, sl, trailer; uint8_t prefix_byte; };

__device__ __forceinline__ unsigned int full_len(const FlatIn& F, const EncOpt& o, unsigned int e) { return o.pl + (F.koff[e + 1] - F.koff[e]) + o.sl; }
__device__ __forceinline__ uint8_t full_byte(const FlatIn& F, const EncOpt& o, unsigned int e, unsigned int j) {
  if (j < o.pl) return o.prefix_byte;
  const unsigned int kl = F.koff[e + 1] - F.koff[e];
  if (j < o.pl + kl) return F.keys[F.koff[e] + (j - o.pl)];
  return j == o.pl + kl ? 1 : 0;  // fixed64 LE of (seq 0 << 8 | kTypeValue)
}
__device__ __forceinline__ unsigned int var32_len(unsigned int v) { return v < (1u << 7) ? 1 : (v < (1u << 14) ? 2 : (v < (1u << 21) ? 3 : (v < (1u << 28) ? 4 : 5))); }
__device__ __forceinline__ unsigned int put_var32(uint8_t* p, unsigned int v) {
  unsigned int i = 0;
  while (v >= 0x80) { p[i++] = (uint8_t)(v | 0x80); v >>= 7; }
  p[i++] = (uint8_t)v;
  return i;
}
__device__ __forceinline__ unsigned int shared_with_prev(const FlatIn& F, const EncOpt& o, unsigned int e) {
  if (e % o.per_block % o.restart == 0) return 0;
  const unsigned int a = full_len(F, o, e - 1), b = full_len(F, o, e), m = a < b ? a : b;
  unsigned int j = 0;
  while (j < m && full_byte(F, o, e - 1, j) == full_byte(F, o, e, j)) ++j;
  return j;
}

__global__ void sst_enc_size_kernel(FlatIn F, EncOpt o, unsigned long long* sizes /* n + 1, last = 0 */) {
  const unsigned int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e > F.n) return;
  if (e == F.n) { sizes[e] = 0; return; }
  const unsigned int sh = shared_with_prev(F, o, e), ns = full_len(F, o, e) - sh, vl = F.voff[e + 1] - F.voff[e];
  sizes[e] = var32_len(sh) + var32_len(ns) + var32_len(vl) + ns + vl;
}

__global__ void sst_enc_write_kernel(FlatIn F, EncOpt o, const unsigned long long* pre /* exclusive sums, n + 1 */, unsigned int n_blocks, uint8_t* out,
                                     unsigned long long* boffs) {
  const unsigned int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= F.n) return;
  const unsigned int b = e / o.per_block, i = e % o.per_block;
  const unsigned int nr_full = (o.per_block + o.restart - 1) / o.restart;
  const unsigned long long ovh = 4ull * nr_full + 4 + o.trailer;  // of every block before the last
  const unsigned int first = b * o.per_block, last = first + o.per_block < F.n ? first + o.per_block : F.n;
  const unsigned long long bstart = pre[first] + ovh * b;
  const unsigned int ent_off = (unsigned int)(pre[e] - pre[first]), ents_len = (unsigned int)(pre[last] - pre[first]);
  const unsigned int nr = (last - first + o.restart - 1) / o.restart;
  uint8_t* p = out + bstart + ent_off;
  const unsigned int sh = shared_with_prev(F, o, e), fl = full_len(F, o, e), ns = fl - sh, vl = F.voff[e + 1] - F.voff[e];
  p += put_var32(p, sh); p += put_var32(p, ns); p += put_var32(p, vl);
  for (unsigned int j = sh; j < fl; ++j) *p++ = full_byte(F, o, e, j);
  const uint8_t* v = F.vals + F.voff[e];
  for (unsigned int j = 0; j < vl; ++j) *p++ = v[j];
  uint8_t* tail = out + bstart + ents_len;
  if (i % o.restart == 0) { const unsigned int r = i / o.restart; tail[4 * r] = (uint8_t)ent_off; tail[4 * r + 1] = (uint8_t)(ent_off >> 8); tail[4 * r + 2] = (uint8_t)(ent_off >> 16); tail[4 * r + 3] = (uint8_t)(ent_off >> 24); }
  if (i == 0) {
    uint8_t* f = tail + 4 * nr;
    f[0] = (uint8_t)nr; f[1] = (uint8_t)(nr >> 8); f[2] = (uint8_t)(nr >> 16); f[3] = (uint8_t)(nr >> 24);
    for (unsigned int j = 0; j < o.trailer; ++j) f[4 + j] = 0;  // compression type 0 (none), checksum field left zero
    boffs[b] = bstart;
    if (b + 1 == n_blocks) boffs[n_blocks] = bstart + ents_len + 4ull * nr + 4 + o.trailer;
  }
}

// A growable device allocation, freed with the buffer (moving leaves the source empty).  Not pooled on purpose: decoded
// blocks are large and long-lived.
struct RawBuf {
  void* p = nullptr;
  size_t cap = 0;
  RawBuf() = default;
  RawBuf(RawBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  RawBuf& operator=(RawBuf&& o) noexcept {
    if (this != &o) { free(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  ~RawBuf() { free(); }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    free();
    n = (n + 255) & ~(size_t)255;
    cudaError_t e = cudaMalloc(&p, n);
    if (e == cudaSuccess) cap = n;
    return e;
  }
  // reserve, keeping the first `used` bytes (the stream's work on them is finished before the old allocation goes)
  cudaError_t grow(size_t n, size_t used, cudaStream_t st) {
    if (n <= cap) return cudaSuccess;
    if (n < 2 * cap) n = 2 * cap;
    n = (n + 255) & ~(size_t)255;
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, n);
    if (e == cudaSuccess && used) e = cudaMemcpyAsync(q, p, used, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { if (q) cudaFree(q); return e; }
    free();
    p = q; cap = n;
    return e;
  }
  void free() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

}  // namespace

struct b2_sst {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;  // ev2 .. ev3: b2_sst_merge's decode and staging
  RawBuf keys, koff, vals, voff;  // decoded block (b2_sst_decode)
  RawBuf enc, enc_offs;           // encoded blocks (b2_sst_encode)
  RawBuf boffs, nres, cnt_n, cnt_k, cnt_v, tmp, err;  // offsets, restart / entry counts and their prefix sums
  RawBuf view_off, view_len, isz, inflated;           // contents views; inflated sizes and bytes of LZ4 blocks
  RawBuf mkeys, mkoff, mvals, mvoff;                  // b2_sst_merge: every run decoded, back to back, footers kept
  RawBuf ids0, ids1, keep_n, keep_k, keep_v, mstat;    // merged order (ping-pong), kept counts / lengths, error + stats
  // (the buffers are freed after this, when the handle is deleted: the device is current and the stream drained by then)
  void destroy() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (ev2) cudaEventDestroy(ev2);
    if (ev3) cudaEventDestroy(ev3);
    if (stream) cudaStreamDestroy(stream);
  }
};

namespace {
// The compressed bytes of a host-resident run are staged in one of two per-device buffers (shared by every handle: the 16
// regions of a request do not keep 16 copies of their compressed form).  Two, so that two requests (threads) overlap:
// while one expands its run, the other's bytes cross PCIe.
struct Staging {
  std::mutex mu;
  RawBuf buf;
};
Staging* staging_acquire(int device) {
  static auto* st = new Staging[64][2];  // leaked on purpose: freeing them at exit would run after the CUDA runtime's teardown
  Staging* a = st[device & 63];
  if (a[0].mu.try_lock()) return &a[0];
  if (a[1].mu.try_lock()) return &a[1];
  a[0].mu.lock();
  return &a[0];
}
int sst_fail(int st, const std::string& m) { b2::set_last_error(m); return st; }
#define SST_TRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return sst_fail(B2_ERR_CUDA, std::string("b2_sst: ") + #x + ": " + cudaGetErrorString(_e)); } while (0)

int sst_handle(int32_t device, b2_sst** h) {
  if (cudaSetDevice(device) != cudaSuccess) return sst_fail(B2_ERR_CUDA, "cudaSetDevice failed");
  if (*h) {
    if ((*h)->device != device) return sst_fail(B2_ERR_INVALID_ARG, "b2_sst: the handle belongs to another device");
    return B2_OK;
  }
  b2_sst* s = new b2_sst();
  s->device = device;
  if (cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreate(&s->ev0) != cudaSuccess || cudaEventCreate(&s->ev1) != cudaSuccess ||
      cudaEventCreate(&s->ev2) != cudaSuccess || cudaEventCreate(&s->ev3) != cudaSuccess) {
    s->destroy(); delete s;
    return sst_fail(B2_ERR_CUDA, "b2_sst: stream / event creation failed");
  }
  *h = s;
  return B2_OK;
}

template <typename T>
int scan_inplace(b2_sst* s, b2_sst& w, T* a, size_t n) {
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, a, a, (int)n, s->stream);
  SST_TRY(w.tmp.reserve(tb + 16));
  SST_TRY(cub::DeviceScan::ExclusiveSum(w.tmp.p, tb, a, a, (int)n, s->stream));
  return B2_OK;
}
int check_err(b2_sst* s, b2_sst& w, const char* who, const char* what) {
  unsigned int code = 0;
  SST_TRY(cudaMemcpyAsync(&code, w.err.p, 4, cudaMemcpyDeviceToHost, s->stream));
  SST_TRY(cudaStreamSynchronize(s->stream));
  if (code == SST_UNSUPPORTED)
    return sst_fail(B2_ERR_UNSUPPORTED, std::string(who) + ": " + what +
                                            ": a block compressed other than LZ4 / LZ4HC / ZSTD, a ZSTD frame that is not a plain frame without a "
                                            "dictionary, a data-block hash index or an entry whose value type is not kTypeValue");
  if (code) return sst_fail(B2_ERR_STORAGE, std::string(who) + ": " + what + ": corrupted data block");
  return B2_OK;
}

int check_blocks_arg(const b2_sst_blocks* in, const char* who) {
  if ((in->n_blocks && (!in->data || !in->block_offs)))
    return sst_fail(B2_ERR_INVALID_ARG, std::string(who) + ": null argument or bad location");
  if ((in->trailer_len != 0 && in->trailer_len != 5) || (in->key_suffix_len != 0 && in->key_suffix_len != 8) || in->key_prefix_len > 64 || in->n_blocks >= (1u << 30))
    return sst_fail(B2_ERR_INVALID_ARG, std::string(who) + ": trailer_len is 0 or 5, key_suffix_len 0 or 8, key_prefix_len <= 64");
  return B2_OK;
}

struct Decoded {
  uint32_t n_ent = 0, n_iv = 0, n_lz4 = 0;
  uint64_t kb = 0, vb = 0, h2d = 0;
  float ms = 0.f;  // device time, ev0 .. ev1
};

// The one decode path: `in` (validated by check_blocks_arg) -> the flat block in the handle's keys / koff / vals / voff,
// padded as b2_cf_block asks.  `sl` is the footer length dropped from every key: in->key_suffix_len for b2_sst_decode,
// 0 for b2_sst_merge, which keeps the footer.  Blocking.
int decode_run(b2_sst* s, int32_t device, int32_t location, const b2_sst_blocks* in, uint32_t sl, const char* who, Decoded* r) {
  int rc;
  b2_sst& w = *s;
  const uint32_t nb = in->n_blocks;
  for (uint32_t b = 0; b < nb; ++b)
    if (in->block_offs[b + 1] < in->block_offs[b]) return sst_fail(B2_ERR_INVALID_ARG, std::string(who) + ": block_offs must ascend");
  const uint64_t lo = nb ? in->block_offs[0] : 0, hi = nb ? in->block_offs[nb] : 0;
  uint64_t h2d = 0;
  SST_TRY(w.err.reserve(32));
  SST_TRY(cudaMemsetAsync(w.err.p, 0, 32, s->stream));
  SST_TRY(w.boffs.reserve(((size_t)nb + 1) * 8));
  std::vector<uint64_t> rel((size_t)nb + 1, 0);
  for (uint32_t b = 0; b <= nb && nb; ++b) rel[b] = in->block_offs[b] - lo;
  SST_TRY(cudaMemcpyAsync(w.boffs.p, rel.data(), rel.size() * 8, cudaMemcpyHostToDevice, s->stream));
  h2d += rel.size() * 8;
  SST_TRY(w.view_off.reserve(((size_t)nb + 1) * 8)); SST_TRY(w.view_len.reserve(((size_t)nb + 1) * 4));
  SstView S;
  const ViewOut V{(unsigned long long*)w.view_off.p, (unsigned int*)w.view_len.p};
  S.inflated = nullptr; S.voff = V.off; S.vlen = V.len;
  S.boffs = (const unsigned long long*)w.boffs.p; S.n_blocks = nb; S.trailer = in->trailer_len; S.pl = in->key_prefix_len; S.sl = sl;
  struct StagingHold {  // released on every return path
    Staging* st = nullptr;
    ~StagingHold() { if (st) st->mu.unlock(); }
  } hold;
  if (location == B2_LOC_HOST) {
    hold.st = staging_acquire(device);
    SST_TRY(hold.st->buf.reserve((size_t)(hi - lo) + 16));
    if (hi > lo) SST_TRY(cudaMemcpyAsync(hold.st->buf.p, in->data + lo, (size_t)(hi - lo), cudaMemcpyHostToDevice, s->stream));
    h2d += hi - lo;
    S.data = (const uint8_t*)hold.st->buf.p;
  } else S.data = in->data + lo;
  SST_TRY(cudaEventRecord(s->ev0, s->stream));
  uint32_t n_iv = 0, n_ent = 0, n_lz4 = 0, n_zstd = 0;
  uint64_t kb = 0, vb = 0;
  if (nb) {
    unsigned int* err = (unsigned int*)w.err.p;  // [0] error code, [1] LZ4 blocks, [2..3] LZ4 and ZSTD inflated bytes (u64), [4] ZSTD blocks
    unsigned long long* lz4_bytes = (unsigned long long*)(err + 2);
    uint32_t counts[4] = {0, 0, 0, 0};  // err[1..4]
    uint64_t total = 0;
    SST_TRY(w.nres.reserve(((size_t)nb + 1) * 4)); SST_TRY(w.isz.reserve(((size_t)nb + 1) * 8));
    sst_blocks_kernel<<<(nb + 1 + 255) / 256, 256, 0, s->stream>>>(S, V, (unsigned int*)w.nres.p, (unsigned long long*)w.isz.p, err + 1, lz4_bytes, err + 4, 0, err);
    if ((rc = scan_inplace(s, w, (unsigned int*)w.nres.p, (size_t)nb + 1))) return rc;
    SST_TRY(cudaMemcpyAsync(&n_iv, (unsigned int*)w.nres.p + nb, 4, cudaMemcpyDeviceToHost, s->stream));
    SST_TRY(cudaMemcpyAsync(counts, err + 1, 16, cudaMemcpyDeviceToHost, s->stream));
    if ((rc = check_err(s, w, who, "block footers"))) return rc;
    n_lz4 = counts[0]; n_zstd = counts[3];
    memcpy(&total, counts + 1, 8);
    if (n_lz4 || n_zstd) {  // inflate the compressed blocks, then count the restarts of every block again from the views: one more round trip
      if ((rc = scan_inplace(s, w, (unsigned long long*)w.isz.p, (size_t)nb + 1))) return rc;
      SST_TRY(w.inflated.reserve((size_t)total + 16));
      S.inflated = (const uint8_t*)w.inflated.p;
      if (n_lz4) sst_inflate_kernel<<<(unsigned int)(((size_t)nb + 7) / 8), 256, 0, s->stream>>>(S, V, (const unsigned long long*)w.isz.p, err);
      if (n_zstd)
        sst_zstd_kernel<<<(unsigned int)(((size_t)nb + kZstdWarps - 1) / kZstdWarps), 32 * kZstdWarps, 0, s->stream>>>(S, V, (const unsigned long long*)w.isz.p, err);
      sst_blocks_kernel<<<(nb + 1 + 255) / 256, 256, 0, s->stream>>>(S, V, (unsigned int*)w.nres.p, nullptr, nullptr, nullptr, nullptr, 1, err);
      if ((rc = scan_inplace(s, w, (unsigned int*)w.nres.p, (size_t)nb + 1))) return rc;
      SST_TRY(cudaMemcpyAsync(&n_iv, (unsigned int*)w.nres.p + nb, 4, cudaMemcpyDeviceToHost, s->stream));
      if ((rc = check_err(s, w, who, "compressed blocks"))) return rc;
    }
    if (n_iv >= 0x7ffffff0u) return sst_fail(B2_ERR_INVALID_ARG, std::string(who) + ": too many restart intervals in one call: pass fewer data blocks");
    SST_TRY(w.cnt_n.reserve(((size_t)n_iv + 1) * 4)); SST_TRY(w.cnt_k.reserve(((size_t)n_iv + 1) * 8)); SST_TRY(w.cnt_v.reserve(((size_t)n_iv + 1) * 8));
    sst_count_kernel<<<(n_iv + 1 + 127) / 128, 128, 0, s->stream>>>(S, (const unsigned int*)w.nres.p, n_iv, (unsigned int*)w.cnt_n.p, (unsigned long long*)w.cnt_k.p,
                                                                   (unsigned long long*)w.cnt_v.p, (unsigned int*)w.err.p);
    if ((rc = scan_inplace(s, w, (unsigned int*)w.cnt_n.p, (size_t)n_iv + 1))) return rc;
    if ((rc = scan_inplace(s, w, (unsigned long long*)w.cnt_k.p, (size_t)n_iv + 1))) return rc;
    if ((rc = scan_inplace(s, w, (unsigned long long*)w.cnt_v.p, (size_t)n_iv + 1))) return rc;
    SST_TRY(cudaMemcpyAsync(&n_ent, (unsigned int*)w.cnt_n.p + n_iv, 4, cudaMemcpyDeviceToHost, s->stream));
    SST_TRY(cudaMemcpyAsync(&kb, (unsigned long long*)w.cnt_k.p + n_iv, 8, cudaMemcpyDeviceToHost, s->stream));
    SST_TRY(cudaMemcpyAsync(&vb, (unsigned long long*)w.cnt_v.p + n_iv, 8, cudaMemcpyDeviceToHost, s->stream));
    if ((rc = check_err(s, w, who, "entries"))) return rc;
    if (kb > 0xfffffff0ull || vb > 0xfffffff0ull) return sst_fail(B2_ERR_INVALID_ARG, std::string(who) + ": a decoded heap exceeds 4 GiB (u32 offsets): pass fewer data blocks per call");
  }
  // heaps padded as b2_cf_block asks (16-byte lines + 16 readable bytes past the end)
  SST_TRY(s->keys.reserve(((size_t)kb + 47) & ~(size_t)15)); SST_TRY(s->vals.reserve(((size_t)vb + 47) & ~(size_t)15));
  SST_TRY(s->koff.reserve(((size_t)n_ent + 1) * 4 + 16)); SST_TRY(s->voff.reserve(((size_t)n_ent + 1) * 4 + 16));
  FlatOut O;
  O.keys = (uint8_t*)s->keys.p; O.koff = (unsigned int*)s->koff.p; O.vals = (uint8_t*)s->vals.p; O.voff = (unsigned int*)s->voff.p;
  if (nb) {
    sst_expand_kernel<<<(unsigned int)(((size_t)n_iv + 1 + 7) / 8), 256, 0, s->stream>>>(S, (const unsigned int*)w.nres.p, n_iv, (const unsigned int*)w.cnt_n.p,
                                                                    (const unsigned long long*)w.cnt_k.p, (const unsigned long long*)w.cnt_v.p, O, (unsigned int*)w.err.p);
    SST_TRY(cudaGetLastError());
  } else {
    SST_TRY(cudaMemsetAsync(s->koff.p, 0, 4, s->stream)); SST_TRY(cudaMemsetAsync(s->voff.p, 0, 4, s->stream));
  }
  SST_TRY(cudaMemsetAsync((uint8_t*)s->keys.p + kb, 0, (((size_t)kb + 47) & ~(size_t)15) - kb, s->stream));
  SST_TRY(cudaMemsetAsync((uint8_t*)s->vals.p + vb, 0, (((size_t)vb + 47) & ~(size_t)15) - vb, s->stream));
  SST_TRY(cudaEventRecord(s->ev1, s->stream));
  if ((rc = check_err(s, w, who, "entries"))) return rc;
  r->n_ent = n_ent; r->n_iv = n_iv; r->n_lz4 = n_lz4; r->kb = kb; r->vb = vb; r->h2d = h2d;
  cudaEventElapsedTime(&r->ms, s->ev0, s->ev1);
  return B2_OK;
}
}  // namespace

extern "C" {

int32_t b2_sst_decode(int32_t device, int32_t location, const b2_sst_blocks* in, b2_sst** hp, b2_cf_block* out, b2_sst_stats* stats) {
  if (!in || !hp || !out || (location != B2_LOC_HOST && location != B2_LOC_DEVICE))
    return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_decode: null argument or bad location");
  int rc = check_blocks_arg(in, "b2_sst_decode");
  if (rc) return rc;
  if ((rc = sst_handle(device, hp))) return rc;
  b2_sst* s = *hp;
  Decoded d;
  if ((rc = decode_run(s, device, location, in, in->key_suffix_len, "b2_sst_decode", &d))) return rc;
  memset(out, 0, sizeof(*out));
  out->keys = (const uint8_t*)s->keys.p; out->key_offs = (const uint32_t*)s->koff.p; out->vals = (const uint8_t*)s->vals.p; out->val_offs = (const uint32_t*)s->voff.p;
  out->n = d.n_ent;
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_entries = d.n_ent; stats->key_bytes = d.kb; stats->val_bytes = d.vb; stats->n_restart_intervals = d.n_iv; stats->h2d_bytes = d.h2d;
    stats->n_lz4_blocks = d.n_lz4;
    stats->decode_ms = d.ms;
  }
  return B2_OK;
}

int32_t b2_sst_merge(int32_t device, int32_t location, const b2_sst_blocks* runs, uint32_t n_runs, const uint64_t* global_seqs, uint64_t snapshot_seq, b2_sst** hp,
                     b2_cf_block* out, b2_sst_merge_stats* stats) {
  const char* who = "b2_sst_merge";
  if (!hp || !out || (n_runs && !runs) || (location != B2_LOC_HOST && location != B2_LOC_DEVICE))
    return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_merge: null argument or bad location");
  if (n_runs > 1024 || snapshot_seq > b2merge::kMaxSeq) return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_merge: n_runs <= 1024 and snapshot_seq <= 2^56 - 1");
  int rc;
  for (uint32_t r = 0; r < n_runs; ++r) {
    if ((rc = check_blocks_arg(&runs[r], who))) return rc;
    if (runs[r].key_suffix_len != 8 || runs[r].key_prefix_len != runs[0].key_prefix_len || (global_seqs && global_seqs[r] > b2merge::kMaxSeq))
      return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_merge: every run has key_suffix_len 8 and the first run's key_prefix_len; global seqnos <= 2^56 - 1");
  }
  if ((rc = sst_handle(device, hp))) return rc;
  b2_sst* s = *hp;
  b2_sst& w = *s;
  // 1. every run decoded with its footers, appended to the staged block (mkeys / mkoff / mvals / mvoff)
  SST_TRY(w.mstat.reserve(32));  // u64 [0] error code (low word), [1] invisible, [2] hidden, [3] deleted
  SST_TRY(cudaMemsetAsync(w.mstat.p, 0, 32, s->stream));
  unsigned int* merr = (unsigned int*)w.mstat.p;
  std::vector<uint32_t> base(n_runs + 1, 0);
  uint64_t k0 = 0, v0 = 0, h2d = 0;
  uint32_t n_lz4 = 0;
  SST_TRY(cudaEventRecord(s->ev2, s->stream));
  for (uint32_t r = 0; r < n_runs; ++r) {
    Decoded d;
    if ((rc = decode_run(s, device, location, &runs[r], 0, who, &d))) return rc;
    h2d += d.h2d; n_lz4 += d.n_lz4;
    const uint64_t n0 = base[r];
    if (n0 + d.n_ent >= 0x7fffff00ull || k0 + d.kb > 0xfffffff0ull || v0 + d.vb > 0xfffffff0ull)
      return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_merge: the runs hold more than 2^31 entries or a heap above 4 GiB (u32 offsets): merge fewer blocks per call");
    // (+16: the footer of a key shorter than 8 bytes, a corrupted run reported after the merge, is read inside the heap)
    SST_TRY(w.mkeys.grow((size_t)(k0 + d.kb) + 16, (size_t)k0, s->stream)); SST_TRY(w.mvals.grow((size_t)(v0 + d.vb) + 16, (size_t)v0, s->stream));
    SST_TRY(w.mkoff.grow((size_t)(n0 + d.n_ent + 1) * 4, (size_t)n0 * 4, s->stream)); SST_TRY(w.mvoff.grow((size_t)(n0 + d.n_ent + 1) * 4, (size_t)n0 * 4, s->stream));
    if (d.kb) SST_TRY(cudaMemcpyAsync((uint8_t*)w.mkeys.p + k0, s->keys.p, (size_t)d.kb, cudaMemcpyDeviceToDevice, s->stream));
    if (d.vb) SST_TRY(cudaMemcpyAsync((uint8_t*)w.mvals.p + v0, s->vals.p, (size_t)d.vb, cudaMemcpyDeviceToDevice, s->stream));
    const Flat R{(const uint8_t*)s->keys.p, (const unsigned int*)s->koff.p, (const uint8_t*)s->vals.p, (const unsigned int*)s->voff.p};
    sst_stage_kernel<<<(d.n_ent + 1 + 255) / 256, 256, 0, s->stream>>>(R, d.n_ent, Staged{(uint8_t*)w.mkeys.p, (unsigned int*)w.mkoff.p}, (unsigned int*)w.mvoff.p,
                                                                       (unsigned int)n0, (unsigned int)k0, (unsigned int)v0, global_seqs ? global_seqs[r] : 0, merr);
    SST_TRY(cudaGetLastError());
    k0 += d.kb; v0 += d.vb; base[r + 1] = (uint32_t)(n0 + d.n_ent);
  }
  SST_TRY(cudaEventRecord(s->ev3, s->stream));
  SST_TRY(cudaEventRecord(s->ev0, s->stream));
  const uint32_t N = base[n_runs];
  const Staged T{(uint8_t*)w.mkeys.p, (unsigned int*)w.mkoff.p};
  // 2. order: ceil(log2 n_runs) rounds of pairwise merges of adjacent segments, ping-ponging between ids0 and ids1
  SST_TRY(w.ids0.reserve((size_t)N * 4 + 16)); SST_TRY(w.ids1.reserve((size_t)N * 4 + 16));
  if (N) sst_iota_kernel<<<(N + 255) / 256, 256, 0, s->stream>>>((unsigned int*)w.ids0.p, N);
  const StagedLess less{T.keys, T.koff};
  unsigned int* ids = (unsigned int*)w.ids0.p;
  size_t tmax = 0;
  for (int run = 0; run < 2; ++run) {  // run 0 sizes the temporary storage of every merge, run 1 merges
    if (run) SST_TRY(w.tmp.reserve(tmax + 16));
    std::vector<uint32_t> b = base;
    unsigned int *src = (unsigned int*)w.ids0.p, *dst = (unsigned int*)w.ids1.p;
    while (b.size() > 2) {
      const size_t m = b.size() - 1;
      std::vector<uint32_t> nb;
      for (size_t j = 0; j < m; j += 2) {
        const uint32_t lo = b[j], mid = b[j + 1], hi = j + 1 < m ? b[j + 2] : mid;
        nb.push_back(lo);
        if (mid > lo && hi > mid) {
          size_t tb = run ? w.tmp.cap : 0;
          SST_TRY(cub::DeviceMerge::MergeKeys(run ? w.tmp.p : nullptr, tb, src + lo, (int)(mid - lo), src + mid, (int)(hi - mid), dst + lo, less, s->stream));
          if (tb > tmax) tmax = tb;
        } else if (run && hi > lo) SST_TRY(cudaMemcpyAsync(dst + lo, src + lo, (size_t)(hi - lo) * 4, cudaMemcpyDeviceToDevice, s->stream));
      }
      nb.push_back(b[m]);
      b.swap(nb);
      std::swap(src, dst);
    }
    ids = src;
  }
  // 3. visibility: kept counts and lengths, then their exclusive sums
  SST_TRY(w.keep_n.reserve((size_t)N * 4 + 16)); SST_TRY(w.keep_k.reserve((size_t)N * 4 + 16)); SST_TRY(w.keep_v.reserve((size_t)N * 4 + 16));
  unsigned int *keep_n = (unsigned int*)w.keep_n.p, *keep_k = (unsigned int*)w.keep_k.p, *keep_v = (unsigned int*)w.keep_v.p;
  sst_visible_kernel<<<(N + 1 + 255) / 256, 256, 0, s->stream>>>(T, ids, N, snapshot_seq, keep_n, keep_k, keep_v, (const unsigned int*)w.mvoff.p,
                                                                 (unsigned long long*)w.mstat.p + 1);
  if ((rc = scan_inplace(s, w, keep_n, (size_t)N + 1))) return rc;
  if ((rc = scan_inplace(s, w, keep_k, (size_t)N + 1))) return rc;
  if ((rc = scan_inplace(s, w, keep_v, (size_t)N + 1))) return rc;
  uint32_t tot[3];
  uint64_t st[4];
  SST_TRY(cudaMemcpyAsync(tot, keep_n + N, 4, cudaMemcpyDeviceToHost, s->stream));
  SST_TRY(cudaMemcpyAsync(tot + 1, keep_k + N, 4, cudaMemcpyDeviceToHost, s->stream));
  SST_TRY(cudaMemcpyAsync(tot + 2, keep_v + N, 4, cudaMemcpyDeviceToHost, s->stream));
  SST_TRY(cudaMemcpyAsync(st, w.mstat.p, 32, cudaMemcpyDeviceToHost, s->stream));
  SST_TRY(cudaStreamSynchronize(s->stream));
  if ((uint32_t)st[0] == SST_UNSUPPORTED)
    return sst_fail(B2_ERR_UNSUPPORTED, "b2_sst_merge: an entry whose value type is not kTypeValue, kTypeDeletion or kTypeSingleDeletion (Merge, BlobIndex, ...)");
  if ((uint32_t)st[0])
    return sst_fail(B2_ERR_STORAGE, "b2_sst_merge: a run not strictly ascending in internal-key order, a key shorter than its footer, or a stored sequence "
                                    "number other than 0 in a run with a global seqno");
  // 4. gather the kept entries into the handle's block, padded as b2_cf_block asks
  const uint32_t n_out = tot[0];
  const uint64_t kb = tot[1], vb = tot[2];
  SST_TRY(s->keys.reserve(((size_t)kb + 47) & ~(size_t)15)); SST_TRY(s->vals.reserve(((size_t)vb + 47) & ~(size_t)15));
  SST_TRY(s->koff.reserve(((size_t)n_out + 1) * 4 + 16)); SST_TRY(s->voff.reserve(((size_t)n_out + 1) * 4 + 16));
  FlatOut O;
  O.keys = (uint8_t*)s->keys.p; O.koff = (unsigned int*)s->koff.p; O.vals = (uint8_t*)s->vals.p; O.voff = (unsigned int*)s->voff.p;
  sst_gather_kernel<<<(unsigned int)(((size_t)N + 1 + 7) / 8), 256, 0, s->stream>>>(T, (const unsigned int*)w.mvoff.p, (const uint8_t*)w.mvals.p, ids, N, keep_n,
                                                                                keep_k, keep_v, O);
  SST_TRY(cudaGetLastError());
  SST_TRY(cudaMemsetAsync((uint8_t*)s->keys.p + kb, 0, (((size_t)kb + 47) & ~(size_t)15) - kb, s->stream));
  SST_TRY(cudaMemsetAsync((uint8_t*)s->vals.p + vb, 0, (((size_t)vb + 47) & ~(size_t)15) - vb, s->stream));
  SST_TRY(cudaEventRecord(s->ev1, s->stream));
  SST_TRY(cudaStreamSynchronize(s->stream));
  memset(out, 0, sizeof(*out));
  out->keys = O.keys; out->key_offs = O.koff; out->vals = O.vals; out->val_offs = O.voff; out->n = n_out;
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_in = N; stats->n_out = n_out; stats->n_invisible = st[1]; stats->n_hidden = st[2]; stats->n_deletions = st[3];
    stats->key_bytes = kb; stats->val_bytes = vb; stats->h2d_bytes = h2d;
    cudaEventElapsedTime(&stats->decode_ms, s->ev2, s->ev3);
    cudaEventElapsedTime(&stats->merge_ms, s->ev0, s->ev1);
    stats->n_lz4_blocks = n_lz4; stats->n_runs = n_runs;
  }
  return B2_OK;
}

void b2_sst_free(b2_sst* h) {
  if (!h) return;
  h->destroy();
  delete h;
}

int32_t b2_sst_encode(int32_t device, const b2_cf_block* flat, uint32_t entries_per_block, uint32_t restart_interval, uint32_t key_prefix_len, uint8_t key_prefix_byte,
                      uint32_t key_suffix_len, uint32_t trailer_len, b2_sst** hp, b2_sst_encoded* out) {
  if (!flat || !hp || !out || !entries_per_block || !restart_interval || (trailer_len != 0 && trailer_len != 5) || (key_suffix_len != 0 && key_suffix_len != 8) || key_prefix_len > 64)
    return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_encode: bad argument");
  int rc = sst_handle(device, hp);
  if (rc) return rc;
  b2_sst* s = *hp;
  b2_sst& w = *s;
  const uint32_t n = flat->n, nb = (n + entries_per_block - 1) / entries_per_block;
  FlatIn F; F.keys = flat->keys; F.koff = flat->key_offs; F.vals = flat->vals; F.voff = flat->val_offs; F.n = n;
  EncOpt o; o.per_block = entries_per_block; o.restart = restart_interval; o.pl = key_prefix_len; o.sl = key_suffix_len; o.trailer = trailer_len; o.prefix_byte = key_prefix_byte;
  memset(out, 0, sizeof(*out));
  SST_TRY(s->enc_offs.reserve(((size_t)nb + 1) * 8));
  SST_TRY(cudaMemsetAsync(s->enc_offs.p, 0, ((size_t)nb + 1) * 8, s->stream));
  uint64_t total = 0;
  if (n) {
    SST_TRY(w.cnt_k.reserve(((size_t)n + 1) * 8));
    sst_enc_size_kernel<<<(n + 1 + 255) / 256, 256, 0, s->stream>>>(F, o, (unsigned long long*)w.cnt_k.p);
    if ((rc = scan_inplace(s, w, (unsigned long long*)w.cnt_k.p, (size_t)n + 1))) return rc;
    uint64_t ent_bytes = 0;
    SST_TRY(cudaMemcpyAsync(&ent_bytes, (unsigned long long*)w.cnt_k.p + n, 8, cudaMemcpyDeviceToHost, s->stream));
    SST_TRY(cudaStreamSynchronize(s->stream));
    const uint32_t nr_full = (entries_per_block + restart_interval - 1) / restart_interval, last_n = n - (nb - 1) * entries_per_block;
    total = ent_bytes + (uint64_t)(nb - 1) * (4ull * nr_full + 4 + trailer_len) + 4ull * ((last_n + restart_interval - 1) / restart_interval) + 4 + trailer_len;
    SST_TRY(s->enc.reserve((size_t)total + 16));
    sst_enc_write_kernel<<<(n + 255) / 256, 256, 0, s->stream>>>(F, o, (const unsigned long long*)w.cnt_k.p, nb, (uint8_t*)s->enc.p, (unsigned long long*)s->enc_offs.p);
    SST_TRY(cudaGetLastError());
  }
  SST_TRY(cudaStreamSynchronize(s->stream));
  out->data = (const uint8_t*)s->enc.p; out->block_offs = (const uint64_t*)s->enc_offs.p; out->data_len = total; out->n_blocks = nb;
  return B2_OK;
}

}  // extern "C"
