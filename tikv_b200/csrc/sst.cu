// RocksDB BlockBasedTable data blocks -> the flat CF block layout of the scan kernels (SURVEY.md §8(f)4, b2_sst_decode),
// and the inverse as tooling (b2_sst_encode).  RocksDB is an external dependency of the reference (librocksdb behind
// components/engine_rocks); the block layout restated here is the published one:
//
//   data block := entry* restart[u32 LE x num_restarts] num_restarts[u32 LE]      (+ 5-byte trailer when stored)
//   entry      := varint32 shared | varint32 non_shared | varint32 value_len | key bytes [shared, shared + non_shared) | value
//   restart[j] := offset of an entry with shared == 0; one every block_restart_interval entries (16 by default)
//
// A restart interval is the unit of parallelism: one thread walks one interval (<= 16 entries in practice).  Three passes,
// each bounded by HBM traffic that is a small multiple of the block bytes:
//   sst_restarts  one thread per data block: reads the footer, validates it           -> restart points per block
//   sst_count     one thread per restart interval: entries, key bytes, value bytes   -> prefix sums give every
//                 interval its place in the flat block
//   sst_expand    one warp per restart interval: the current key lives in the warp's registers (byte j in lane j % 32),
//                 every entry overwrites the bytes past `shared` and streams the key, minus the data prefix and the
//                 internal-key footer (whose value type must be kTypeValue), and the value out as consecutive bytes
// The expansion runs an order of magnitude above the PCIe link the compressed bytes arrive over, which is the point:
// fewer bytes cross the link (53 instead of 69 per C3 entry).
#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b2_copr.h"

namespace b2 {
void set_last_error(const std::string& m);  // engine.cu (thread-local message behind b2_last_error_message)
}

namespace {

enum { SST_OK = 0, SST_CORRUPT = 1, SST_UNSUPPORTED = 2 };

struct SstView {
  const uint8_t* data;
  const unsigned long long* boffs;  // n_blocks + 1
  unsigned int n_blocks, trailer, pl, sl;
};

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

__global__ void sst_restarts_kernel(SstView S, unsigned int* nres /* n_blocks + 1, last = 0 */, unsigned int* err) {
  const unsigned int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > S.n_blocks) return;
  if (b == S.n_blocks) { nres[b] = 0; return; }
  const unsigned long long lo = S.boffs[b], hi = S.boffs[b + 1];
  unsigned int nr = 0;
  if (hi < lo || hi - lo < (unsigned long long)S.trailer + 4 || hi - lo > 0xffffff00ull) raise(err, SST_CORRUPT);
  else {
    const unsigned int len = (unsigned int)(hi - lo) - S.trailer;
    const unsigned int foot = ld_le32(S.data + lo + len - 4);
    if (foot >> 31) raise(err, SST_UNSUPPORTED);  // data block hash index packed into the footer
    else if (foot == 0 || (unsigned long long)foot * 4 + 4 > len) raise(err, SST_CORRUPT);
    else nr = foot;
  }
  nres[b] = nr;
}

struct Interval { const uint8_t *p, *end; };

// the entry bytes of restart interval t
__device__ __forceinline__ bool interval_of(const SstView& S, const unsigned int* ibase, unsigned int t, Interval* iv, unsigned int* err) {
  unsigned int lo = 0, hi = S.n_blocks;  // last block with ibase[b] <= t
  while (hi - lo > 1) { const unsigned int mid = (lo + hi) >> 1; if (ibase[mid] <= t) lo = mid; else hi = mid; }
  const unsigned int b = lo, j = t - ibase[b], nr = ibase[b + 1] - ibase[b];
  const uint8_t* base = S.data + S.boffs[b];
  const unsigned int len = (unsigned int)(S.boffs[b + 1] - S.boffs[b]) - S.trailer;
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
  void free() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

}  // namespace

struct b2_sst {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  RawBuf keys, koff, vals, voff;  // decoded block (b2_sst_decode)
  RawBuf enc, enc_offs;           // encoded blocks (b2_sst_encode)
  RawBuf boffs, nres, cnt_n, cnt_k, cnt_v, tmp, err;  // offsets, restart / entry counts and their prefix sums
  // (the buffers are freed after this, when the handle is deleted: the device is current and the stream drained by then)
  void destroy() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
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
  if (cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreate(&s->ev0) != cudaSuccess || cudaEventCreate(&s->ev1) != cudaSuccess) {
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
int check_err(b2_sst* s, b2_sst& w, const char* what) {
  unsigned int code = 0;
  SST_TRY(cudaMemcpyAsync(&code, w.err.p, 4, cudaMemcpyDeviceToHost, s->stream));
  SST_TRY(cudaStreamSynchronize(s->stream));
  if (code == SST_UNSUPPORTED) return sst_fail(B2_ERR_UNSUPPORTED, std::string("b2_sst_decode: ") + what + ": data-block hash index or an entry whose value type is not kTypeValue");
  if (code) return sst_fail(B2_ERR_STORAGE, std::string("b2_sst_decode: ") + what + ": corrupted data block");
  return B2_OK;
}
}  // namespace

extern "C" {

int32_t b2_sst_decode(int32_t device, int32_t location, const b2_sst_blocks* in, b2_sst** hp, b2_cf_block* out, b2_sst_stats* stats) {
  if (!in || !hp || !out || (location != B2_LOC_HOST && location != B2_LOC_DEVICE) || (in->n_blocks && (!in->data || !in->block_offs)))
    return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_decode: null argument or bad location");
  if ((in->trailer_len != 0 && in->trailer_len != 5) || (in->key_suffix_len != 0 && in->key_suffix_len != 8) || in->key_prefix_len > 64 || in->n_blocks >= (1u << 30))
    return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_decode: trailer_len is 0 or 5, key_suffix_len 0 or 8, key_prefix_len <= 64");
  int rc = sst_handle(device, hp);
  if (rc) return rc;
  b2_sst* s = *hp;
  b2_sst& w = *s;
  const uint32_t nb = in->n_blocks;
  for (uint32_t b = 0; b < nb; ++b)
    if (in->block_offs[b + 1] < in->block_offs[b]) return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_decode: block_offs must ascend");
  const uint64_t lo = nb ? in->block_offs[0] : 0, hi = nb ? in->block_offs[nb] : 0;
  uint64_t h2d = 0;
  SST_TRY(w.err.reserve(16));
  SST_TRY(cudaMemsetAsync(w.err.p, 0, 16, s->stream));
  SST_TRY(w.boffs.reserve(((size_t)nb + 1) * 8));
  std::vector<uint64_t> rel((size_t)nb + 1, 0);
  for (uint32_t b = 0; b <= nb && nb; ++b) rel[b] = in->block_offs[b] - lo;
  SST_TRY(cudaMemcpyAsync(w.boffs.p, rel.data(), rel.size() * 8, cudaMemcpyHostToDevice, s->stream));
  h2d += rel.size() * 8;
  SstView S;
  S.boffs = (const unsigned long long*)w.boffs.p; S.n_blocks = nb; S.trailer = in->trailer_len; S.pl = in->key_prefix_len; S.sl = in->key_suffix_len;
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
  uint32_t n_iv = 0, n_ent = 0;
  uint64_t kb = 0, vb = 0;
  if (nb) {
    SST_TRY(w.nres.reserve(((size_t)nb + 1) * 4));
    sst_restarts_kernel<<<(nb + 1 + 255) / 256, 256, 0, s->stream>>>(S, (unsigned int*)w.nres.p, (unsigned int*)w.err.p);
    if ((rc = scan_inplace(s, w, (unsigned int*)w.nres.p, (size_t)nb + 1))) return rc;
    SST_TRY(cudaMemcpyAsync(&n_iv, (unsigned int*)w.nres.p + nb, 4, cudaMemcpyDeviceToHost, s->stream));
    if ((rc = check_err(s, w, "block footers"))) return rc;
    if (n_iv >= 0x7ffffff0u) return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_decode: too many restart intervals in one call: pass fewer data blocks");
    SST_TRY(w.cnt_n.reserve(((size_t)n_iv + 1) * 4)); SST_TRY(w.cnt_k.reserve(((size_t)n_iv + 1) * 8)); SST_TRY(w.cnt_v.reserve(((size_t)n_iv + 1) * 8));
    sst_count_kernel<<<(n_iv + 1 + 127) / 128, 128, 0, s->stream>>>(S, (const unsigned int*)w.nres.p, n_iv, (unsigned int*)w.cnt_n.p, (unsigned long long*)w.cnt_k.p,
                                                                   (unsigned long long*)w.cnt_v.p, (unsigned int*)w.err.p);
    if ((rc = scan_inplace(s, w, (unsigned int*)w.cnt_n.p, (size_t)n_iv + 1))) return rc;
    if ((rc = scan_inplace(s, w, (unsigned long long*)w.cnt_k.p, (size_t)n_iv + 1))) return rc;
    if ((rc = scan_inplace(s, w, (unsigned long long*)w.cnt_v.p, (size_t)n_iv + 1))) return rc;
    SST_TRY(cudaMemcpyAsync(&n_ent, (unsigned int*)w.cnt_n.p + n_iv, 4, cudaMemcpyDeviceToHost, s->stream));
    SST_TRY(cudaMemcpyAsync(&kb, (unsigned long long*)w.cnt_k.p + n_iv, 8, cudaMemcpyDeviceToHost, s->stream));
    SST_TRY(cudaMemcpyAsync(&vb, (unsigned long long*)w.cnt_v.p + n_iv, 8, cudaMemcpyDeviceToHost, s->stream));
    if ((rc = check_err(s, w, "entries"))) return rc;
    if (kb > 0xfffffff0ull || vb > 0xfffffff0ull) return sst_fail(B2_ERR_INVALID_ARG, "b2_sst_decode: a decoded heap exceeds 4 GiB (u32 offsets): pass fewer data blocks per call");
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
  if ((rc = check_err(s, w, "entries"))) return rc;
  memset(out, 0, sizeof(*out));
  out->keys = O.keys; out->key_offs = O.koff; out->vals = O.vals; out->val_offs = O.voff; out->n = n_ent;
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_entries = n_ent; stats->key_bytes = kb; stats->val_bytes = vb; stats->n_restart_intervals = n_iv; stats->h2d_bytes = h2d;
    cudaEventElapsedTime(&stats->decode_ms, s->ev0, s->ev1);
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
