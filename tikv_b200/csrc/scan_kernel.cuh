// Device side of the fused scan kernel: helpers + scan_body<MODE>.  Included by kernels.cu (offline build) and, as is,
// by the translation unit NVRTC compiles for one plan at run time (B2_NVRTC defined; see jit.cpp).
#pragma once
#include "kernels.cuh"

namespace b2 {

template <class T> struct b2_remove_cvref { typedef T type; };
template <class T> struct b2_remove_cvref<const T&> { typedef T type; };
template <class T> struct b2_remove_cvref<T&> { typedef T type; };
template <class T> struct b2_remove_cvref<const T> { typedef T type; };

// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void report_err(Counters* c, uint64_t global_entry, int code) {
  atomicMin(&c->err, (unsigned long long)((global_entry << 8) | (unsigned)code));
  atomicMax(&c->err_max, (unsigned long long)((global_entry << 8) | (unsigned)code));
}

__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* p) {
  return *(const volatile unsigned long long*)p;
}
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned int* p, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---- HBM group table ----------------------------------------------------------------------------------
// returns slot index, or 0xffffffff when the table is full.  A key probes at most AGG_MAX_PROBES slots (the table has at
// least 2^16): a run that long only forms in a table close to full, and the engine then grows it and runs the request
// again.  Without the bound, the inserts after the table fills would each walk the whole table before giving up.
__device__ unsigned int table_find_or_insert(const AggTable& t, uint64_t key, bool is_null) {
  if (is_null || key == AGG_EMPTY_KEY) {
    const unsigned int which = is_null ? 0u : 1u;
    if (*(volatile unsigned int*)&t.special[which] == 0) atomicExch(&t.special[which], 1u);
    return t.cap + which;
  }
  unsigned int mask = t.cap - 1;
  unsigned int s = (unsigned int)mix64(key) & mask;
  for (unsigned int probes = 0; probes < AGG_MAX_PROBES; ++probes) {
    unsigned long long kk = ld_volatile_u64(&t.keys[s]);  // one L2 round trip per probe
    if (kk == AGG_EMPTY_KEY) kk = atomicCAS(&t.keys[s], AGG_EMPTY_KEY, (unsigned long long)key);
    if (kk == AGG_EMPTY_KEY || kk == key) return s;
    s = (s + 1) & mask;
  }
  return 0xffffffffu;
}

// Composite keys (BatchSlowHashAggregation): the table is keyed by a hash tag, claimed with one CAS; the winner then
// publishes the key words (release on ready[s]); a later arrival with an equal tag waits for them and compares: equal
// -> same group, different (a hash collision) -> keep probing.  `kw` = n_group value words + NULL mask.
//
// Called by all lanes `lanes` of one warp together, converged (`want`: this lane has a key to insert), which probe in
// lock step: every lane takes one probe step, the lanes that claimed a slot publish its key words, the lanes sync, and
// only then do the lanes that met an equal tag wait for that slot's key.  So no lane ever waits for a warp-mate that has
// yet to publish, and every wait is on a publisher that is already past its CAS and has nothing left to wait for.  A call
// still gives up after AGG_POLL_BUDGET reads of `ready` in all its probes (counted in agg_stuck; the engine then fails
// the request), so that a broken protocol shows up as a failed request rather than as a kernel that does not finish.
// Returns the slot, or 0xffffffff when the table is full (agg_overflow is set), the call gave up, or !want.
#define AGG_POLL_BUDGET (1u << 20)
__device__ __forceinline__ unsigned int table_find_or_insert_multi(const AggTable& t, Counters* ctr, unsigned int lanes, bool want, uint64_t tag,
                                                                   const uint64_t (&kw)[MAX_GROUP + 1], int n_words) {
  const unsigned int mask = t.cap - 1;
  unsigned int s = (unsigned int)tag & mask, probes = 0, polls = 0, slot = 0xffffffffu;
  bool done = !want;
  do {
    bool check = false;
    if (!done) {
      unsigned long long kk = ld_volatile_u64(&t.keys[s]);
      if (kk == AGG_EMPTY_KEY) {
        kk = atomicCAS(&t.keys[s], AGG_EMPTY_KEY, (unsigned long long)tag);
        if (kk == AGG_EMPTY_KEY) {
#pragma unroll
          for (int q = 0; q <= MAX_GROUP; ++q)
            if (q < n_words) t.gkeys[(size_t)s * n_words + q] = kw[q];
          __threadfence();
          st_release_u32(&t.ready[s], 1u);
          slot = s; done = true;
        }
      }
      check = !done && kk == tag;
    }
    __syncwarp(lanes);  // the claims of this step are published
    if (check) {
      bool published = false;
      while (!(published = ld_acquire_u32(&t.ready[s]) != 0) && ++polls < AGG_POLL_BUDGET) {}
      if (!published) { atomicAdd(&ctr->agg_stuck, 1u); done = true; }
      else {
        bool same = true;
#pragma unroll
        for (int q = 0; q <= MAX_GROUP; ++q)
          if (q < n_words) same = same && ld_volatile_u64(&t.gkeys[(size_t)s * n_words + q]) == kw[q];
        if (same) { slot = s; done = true; }
      }
    }
    if (!done) {
      s = (s + 1) & mask;
      if (++probes == AGG_MAX_PROBES) { atomicExch(&ctr->agg_overflow, 1u); done = true; }
    }
  } while (!__all_sync(lanes, done));
  if (probes > 64) atomicMax(&ctr->agg_probe_max, probes);  // (a healthy table at most half full stays far below)
  return slot;
}

// barrier over the 256 row-decoding threads only (the scan kernel runs a 9th, producer-only warp)
__device__ __forceinline__ void cta256_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// ---- TopN helpers --------------------------------------------------------------------------------------------
// Candidate buffer of a CTA (shared memory): `cap` packed candidates that never move plus a permutation `idx` (u16) of
// the slots.  A packed candidate is n_order + 2 u64 words: [order-by words][entry id][nulls | slot << 32] (32 bytes for
// two sort columns instead of the 48-byte TopItem, which keeps two CTAs per SM).  Positions [0, cnt) of `idx` are
// occupied; a new candidate takes position atomicAdd(cnt) -> slot idx[pos].  Compaction sorts the permutation (bitonic
// network over positions, every thread owns one compare-exchange per step) and keeps the best `limit` positions: only
// 2-byte indices are swapped.
struct TopBuf {
  unsigned long long* w;  // cap * stride words
  unsigned short* idx;    // cap
  unsigned int cap, stride, n;  // n = number of order-by columns
};
__device__ __forceinline__ TopBuf topbuf_make(unsigned char* smem, unsigned int cap, const DevPlan& P) {
  TopBuf t;
  t.n = (unsigned int)P.n_order; t.stride = t.n + 2; t.cap = cap;
  t.w = reinterpret_cast<unsigned long long*>(smem);
  t.idx = reinterpret_cast<unsigned short*>(t.w + (size_t)cap * t.stride);
  return t;
}
__device__ __forceinline__ void topbuf_put(const TopBuf& t, unsigned int slot, const TopItem& it) {
  unsigned long long* d = t.w + (size_t)slot * t.stride;
  for (unsigned int k = 0; k < t.n; ++k) d[k] = it.w[k];
  d[t.n] = it.id;
  d[t.n + 1] = (unsigned long long)it.nulls | ((unsigned long long)it.slot << 32);
}
__device__ __forceinline__ TopItem topbuf_get(const TopBuf& t, unsigned int slot) {
  const unsigned long long* d = t.w + (size_t)slot * t.stride;
  TopItem it;
  for (unsigned int k = 0; k < MAX_ORDER; ++k) it.w[k] = k < t.n ? d[k] : 0ull;
  it.id = d[t.n];
  it.nulls = (unsigned int)d[t.n + 1]; it.slot = (unsigned int)(d[t.n + 1] >> 32);
  return it;
}
// item_less on packed candidates (same order as b2_device.h item_less)
__device__ __forceinline__ bool topbuf_less(const TopBuf& t, unsigned int sa, unsigned int sb, const DevPlan& P) {
  const unsigned long long* a = t.w + (size_t)sa * t.stride;
  const unsigned long long* b = t.w + (size_t)sb * t.stride;
  const unsigned int na_all = (unsigned int)a[t.n + 1], nb_all = (unsigned int)b[t.n + 1];
  const bool ea = na_all >> 31, eb = nb_all >> 31;
  if (ea || eb) return !ea && eb;
  for (unsigned int k = 0; k < t.n; ++k) {
    unsigned int na = (na_all >> k) & 1, nb = (nb_all >> k) & 1;
    int c;
    if (na || nb) c = (int)nb - (int)na;
    else c = a[k] < b[k] ? -1 : (a[k] > b[k] ? 1 : 0);
    if (c == 0) continue;
    if (P.order[k].desc) c = -c;
    return c < 0;
  }
  return a[t.n] < b[t.n];
}

__device__ void cta_topn_compact(const TopBuf& t, unsigned int limit, unsigned int* s_cnt, unsigned int* s_have_thr, TopItem* s_thr, const DevPlan& P) {
  const unsigned int tid = threadIdx.x, nt = TILE;  // always called by exactly 256 threads
  unsigned short* idx = t.idx;
  unsigned int cnt = *s_cnt;
  unsigned int cap = 2;  // the sorting network covers the occupied prefix only (a nearly empty buffer costs next to nothing)
  while (cap < cnt) cap <<= 1;
  for (unsigned int i = cnt + tid; i < cap; i += nt) t.w[(size_t)idx[i] * t.stride + t.n + 1] = 0x80000000ull;  // free slots sort last
  cta256_sync();
  for (unsigned int k = 2; k <= cap; k <<= 1) {
    for (unsigned int j = k >> 1; j > 0; j >>= 1) {
      // a thread's compare-exchanges of one step touch disjoint pairs: issue the loads of four of them before the first
      // store (written as one loop the compiler has to assume the index stores alias the next pair's loads)
      for (unsigned int base = 0; base < cap / 2; base += 4 * nt) {
        unsigned int pi[4], px[4];
        unsigned short va[4], vb[4];
        bool sw[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const unsigned int p = base + tid + (unsigned int)u * nt;
          const unsigned int i = ((p & ~(j - 1)) << 1) | (p & (j - 1));
          pi[u] = i; px[u] = i | j;
          const bool on = p < cap / 2;
          va[u] = on ? idx[pi[u]] : (unsigned short)0; vb[u] = on ? idx[px[u]] : (unsigned short)0;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const bool on = base + tid + (unsigned int)u * nt < cap / 2;
          const bool up = (pi[u] & k) == 0;
          sw[u] = on && (up ? topbuf_less(t, vb[u], va[u], P) : topbuf_less(t, va[u], vb[u], P));
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (sw[u]) { idx[pi[u]] = vb[u]; idx[px[u]] = va[u]; }
      }
      cta256_sync();
    }
  }
  if (tid == 0) {
    unsigned int keep = cnt < limit ? cnt : limit;
    *s_cnt = keep;
    if (keep == limit && limit > 0) { *s_thr = topbuf_get(t, idx[limit - 1]); *s_have_thr = 1; }
  }
  cta256_sync();
}

// ---- TMA bulk staging of a tile's bytes into shared memory --------------------------------------------------------
// Each 256-entry tile's key bytes, value bytes and offset slices are contiguous in the block's heaps, so one elected
// thread moves them with four 1-D bulk copies (cp.async.bulk, completion on an mbarrier) while the CTA is still
// decoding the previous tile.  Threads then parse rows out of shared memory: HBM sees only full-line streaming
// reads instead of 32 scattered byte addresses per warp instruction.
// Stage capacities (key / value bytes) are chosen per launch from the block's average entry size (ScanArgs); a tile
// that does not fit is simply read from HBM.
enum { STAGE_LOOK = 8, STAGE_OFF_CAP = 1104, N_STAGES = 2, OBUF_COLS = 4, N_OBUF = 3, N_CNT = 4 };
enum { OBUF_BYTES = OBUF_COLS * TILE * 8, ONULL_WORDS = OBUF_COLS * (TILE / 32) };
// A chunk buffer (OBUF_BYTES) is laid out per tile: [4 columns][256 rows] in general, [8 columns][128 rows] when the tile
// selected at most 128 rows, so that such a tile needs one chunk for 8 output columns instead of two and the ring of
// N_OBUF buffers gives the scan warp twice the time to finish its look-back before the decode warps need the buffer back.
static_assert(OBUF_COLS == 4, "chunk layouts are 4 or 8 columns wide (shifts 2 / 3 below)");
__device__ __forceinline__ uint32_t obuf_cols(unsigned int total) { return total <= TILE / 2 ? 2u * OBUF_COLS : (uint32_t)OBUF_COLS; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!ok);
}
// same, for the service warps whose waits last a whole tile: let the hardware suspend the thread (time hint in ns)
// instead of burning issue slots on polls
__device__ __forceinline__ void mbar_wait_sleep(unsigned long long* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(20000u)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

struct TileMeta {
  uint32_t tile;            // tile index, >= n_tiles means "no more work"
  uint32_t staged;          // 1: entries [w_lo, w_hi) are resident in the stage
  uint32_t w_lo, w_hi;
  long long keys_adj, vals_adj;  // stage_ptr + adj + heap_offset = address of that heap byte in shared memory
  int koff_adj, voff_adj;        // stage_off_ptr[adj + entry] = offset of `entry`
};

// A tile's window of the block, resident in shared memory (all four pointers are shared-memory addresses, which the
// compiler can see: every access below compiles to LDS with 32-bit addressing).  Only entries [w_lo, w_hi) exist here.
struct SmemView {
  const uint8_t* skeys; const uint32_t* skoff; const uint8_t* svals; const uint32_t* svoff;
  const uint8_t* gvals;  // the block's value heap in HBM: svals + o and gvals + o hold the same byte
  static constexpr bool kWholeBlock = false;
  __device__ __forceinline__ const uint8_t* gval(const uint8_t* p) const { return gvals + (p - svals); }
  __device__ __forceinline__ const uint8_t* kptr(uint32_t i) const { return skeys + skoff[i]; }
  __device__ __forceinline__ uint32_t klen(uint32_t i) const { return skoff[i + 1] - skoff[i]; }
  __device__ __forceinline__ const uint8_t* vptr(uint32_t i) const { return svals + svoff[i]; }
  __device__ __forceinline__ uint32_t vlen(uint32_t i) const { return svoff[i + 1] - svoff[i]; }
};

// ---- per-entry front end: MVCC resolve -> row open/split -> predicate (or CRC in PM_CHECKSUM) ----------------------
struct EntryStats {  // per-thread partial statistics / checksum state
  unsigned long long keys, size, dflt, ck_x, ck_kvs, ck_bytes;
  unsigned int newer;
  unsigned int last;  // 1 + largest block entry index a row was returned for
  unsigned int warn;  // evaluation warnings (Division by 0)
};
enum { P1_NONE = 0, P1_LIVE = 1, P1_REDO = 2, P1_GENERAL = 3 /* entry_fast only: not a clean entry, run entry_phase1 */ };

// The thread sitting on the first version of a user key resolves that key.  P1_REDO: the shared-memory window was not
// enough (run longer than the look-ahead, or a long value in CF_DEFAULT) and nothing has been committed: the caller
// repeats the entry on the whole block.
template <int MODE, class V>
__device__ __forceinline__ int entry_phase1(const DevPlan& P, const ScanArgs& A, const V& view, uint32_t walk_hi, uint32_t e, Row& row, Cells& cells,
                                            EntryStats& ts, const unsigned long long* crc_tab, unsigned int lane, uint8_t* idx_buf) {
  bool start = (e == A.e_lo) || !same_user_key(view, e - 1, e);
  if (!start) return P1_NONE;
  RunOut ro;
  resolve_run(view, e, A.e_hi, walk_hi, A.read_ts, A.isolation, A.dflt, &ro);
  if (ro.truncated) return P1_REDO;
  ts.newer |= ro.met_newer;
  ts.dflt += ro.dflt_lookup;
  if (ro.err) { report_err(A.ctr, A.entry_base + e, ro.err); return P1_NONE; }
  if (!ro.found) return P1_NONE;
  const uint32_t kl = view.klen(e);
  const uint8_t* ek = view.kptr(e);
  ts.keys += 1;
  ts.size += (kl - 8) + ro.val_len;
  ts.last = e + 1;
  if (MODE == PM_CHECKSUM) {
    // checksum_crc64_xor (checksum.rs:105-114): CRC-64/XZ of old_prefix ‖ raw_key[len(new_prefix)..] ‖ value
    int rawlen = raw_key_len(ek, kl - 8);
    bool okp = rawlen >= 0 && (uint32_t)rawlen >= A.ck_new_prefix_len;
    for (uint32_t j = 0; okp && j < A.ck_new_prefix_len; ++j) okp = raw_at(ek, j) == A.ck_new_prefix[j];
    if (rawlen < 0) report_err(A.ctr, A.entry_base + e, DE_BAD_USER_KEY);
    else if (!okp) { atomicExch(&A.ctr->bad_prefix, 1u); report_err(A.ctr, A.entry_base + e, DE_BAD_RECORD_KEY); }
    else {
      // slicing-by-8: T[k][i] = CRC of byte i followed by k zero bytes (crc_tab[k * 256 + i]); eight independent lookups
      // consume eight message bytes, instead of eight dependent ones
      const unsigned long long* T = crc_tab;
      auto step1 = [&](unsigned long long c, uint32_t byte) { return T[((uint32_t)c ^ byte) & 0xffu] ^ (c >> 8); };
      auto step8 = [&](unsigned long long c, unsigned long long w) {
        c ^= w;
        const uint32_t lo = (uint32_t)c, hi = (uint32_t)(c >> 32);
        return T[7 * 256 + (lo & 0xffu)] ^ T[6 * 256 + ((lo >> 8) & 0xffu)] ^ T[5 * 256 + ((lo >> 16) & 0xffu)] ^ T[4 * 256 + (lo >> 24)] ^
               T[3 * 256 + (hi & 0xffu)] ^ T[2 * 256 + ((hi >> 8) & 0xffu)] ^ T[1 * 256 + ((hi >> 16) & 0xffu)] ^ T[hi >> 24];
      };
      unsigned long long c = A.ck_init_state;
      // raw key bytes [new_prefix_len, rawlen): raw byte j lives at enc[j + j / 8]; whole 8-byte groups are contiguous
      uint32_t j = A.ck_new_prefix_len;
      for (; j < (uint32_t)rawlen && (j & 7u); ++j) c = step1(c, raw_at(ek, j));
      for (; j + 8 <= (uint32_t)rawlen; j += 8) c = step8(c, ld64(ek + j + (j >> 3)));
      for (; j < (uint32_t)rawlen; ++j) c = step1(c, raw_at(ek, j));
      const uint8_t* vp = ro.val;
      const uint32_t vn = ro.val_len;
      uint32_t i = 0;
      for (; i + 8 <= vn; i += 8) c = step8(c, ld64(vp + i));
      if (i < vn) {
        unsigned long long w = ld64(vp + i);
        for (; i < vn; ++i) { c = step1(c, (uint32_t)w & 0xffu); w >>= 8; }
      }
      ts.ck_x ^= ~c;
      ts.ck_kvs += 1;
      ts.ck_bytes += (unsigned long long)rawlen + ro.val_len + A.ck_old_prefix_len - A.ck_new_prefix_len;
    }
    return P1_NONE;
  }
  row.enc_key = ek;
  row.enc_key_len = kl - 8;
  row.commit_ts = ro.commit_ts;
  row.imms = A.imms;
  int err;
#ifndef B2_NO_IDX
  if (P.idx_cols > 0) err = index_row_split(P, row, cells, ro.val, ro.val_len, idx_buf);  // BatchIndexScan: the columns are the key's datums
  else
#endif
  {
    err = row_open(ro.val, ro.val_len, &row.rv);
    if (P.n_raw || P.expr_refs) row.gv = ro.dflt_lookup ? ro.val : view.gval(ro.val);  // (a CF_DEFAULT value is always read in place)
    if (!err) err = row_split(P, row, cells);
  }
  bool keep = false;
  if (!err) err = eval_conds(P, row, cells, &keep);
  if (err) { report_err(A.ctr, A.entry_base + e, err); return P1_NONE; }
  ts.warn += row.warn; row.warn = 0;
  return keep ? P1_LIVE : P1_NONE;
}

// Clean-entry front end (b2_device.h: fast_key_tail / fast_write_head / fast_row_v2) for one warp's 32 entries of a
// staged tile.  Every lane calls it (the predecessor's key words travel by shuffle; lane 0 reads its predecessor
// itself); `valid` says whether the lane holds an entry of the chunk.  P1_GENERAL from any lane sends the whole warp
// through entry_phase1 instead: nothing has been counted or reported by then.
template <int MODE>
__device__ __forceinline__ int entry_fast(const DevPlan& P, const ScanArgs& A, const SmemView& view, uint32_t e, bool valid, Row& row, Cells& cells,
                                          EntryStats& ts, unsigned int lane) {
  const uint32_t ko = view.skoff[e], kl = view.skoff[e + 1] - ko;
  const uint8_t* kp = view.skeys + ko;
  KeyTail t;
  t.a = t.b = t.c = 0;
  bool ok = fast_key_tail(kp, kl, &t);
  unsigned long long pa = __shfl_up_sync(0xffffffffu, (unsigned long long)t.a, 1), pb = __shfl_up_sync(0xffffffffu, (unsigned long long)t.b, 1);
  bool pok = __shfl_up_sync(0xffffffffu, (int)ok, 1) != 0;
  const bool first = e == A.e_lo;  // the range starts here: a run start whatever lies before it
  if (lane == 0 && !first) {
    KeyTail q;
    q.a = q.b = q.c = 0;
    pok = fast_key_tail(view.kptr(e - 1), view.klen(e - 1), &q);
    pa = q.a; pb = q.b;
  }
  if (!valid) return P1_NONE;
  if (!ok || (!first && !pok)) return P1_GENERAL;
  if (!first && key_tail_same(t.a, t.b, pa, pb)) return P1_NONE;  // an older version of the lane below's key
  const uint64_t cts = key_tail_commit_ts(t);
  if (cts > A.read_ts) return P1_GENERAL;  // newer than the snapshot: the general walk steps through the versions
  const uint32_t vo = view.svoff[e], vl = view.svoff[e + 1] - vo;
  const uint8_t* vp = view.svals + vo;
  uint32_t roff, rlen;
  if (!fast_write_head(vp, vl, &roff, &rlen)) return P1_GENERAL;
  row.enc_key = kp; row.enc_key_len = 27; row.commit_ts = cts; row.imms = A.imms;
  if (!fast_row_v2(P, vp + roff, rlen, row)) return P1_GENERAL;
  row.filled = P.fast_filled;
  if (P.n_raw || P.expr_refs) row.gv = view.gval(vp + roff);
  bool keep = false;
  if (eval_conds(P, row, cells, &keep)) return P1_GENERAL;  // evaluation errors are raised by the general path
  ts.keys += 1;
  ts.size += 27u + rlen;
  ts.last = e + 1;
  ts.warn += row.warn; row.warn = 0;
  return keep ? P1_LIVE : P1_NONE;
}

// ---- the fused scan kernel -------------------------------------------------------------------------------
struct SmemTable {  // per-CTA group table (dynamic shared memory): keys | acc.  A slot is free while its key is SMEM_EMPTY_KEY
  unsigned long long* keys;
  unsigned long long* acc;
  unsigned int slots;
};
// (a group whose key happens to be this value simply lives in the HBM table only)
#define SMEM_EMPTY_KEY 0xffffffffffffffffull

// The whole kernel as a device function: instantiated by the generic __global__ wrapper (plan in a __grid_constant__
// parameter) and by the per-plan JIT translation unit (plan as a compile-time constant, jit.cpp).
template <int MODE>
__device__ __forceinline__ void scan_body(const DevPlan& P, const ScanArgs& A) {
  // PM_PROJ is PM_SCAN with expression-valued output cells: a separate instantiation, so that the expression evaluator
  // stays out of the plain scan's hot loop (inlined there it cost 3.5x)
  constexpr bool IS_SCAN = (MODE == PM_SCAN) || (MODE == PM_PROJ);
  constexpr bool IS_AGG = (MODE == PM_AGG) || (MODE == PM_AGGM);  // PM_AGGM: composite group key, no CTA table
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  __shared__ unsigned int s_warp_cnt[2][TILE / 32];  // by tile parity: a fast warp may start the next tile while others still read
  __shared__ unsigned int s_tbl_used, s_tbl_miss, s_tbl_off;  // resident groups; rows that fell through to HBM; table given up

  const unsigned int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // list mode (order-free pipelines): the entries the lean kernel handed over, 256 per tile, read from the HBM arrays
  const uint32_t n_list = !IS_SCAN && A.list_mode ? *(volatile unsigned int*)A.slow_count : 0u;
  const uint32_t n_tiles = !IS_SCAN && A.list_mode ? (n_list + TILE - 1) / TILE : (A.c_hi - A.c_lo + TILE - 1) / TILE;
  const unsigned long long out_base = IS_SCAN ? A.ctr->out_base : 0ull;  // stable during this launch
  if (!IS_SCAN && A.list_mode && n_list == 0) {  // the lean kernel handed nothing over (the usual case on clean data)
    if (MODE == PM_TOPN && tid == 0) A.topn.counts[blockIdx.x] = 0;
    return;
  }

  SmemTable st;
  st.slots = 0;
  if (MODE == PM_AGG && P.has_group && A.smem_slots) {
    st.slots = A.smem_slots;
    st.keys = reinterpret_cast<unsigned long long*>(dyn_smem);
    st.acc = st.keys + st.slots;
    for (unsigned int i = tid; i < st.slots; i += TILE) st.keys[i] = SMEM_EMPTY_KEY;
    for (unsigned int i = tid; i < st.slots * P.acc_words; i += TILE) st.acc[i] = 0;
    if (tid == 0) { s_tbl_used = 0; s_tbl_miss = 0; s_tbl_off = 0; }
    __syncthreads();
  }

  // PM_TOPN: per-CTA candidate buffer (dynamic shared memory) + current threshold
  __shared__ unsigned int s_top_cnt, s_top_have_thr;
  __shared__ TopItem s_top_thr;
  const TopBuf tb = topbuf_make(dyn_smem, MODE == PM_TOPN ? A.topn_cap : 0u, P);
  if (MODE == PM_TOPN) {
    if (tid == 0) {
      s_top_cnt = 0; s_top_have_thr = 0;
      if (A.topn_seed && A.limit > 0 && *A.topn_seed_cnt >= (unsigned int)A.limit) { s_top_thr = A.topn_seed[A.limit - 1]; s_top_have_thr = 1; }
    }
    for (unsigned int i = tid; i < A.topn_cap; i += blockDim.x) tb.idx[i] = (unsigned short)i;
    __syncthreads();
  }

  // PM_CHECKSUM: CRC-64/XZ slicing-by-8 tables (8 x 256 x u64 = 16 KB)
  unsigned long long* crc_tab = reinterpret_cast<unsigned long long*>(dyn_smem);
  if (MODE == PM_CHECKSUM) {
    // slicing-by-8 tables of CRC-64/XZ (reflected): T[0] is the byte table, T[k][i] = T[0][T[k-1][i] & 0xff] ^ (T[k-1][i] >> 8)
    for (unsigned int i = tid; i < 256; i += blockDim.x) crc_tab[i] = crc64_table_entry(i);
    __syncthreads();
    for (unsigned int i = tid; i < 256; i += blockDim.x) {
      unsigned long long t = crc_tab[i];
      for (int kk = 1; kk < 8; ++kk) { t = crc_tab[(uint32_t)t & 0xffu] ^ (t >> 8); crc_tab[kk * 256 + i] = t; }
    }
    __syncthreads();
  }

  // per-thread statistics, reduced once at the end
  EntryStats ts;
  ts.keys = ts.size = ts.dflt = ts.ck_x = ts.ck_kvs = ts.ck_bytes = 0; ts.newer = 0; ts.last = 0; ts.warn = 0;
  unsigned long long t_live = 0;
  unsigned int t_first = 0xffffffffu;  // smallest block entry index a row was returned for
  // no-group aggregation: one accumulator set per CTA in shared memory, flushed at the end
  __shared__ __align__(16) unsigned long long s_simple_acc[MODE == PM_AGG ? MAX_ACC_WORDS : 1];  // (FIRST: 16-byte pairs)
  if (MODE == PM_AGG) {
    for (unsigned int i = tid; i < MAX_ACC_WORDS; i += blockDim.x) s_simple_acc[i] = 0;
  }

  // ---- tile pipeline --------------------------------------------------------------------------------------------
  // Warp 8 is the producer: it claims tiles, reads the four offsets that bound a tile's bytes and issues the bulk
  // copies, running up to N_STAGES tiles ahead.  Warps 0-7 decode.  full[s]: producer -> consumers (bytes landed, meta
  // published); empty[s]: consumers -> producer (stage may be refilled).
  __shared__ __align__(8) unsigned long long s_full[N_STAGES];
  __shared__ __align__(8) unsigned long long s_empty[N_STAGES];
  __shared__ TileMeta s_meta[N_STAGES];
  // PM_SCAN: consumers -> scan warp.  cnt_ready[k % N_CNT]: tile k's row count (and tile index) posted;
  // obuf_full / obuf_empty[q]: output chunk buffer q handed to the scan warp / drained to HBM
  __shared__ __align__(8) unsigned long long s_cnt_ready[N_CNT], s_obuf_full[N_OBUF], s_obuf_empty[N_OBUF];
  __shared__ unsigned int s_total[N_CNT], s_tile_of[N_CNT];
  __shared__ unsigned int s_redo[4];  // per tile (mod 4): some thread could not resolve its row inside the shared-memory window
  unsigned char* stage_base = dyn_smem + A.stage_off;
  const uint32_t STAGE_KEY_CAP = A.stage_key_cap, STAGE_VAL_CAP = A.stage_val_cap;
  const uint32_t STAGE_BYTES = STAGE_KEY_CAP + STAGE_VAL_CAP + 2 * STAGE_OFF_CAP;
  // PM_SCAN output chunk buffers (dynamic shared memory): N_OBUF x [OBUF_COLS][TILE] values, then the NULL masks
  unsigned long long* obuf_base = reinterpret_cast<unsigned long long*>(dyn_smem + A.out_stage_off);
  unsigned int* onull_base = reinterpret_cast<unsigned int*>(dyn_smem + A.out_stage_off + N_OBUF * OBUF_BYTES);
  if (IS_SCAN)
    for (unsigned int i = tid; i < N_OBUF * ONULL_WORDS; i += blockDim.x) onull_base[i] = 0;
  if (tid == 0) {
    for (int i = 0; i < N_STAGES; ++i) { mbar_init(&s_full[i], 1); mbar_init(&s_empty[i], TILE / 32); }
    for (int i = 0; i < N_CNT; ++i) mbar_init(&s_cnt_ready[i], 1);
    for (int i = 0; i < 4; ++i) s_redo[i] = 0;
    for (int i = 0; i < N_OBUF; ++i) { mbar_init(&s_obuf_full[i], TILE / 32); mbar_init(&s_obuf_empty[i], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();  // last CTA-wide barrier: from here on the two roles only meet through the mbarriers

  if (wid == TILE / 32) {
    if (lane == 0) {
      // software-pipelined by one tile: the ticket and the four bounding offsets of tile k+1 are fetched while the
      // producer would otherwise idle on empty[slot]; only the bulk copies themselves wait for the stage
      uint32_t nx_tile, nx_wlo = 0, nx_whi = 0, nx_k0 = 0, nx_k1 = 0, nx_v0 = 0, nx_v1 = 0;
      auto claim = [&](uint32_t k) {
        // PM_SCAN claims tiles in order so that the decoupled look-back only ever waits on running CTAs
        if (IS_SCAN) nx_tile = (uint32_t)atomicAdd(&A.tile_status[n_tiles], 1ull);
        else nx_tile = blockIdx.x + k * gridDim.x;
        if (nx_tile < n_tiles && A.staging) {
          uint32_t e0 = A.c_lo + nx_tile * TILE;
          uint32_t e1 = e0 + TILE < A.c_hi ? e0 + TILE : A.c_hi;
          nx_wlo = e0 > A.e_lo ? e0 - 1 : e0;
          nx_whi = e1 + STAGE_LOOK < A.e_hi ? e1 + STAGE_LOOK : A.e_hi;
          nx_k0 = A.blk.koff[nx_wlo]; nx_k1 = A.blk.koff[nx_whi]; nx_v0 = A.blk.voff[nx_wlo]; nx_v1 = A.blk.voff[nx_whi];
        }
      };
      // (ordered mode claims late instead: a ticket held early would stall every successor's look-back)
      if (!IS_SCAN) claim(0);
      for (uint32_t k = 0;; ++k) {
        const int slot = (int)(k % N_STAGES);
        TileMeta m;
        m.staged = 0; m.w_lo = 0; m.w_hi = 0; m.keys_adj = 0; m.vals_adj = 0; m.koff_adj = 0; m.voff_adj = 0;
        if (IS_SCAN) { mbar_wait_sleep(&s_empty[slot], ((k / N_STAGES) & 1) ^ 1); claim(k); }
        m.tile = nx_tile;
        const uint32_t w_lo = nx_wlo, w_hi = nx_whi, k0 = nx_k0, k1 = nx_k1, v0 = nx_v0, v1 = nx_v1;
        if (!IS_SCAN) mbar_wait_sleep(&s_empty[slot], ((k / N_STAGES) & 1) ^ 1);
        uint32_t tx = 0;
        if (m.tile < n_tiles && A.staging) {
          unsigned long long ka = (unsigned long long)(A.blk.keys + k0), va = (unsigned long long)(A.blk.vals + v0);
          unsigned long long oa = (unsigned long long)(A.blk.koff + w_lo), ob = (unsigned long long)(A.blk.voff + w_lo);
          uint32_t kpad = (uint32_t)(ka & 15), vpad = (uint32_t)(va & 15), opad = (uint32_t)(oa & 15), qpad = (uint32_t)(ob & 15);
          uint32_t kbytes = (kpad + (k1 - k0) + 15) & ~15u, vbytes = (vpad + (v1 - v0) + 15) & ~15u;
          uint32_t obytes = (opad + (w_hi - w_lo + 1) * 4 + 15) & ~15u, qbytes = (qpad + (w_hi - w_lo + 1) * 4 + 15) & ~15u;
          if (kbytes + 16 <= STAGE_KEY_CAP && vbytes + 16 <= STAGE_VAL_CAP && obytes <= STAGE_OFF_CAP && qbytes <= STAGE_OFF_CAP) {
            m.staged = 1; m.w_lo = w_lo; m.w_hi = w_hi;
            m.keys_adj = (long long)kpad - (long long)k0; m.vals_adj = (long long)vpad - (long long)v0;
            m.koff_adj = (int)(opad / 4) - (int)w_lo; m.voff_adj = (int)(qpad / 4) - (int)w_lo;
            s_meta[slot] = m;
            unsigned char* st = stage_base + (size_t)slot * STAGE_BYTES;
            tx = kbytes + vbytes + obytes + qbytes;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // consumers' generic reads of this stage vs. the async writes
            mbar_expect_tx(&s_full[slot], tx);
            bulk_g2s(st, (const void*)(ka - kpad), kbytes, &s_full[slot]);
            bulk_g2s(st + STAGE_KEY_CAP, (const void*)(va - vpad), vbytes, &s_full[slot]);
            bulk_g2s(st + STAGE_KEY_CAP + STAGE_VAL_CAP, (const void*)(oa - opad), obytes, &s_full[slot]);
            bulk_g2s(st + STAGE_KEY_CAP + STAGE_VAL_CAP + STAGE_OFF_CAP, (const void*)(ob - qpad), qbytes, &s_full[slot]);
          }
        }
        if (!tx) {
          s_meta[slot] = m;
          asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&s_full[slot])) : "memory");
        }
        if (m.tile >= n_tiles) break;
        if (!IS_SCAN) claim(k + 1);
      }
    }
    return;
  }

  if (wid == TILE / 32 + 1) {
    // ---- scan warp (PM_SCAN): turns each tile's row count into its global output base (decoupled look-back, one
    // warp wide: lane l inspects tile (j - l); the nearest tile that already knows its inclusive prefix ends the walk,
    // the aggregates in between are summed with shuffles), then drains the tile's output chunks from shared memory to
    // HBM.  The decoding warps never wait for the look-back.
    if (!IS_SCAN) return;
    const unsigned long long F_AGG = 1ull << 62, F_INC = 2ull << 62, VMASK = (1ull << 62) - 1;
    uint32_t sw_q = 0, sw_phase = 0;
    for (uint32_t k = 0;; ++k) {
      mbar_wait_sleep(&s_cnt_ready[k % N_CNT], (k / N_CNT) & 1);
      const uint32_t tile = s_tile_of[k % N_CNT];
      if (tile >= n_tiles) break;
      const unsigned long long total = s_total[k % N_CNT];
      unsigned long long excl = 0;
      // (the tile's own aggregate was published by the decode warps the moment they knew it)
      if (tile != 0) {
        long long j = (long long)tile - 1;
        for (;;) {
          long long idx = j - (long long)lane;
          unsigned long long sres = idx >= 0 ? ld_volatile_u64(&A.tile_status[idx]) : F_INC;  // before tile 0: prefix 0
          unsigned int flag = (unsigned int)(sres >> 62);
          unsigned int m_inc = __ballot_sync(0xffffffffu, flag == 2), m_zero = __ballot_sync(0xffffffffu, flag == 0);
          unsigned int upto = m_inc ? (__ffs(m_inc) - 1) : 31;             // lanes 0..upto matter
          unsigned int need = upto == 31 ? 0xffffffffu : ((2u << upto) - 1);
          if (m_zero & need) continue;                                       // a needed predecessor has not published yet
          unsigned long long v = (lane <= upto) ? (sres & VMASK) : 0ull;
          for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
          excl += v;
          if (m_inc) break;
          j -= 32;
        }
        if (lane == 0) atomicExch(&A.tile_status[tile], F_INC | (excl + total));
      }
      if (lane == 0 && total) atomicAdd(&A.ctr->out_rows, total);
      const unsigned long long base = out_base + excl;
      const unsigned int lim = base + total <= A.out_cap ? (unsigned int)total : (base < A.out_cap ? (unsigned int)(A.out_cap - base) : 0u);
      const uint32_t cpc = obuf_cols((unsigned int)total), cshift = cpc == OBUF_COLS ? 2u : 3u, rstride = (OBUF_COLS * TILE) >> cshift;
      const uint32_t n_rounds = P.n_out > 0 ? ((uint32_t)P.n_out + cpc - 1) >> cshift : 1u;
      for (uint32_t r = 0; r < n_rounds; ++r) {
        const uint32_t q = sw_q;
        mbar_wait_sleep(&s_obuf_full[q], sw_phase);
        if (++sw_q == N_OBUF) { sw_q = 0; sw_phase ^= 1; }
        const int c0 = (int)(r * cpc);
        const int nc = P.n_out - c0 < (int)cpc ? P.n_out - c0 : (int)cpc;
        const unsigned long long* ob = obuf_base + (size_t)q * (OBUF_COLS * TILE);
        unsigned long long* dst = A.out_data + (size_t)c0 * A.out_cap + base;
        for (unsigned int i = lane; i < lim; i += 32) {
#pragma unroll
          for (int c = 0; c < 2 * OBUF_COLS; ++c)
            if (c < nc) dst[(size_t)c * A.out_cap + i] = ob[c * rstride + i];
        }
        // NULL cells are rare: the bitmap is pre-filled with ones and only cleared where needed
        unsigned int* on = onull_base + q * ONULL_WORDS;
        unsigned int w = on[lane];  // ONULL_WORDS == 32: word (column c, rows 32 j ..) at [c * (rstride / 32) + j]
        if (w) {
          on[lane] = 0;
          const int c = (int)(lane >> (5 - cshift));  // rstride / 32 words per column: 8 (4 columns) or 4 (8 columns)
          while (w) {
            unsigned int bit = __ffs(w) - 1;
            w &= w - 1;
            unsigned long long row_at = base + (lane & ((rstride >> 5) - 1)) * 32 + bit;
            if (row_at < A.out_cap) atomicAnd(&A.out_bitmap[(size_t)(c0 + c) * (A.out_cap / 64) + (row_at >> 6)], ~(1ull << (row_at & 63)));
          }
        }
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&s_obuf_empty[q])) : "memory");
      }
    }
    return;
  }

  // One tile, front end to back end, over a view of the block.  Instantiated twice: on the shared-memory window (hot:
  // every byte access is an LDS) and on the HBM arrays (tiles that did not fit the stage, or that hold a row the window
  // cannot resolve: a version run longer than the look-ahead, a long value in CF_DEFAULT).  Returns true when the
  // shared-memory attempt must be repeated on the whole block; nothing has been committed in that case.
  uint32_t ob_q = 0, ob_phase = 0;  // PM_SCAN: next output chunk buffer and how often the ring has wrapped (parity)
  auto tile_body = [&](const auto& view, const uint32_t walk_hi, const uint32_t k, const uint32_t tile) __attribute__((always_inline)) -> bool {
    using V = typename b2_remove_cvref<decltype(view)>::type;
    const uint32_t e = !IS_SCAN && A.list_mode ? (tile * TILE + tid < n_list ? A.slow_list[tile * TILE + tid] : A.c_hi) : A.c_lo + tile * TILE + tid;
    bool live = false;
    Row row;
    Cells cells;
#ifndef B2_NO_IDX
    uint8_t idx_buf[IDX_RAW_MAX];  // BatchIndexScan: the row's raw key bytes after the index id (unused, and optimised away, otherwise)
#else
    uint8_t* idx_buf = nullptr;    // (a kernel specialised for a table scan carries none of the index-row decoder)
#endif
    EntryStats d;
    d.keys = d.size = d.dflt = d.ck_x = d.ck_kvs = d.ck_bytes = 0; d.newer = 0; d.last = 0; d.warn = 0;
    int r1 = P1_NONE;
    bool general = true;
    if constexpr (!V::kWholeBlock && MODE != PM_CHECKSUM) {
      // clean entries take the word-wise front end; one odd entry sends its warp through the general one
      if (A.fast_ok && P.fast_n > 0) {
        const bool valid = e < A.c_hi;
        r1 = entry_fast<MODE>(P, A, view, valid ? e : A.c_hi - 1, valid, row, cells, d, lane);
        general = __any_sync(0xffffffffu, r1 == P1_GENERAL);
        if (general) { d.keys = d.size = 0; d.last = 0; d.warn = 0; }
      }
    }
    if (general) r1 = e < A.c_hi ? entry_phase1<MODE>(P, A, view, walk_hi, e, row, cells, d, crc_tab, lane, idx_buf) : (int)P1_NONE;
    live = r1 == P1_LIVE;
    if (!V::kWholeBlock) {
      if (__any_sync(0xffffffffu, r1 == P1_REDO) && lane == 0) s_redo[k & 3] = 1;
    }
    unsigned int warp_off = 0, total = 0, lane_off = 0;
    if (IS_SCAN) {
      // ---- ordered compaction: ballot/popc inside the warp, smem across warps, look-back across tiles ----
      unsigned int bal = __ballot_sync(0xffffffffu, live);
      lane_off = __popc(bal & ((1u << lane) - 1));
      if (lane == 0) s_warp_cnt[k & 1][wid] = __popc(bal);
      cta256_sync();
    } else if (!V::kWholeBlock) {
      cta256_sync();  // the vote below
    }
    if (!V::kWholeBlock) {
      if (s_redo[k & 3]) return true;
    }
    // ---- commit ----
    ts.keys += d.keys; ts.size += d.size; ts.dflt += d.dflt; ts.newer |= d.newer; ts.warn += d.warn;
    if (d.last > ts.last) ts.last = d.last;
    if (d.last && d.last - 1 < t_first) t_first = d.last - 1;
    if (MODE == PM_CHECKSUM) { ts.ck_x ^= d.ck_x; ts.ck_kvs += d.ck_kvs; ts.ck_bytes += d.ck_bytes; }
    t_live += live;

    if (IS_SCAN) {
#pragma unroll
      for (int w = 0; w < TILE / 32; ++w) {
        unsigned int c = s_warp_cnt[k & 1][w];
        if (w < (int)wid) warp_off += c;
        total += c;
      }
      // Selected rows go to shared memory at their tile-local compacted position, OBUF_COLS columns per chunk; the
      // scan warp (warp 9) turns the tile's row count into its global output base and drains the chunks to HBM as
      // contiguous 8-byte runs, so the look-back latency never stalls the decode.
      const unsigned int pos = warp_off + lane_off;
      // publish the tile's row count for the look-backs of later tiles right away (flag AGGREGATE; tile 0: INCLUSIVE):
      // the scan warp may be several tiles behind, other CTAs must not wait for it to get here
      if (tid == 0) atomicExch(&A.tile_status[tile], ((tile == 0 ? 2ull : 1ull) << 62) | total);
      const bool fast = live && row.fast;
      const uint32_t cpc = obuf_cols(total), cshift = cpc == OBUF_COLS ? 2u : 3u, rstride = (OBUF_COLS * TILE) >> cshift;  // columns per chunk (4 or 8), row stride
      const uint32_t n_rounds = P.n_out > 0 ? ((uint32_t)P.n_out + cpc - 1) >> cshift : 1u;
      for (uint32_t r = 0; r < n_rounds; ++r) {
        const uint32_t q = ob_q;  // next buffer of the ring, its use count parity in ob_phase
        mbar_wait(&s_obuf_empty[q], ob_phase ^ 1);  // chunk buffer drained (N_OBUF chunks ago)
        if (++ob_q == N_OBUF) { ob_q = 0; ob_phase ^= 1; }
        if (r == 0) {
          // (posted after the wait: at most N_OBUF <= N_CNT - 1 tiles are ever pending at the scan warp)
          if (tid == 0) { s_total[k % N_CNT] = total; s_tile_of[k % N_CNT] = tile; asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&s_cnt_ready[k % N_CNT])) : "memory"); }
        }
        if (live) {
          unsigned long long* ob = obuf_base + (size_t)q * (OBUF_COLS * TILE) + pos;
          auto put = [&](int oc) {  // general cell: any role / kind, may be NULL
            Value v;
            int err = MODE == PM_PROJ ? eval_expr(P, P.proj[P.out_cols[oc]], row, cells, &v, nullptr) : cell_value(P, row, cells, P.out_cols[oc], &v);
            if (err) { report_err(A.ctr, A.entry_base + e, err); v.null = true; }
            ob[((uint32_t)oc & (cpc - 1)) * rstride] = v.null ? 0ull : v.bits;
            if (v.null) atomicOr(&onull_base[q * ONULL_WORDS + ((uint32_t)oc & (cpc - 1)) * (rstride / 32) + (pos >> 5)], 1u << (pos & 31));
          };
          if (fast) {
            if ((!P.fast_v1 || row.fast == 1) && fast_all8(P, row)) {
              // every stored column is 8 bytes wide: the cells this chunk needs come out of one run of aligned words
              uint32_t need = 0;
#pragma unroll
              for (int h = 0; h < 8; ++h)
                if (h < P.fast_n && P.fast_out[h] >= 0 && ((uint32_t)P.fast_out[h] >> cshift) == r) need |= 1u << h;
              uint64_t cv[8];
              fast_cells8(row, need, cv);
#pragma unroll
              for (int h = 0; h < 8; ++h)
                if ((need >> h) & 1u) ob[((uint32_t)P.fast_out[h] & (cpc - 1)) * rstride] = cv[h];
            } else if (!P.fast_v1 || row.fast == 1) {
              // exact-layout v2 row: the (at most 8) stored integer columns are decoded by stored position, so every
              // shift is a compile-time constant; the value goes from the staged row bytes to the chunk buffer in one step
              uint32_t prev = 0;
#pragma unroll
              for (int h = 0; h < 8; ++h) {
                if (h < P.fast_n) {
                  const uint32_t end = fast_end(row, h);
                  const int oc = P.fast_out[h];
                  if (oc >= 0 && ((uint32_t)oc >> cshift) == r) ob[((uint32_t)oc & (cpc - 1)) * rstride] = fast_int_cell(row, prev, end, (P.fast_uns >> h) & 1u);
                  prev = end;
                }
              }
            } else {
              // exact-layout v1 row: same positions, datums decoded by flag (one rolled loop: the varint reader is big)
#pragma unroll 1
              for (int h = 0; h < P.fast_n; ++h) {
                const int oc = P.fast_out[h];
                if (oc >= 0 && ((uint32_t)oc >> cshift) == r) ob[((uint32_t)oc & (cpc - 1)) * rstride] = fast_cell_dyn(row, (uint32_t)h, false, true);
              }
            }
            for (int j = 0; j < P.n_out_slow; ++j)  // handle / Real / repeated columns of such a row
              if (((uint32_t)P.out_slow[j] >> cshift) == r) put(P.out_slow[j]);
          } else {
            const int c_end = (int)((r + 1) * cpc) < P.n_out ? (int)((r + 1) * cpc) : P.n_out;
            for (int oc = (int)(r * cpc); oc < c_end; ++oc) put(oc);
          }
        }
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&s_obuf_full[q])) : "memory");
      }
    } else if (MODE == PM_TOPN) {
      // BatchTopN: keep the `limit` smallest rows under the order-by key.  A row is a candidate only if it beats
      // the CTA's current threshold (the limit-th best seen so far); candidates are sorted when the buffer fills.
      if (live) {
        TopItem it;
        int err = make_item(P, row, cells, A.desc ? ~(A.entry_base + e) : A.entry_base + e, &it);  // (ties go to the row scanned first)
        if (err) report_err(A.ctr, A.entry_base + e, err);
        else if (!s_top_have_thr || item_less(it, s_top_thr, P)) {
          unsigned int pos = atomicAdd(&s_top_cnt, 1u);
          topbuf_put(tb, tb.idx[pos], it);  // pos < topn_cap: the buffer is compacted whenever fewer than TILE slots remain
        }
      }
      cta256_sync();
      if (s_top_cnt + TILE > A.topn_cap) cta_topn_compact(tb, (unsigned int)A.limit, &s_top_cnt, &s_top_have_thr, &s_top_thr, P);
    } else if (IS_AGG) {
      // BatchSimpleAggregation / BatchFastHashAggregation / BatchSlowHashAggregation (PM_AGGM).  Rows of one warp that share a group key are combined with
      // warp reductions first (match.any + redux); the group's leader lane then issues one atomic per accumulator
      // word, into the CTA's shared-memory table when the key is resident there, else into the HBM table.
      Value gk;
      gk.bits = 0; gk.null = false;
      bool ok = live;
      uint64_t gw[MAX_GROUP + 1];  // PM_AGGM: the composite key (value words, then the NULL mask); gk.bits = its hash tag
      if (MODE == PM_AGGM) {
        // slow_hash_aggr_executor.rs:209-239: groups are distinguished by the encoded sort key of every group-by value,
        // i.e. by value bits and NULL-ness per column (0.0 and -0.0 are different groups here, unlike the fast executor)
        uint64_t tag = 0x9e3779b97f4a7c15ull, nm = 0;
#pragma unroll
        for (int q = 0; q < MAX_GROUP; ++q) {
          gw[q] = 0;
          if (q < P.n_group && ok) {
            Value v;
            int err = eval_expr(P, P.groups[q], row, cells, &v, nullptr);
            if (err) { report_err(A.ctr, A.entry_base + e, err); ok = false; }
            else { gw[q] = v.null ? 0ull : v.bits; nm |= v.null ? (1ull << q) : 0ull; tag = mix64(tag ^ gw[q]); }
          }
        }
#pragma unroll
        for (int q = MAX_GROUP; q > 0; --q)
          if (q == P.n_group) { gw[q] = nm; }
        tag = mix64(tag + nm);
        if (A.tbl.hash_mask_bits) tag &= (1ull << A.tbl.hash_mask_bits) - 1;
        if (tag == AGG_EMPTY_KEY) tag = 0;
        gk.bits = tag;
      } else if (live && P.has_group) {
        int err = eval_expr(P, P.group, row, cells, &gk, nullptr);  // calc_groups_each_row
        if (err) { report_err(A.ctr, A.entry_base + e, err); ok = false; }
        else if (gk.null) gk.bits = 0;
        else if (P.group_et == 1 && bits_f64(gk.bits) == 0.0) gk.bits = 0;  // -0.0 and 0.0 are one group
      }
      const unsigned int active = __ballot_sync(0xffffffffu, ok);
      if (ok) {
        unsigned int peers = active;
        // A redux / shuffle over `peers` is replayed once per distinct mask in the warp, so pre-aggregating a warp that
        // holds many groups costs more than it saves: past a few groups every lane commits its own row instead.
        if (MODE == PM_AGGM) {
          peers = __match_any_sync(active, gk.bits);
          const int lead = __ffs(peers) - 1;
          if (__popc(__ballot_sync(active, lead == (int)lane)) > 28) peers = 1u << lane;  // (nearly) one group per lane
          else {
            // every lane of `peers` takes part in every shuffle: a `same && __shfl_sync(..)` would skip the shuffles of a
            // lane that already differs, and its warp-mates would wait for it (equal tags, different keys)
            bool same = true;
#pragma unroll
            for (int q = 0; q <= MAX_GROUP; ++q)
              if (q <= P.n_group) {
                const uint64_t lw = __shfl_sync(peers, gw[q], lead);
                same = same && lw == gw[q];
              }
            if (__any_sync(active, !same)) peers = 1u << lane;  // equal tags, different keys inside the warp: no pre-aggregation
          }
        } else if (P.has_group) {
          const unsigned int nm = __ballot_sync(active, gk.null);
          peers = __match_any_sync(active, gk.bits) & (gk.null ? nm : ~nm);
          if (__popc(__ballot_sync(active, (unsigned int)(__ffs(peers) - 1) == lane)) > 4) peers = 1u << lane;
        }
        bool real_sum = false;  // (folds to a constant in a specialised kernel)
        for (int a = 0; a < P.n_aggs; ++a) real_sum |= (P.aggs[a].kind == 1 || P.aggs[a].kind == 2) && P.aggs[a].arg_et == 1;
        if (real_sum) peers = 1u << lane;
        const bool leader = (unsigned int)(__ffs(peers) - 1) == lane;
        const bool solo = (peers & (peers - 1)) == 0;
        unsigned long long* acc = nullptr;
        // (all lanes of `active` take part, so that none of them waits at another warp-synchronous instruction meanwhile)
        const unsigned int mslot = MODE == PM_AGGM ? table_find_or_insert_multi(A.tbl, A.ctr, active, leader, gk.bits, gw, P.n_group + 1) : 0xffffffffu;
        if (leader) {
          if (MODE == PM_AGGM) {
            if (mslot != 0xffffffffu) acc = A.tbl.acc + (size_t)mslot * P.acc_words;
          } else if (!P.has_group) acc = s_simple_acc;
          else {
            if (st.slots && !s_tbl_off && !gk.null && gk.bits != SMEM_EMPTY_KEY) {
              // open addressing on the key words themselves: claim a free slot with one 64-bit CAS; accumulators start
              // at zero and are only ever added to, so there is no "being initialised" state to wait for
              const unsigned int mask = st.slots - 1, limit = (st.slots >> 1) + (st.slots >> 2);
              unsigned int s = (unsigned int)(mix64(gk.bits) >> 20) & mask;
              for (int probes = 0; probes < 8; ++probes) {
                unsigned long long kk = *(volatile unsigned long long*)&st.keys[s];
                if (kk == SMEM_EMPTY_KEY) {
                  if (*(volatile unsigned int*)&s_tbl_used >= limit) break;  // table is at its load limit: go to HBM
                  kk = atomicCAS(&st.keys[s], SMEM_EMPTY_KEY, gk.bits);
                  if (kk == SMEM_EMPTY_KEY) { atomicAdd(&s_tbl_used, 1u); kk = gk.bits; }
                }
                if (kk == gk.bits) { acc = st.acc + (size_t)s * P.acc_words; break; }
                s = (s + 1) & mask;
              }
            }
            if (!acc) {
              if (st.slots && !s_tbl_off) atomicAdd(&s_tbl_miss, 1u);
              unsigned int gslot = table_find_or_insert(A.tbl, gk.bits, gk.null);
              if (gslot == 0xffffffffu) atomicExch(&A.ctr->agg_overflow, 1u);
              else acc = A.tbl.acc + (size_t)gslot * P.acc_words;
            }
          }
        }
        for (int a = 0; a < P.n_aggs; ++a) {
          const DevAgg g = P.aggs[a];
          Value v;
          int err2 = eval_expr(P, g.arg, row, cells, &v, nullptr);
          if (err2) report_err(A.ctr, A.entry_base + e, err2);
          const bool has = !err2 && !v.null;
          const unsigned int cnt = solo ? (has ? 1u : 0u) : __reduce_add_sync(peers, has ? 1u : 0u);
          unsigned long long* w = acc + g.acc_off;  // only dereferenced by a leader that found a slot
          const bool commit = leader && acc != nullptr && cnt != 0;
          if (g.kind == AGG_COUNT) {
            if (commit) atomicAdd(&w[0], (unsigned long long)cnt);
          } else if (agg_is_extremum(g.kind)) {  // MAX / MIN: running unsigned maximum of the (complemented) order-preserving key
            unsigned long long key = has ? extremum_key(v.bits, g.arg_et, g.arg_unsigned, g.kind == AGG_MIN) : 0ull;
            if (!solo)
              for (unsigned int mm = peers & (peers - 1); mm; mm &= mm - 1) {  // the leader is the lowest lane
                unsigned long long other = __shfl_sync(peers, key, __ffs(mm) - 1);
                key = other > key ? other : key;
              }
            if (commit) { atomicAdd(&w[0], (unsigned long long)cnt); atomicMax(&w[1], key); }
          } else if (g.kind == AGG_FIRST) {  // every row counts, a NULL one too: the peers' earliest (key, value)
            unsigned long long key = err2 ? 0ull : first_agg_key(A.entry_base + e, A.desc, v.null), val = has ? v.bits : 0ull;
            if (!solo)
              for (unsigned int mm = peers & (peers - 1); mm; mm &= mm - 1) {
                const unsigned long long ok2 = __shfl_sync(peers, key, __ffs(mm) - 1), ov = __shfl_sync(peers, val, __ffs(mm) - 1);
                if (ok2 > key) { key = ok2; val = ov; }
              }
            if (leader && acc != nullptr && key) first_agg_update(w, key, val);
          } else if (agg_is_bit(g.kind)) {
            unsigned long long x = bit_agg_word(g.kind, has, v.bits);
            if (!solo) {
              const unsigned int lo = g.kind == AGG_BIT_XOR ? __reduce_xor_sync(peers, (unsigned int)x) : __reduce_or_sync(peers, (unsigned int)x);
              const unsigned int hi = g.kind == AGG_BIT_XOR ? __reduce_xor_sync(peers, (unsigned int)(x >> 32)) : __reduce_or_sync(peers, (unsigned int)(x >> 32));
              x = ((unsigned long long)hi << 32) | lo;
            }
            if (leader && acc != nullptr && x) { if (g.kind == AGG_BIT_XOR) atomicXor(&w[0], x); else atomicOr(&w[0], x); }
          } else if (g.arg_et == 1) {
            // exact: every lane adds its own value into the group's fixed-point accumulator (plans with a Real SUM / AVG run
            // without warp pre-aggregation: `peers` is the lane itself, see above)
            if (commit) {
              atomicAdd(&w[0], (unsigned long long)cnt);
              f64_acc_add(v.bits, [&](uint32_t d, int64_t x) { atomicAdd(&w[1 + d], (unsigned long long)x); });
            }
          } else {
            const uint32_t lo = has ? (uint32_t)v.bits : 0u, hi = has ? (uint32_t)(v.bits >> 32) : 0u;
            unsigned long long lo_sum, hi_sum;
            if (solo) {
              lo_sum = lo;
              hi_sum = g.arg_unsigned ? (unsigned long long)hi : (unsigned long long)(long long)(int32_t)hi;
            } else {  // 16-bit pieces: 32 of them cannot overflow a 32-bit redux
              const unsigned int s0 = __reduce_add_sync(peers, lo & 0xffffu), s1 = __reduce_add_sync(peers, lo >> 16);
              lo_sum = (unsigned long long)s0 + ((unsigned long long)s1 << 16);
              const unsigned int t0 = __reduce_add_sync(peers, hi & 0xffffu);
              if (g.arg_unsigned) hi_sum = (unsigned long long)t0 + ((unsigned long long)__reduce_add_sync(peers, hi >> 16) << 16);
              else hi_sum = (unsigned long long)((long long)__reduce_add_sync(peers, (int)hi >> 16) * 65536ll + (long long)t0);
            }
            if (commit) { atomicAdd(&w[0], (unsigned long long)cnt); atomicAdd(&w[1], lo_sum); atomicAdd(&w[2], hi_sum); }
          }
        }
      }
    }
    if (live) ts.warn += row.warn;  // warnings of the expressions evaluated after the commit point (outputs, group keys, arguments, sort keys)
    return false;
  };

  for (uint32_t k = 0;; ++k) {
    const int cur = (int)(k % N_STAGES);
    mbar_wait_sleep(&s_full[cur], (k / N_STAGES) & 1);
    const TileMeta m = s_meta[cur];
    const uint32_t tile = m.tile;
    if (tile >= n_tiles) {
      if (IS_SCAN && tid == 0) {  // tell the scan warp there is no tile k
        s_tile_of[k % N_CNT] = tile;
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&s_cnt_ready[k % N_CNT])) : "memory");
      }
      break;
    }
    if (tid == 0) s_redo[(k + 2) & 3] = 0;  // last read two tiles ago, next written two tiles ahead
    // high-cardinality GROUP BY: once three quarters of the entries seen went past the CTA table, stop probing it
    if (MODE == PM_AGG && tid == 0 && k >= 16 && !s_tbl_off && s_tbl_miss * 4u > k * TILE * 3u) s_tbl_off = 1;
    bool redo = true;
    if (m.staged) {
      unsigned char* st = stage_base + (size_t)cur * STAGE_BYTES;
      SmemView sv;
      sv.skeys = st + m.keys_adj;
      sv.svals = st + STAGE_KEY_CAP + m.vals_adj;
      sv.skoff = reinterpret_cast<const uint32_t*>(st + STAGE_KEY_CAP + STAGE_VAL_CAP) + m.koff_adj;
      sv.svoff = reinterpret_cast<const uint32_t*>(st + STAGE_KEY_CAP + STAGE_VAL_CAP + STAGE_OFF_CAP) + m.voff_adj;
      sv.gvals = A.blk.vals;
      redo = tile_body(sv, m.w_hi < A.e_hi ? m.w_hi : A.e_hi, k, tile);
    }
    if (redo) tile_body(A.blk, A.e_hi, k, tile);
    __syncwarp();  // this warp is done with stage `cur`: let the producer refill it
    if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&s_empty[cur])) : "memory");
  }
  // ---- epilogue: flush CTA-private state ----
  if (MODE == PM_CHECKSUM) {
    for (int off = 16; off > 0; off >>= 1) {
      ts.ck_x ^= __shfl_xor_sync(0xffffffffu, ts.ck_x, off);
      ts.ck_kvs += __shfl_xor_sync(0xffffffffu, ts.ck_kvs, off);
      ts.ck_bytes += __shfl_xor_sync(0xffffffffu, ts.ck_bytes, off);
    }
    if (lane == 0 && ts.ck_kvs) { atomicXor(&A.ctr->checksum, ts.ck_x); atomicAdd(&A.ctr->total_kvs, ts.ck_kvs); atomicAdd(&A.ctr->total_bytes, ts.ck_bytes); }
  }
  if (MODE == PM_TOPN) {
    cta256_sync();
    cta_topn_compact(tb, (unsigned int)A.limit, &s_top_cnt, &s_top_have_thr, &s_top_thr, P);
    unsigned int keep = s_top_cnt;
    for (unsigned int i = tid; i < keep; i += TILE) A.topn.items[(size_t)blockIdx.x * A.topn.stride + i] = topbuf_get(tb, tb.idx[i]);
    if (tid == 0) A.topn.counts[blockIdx.x] = keep;
  }
  if (MODE == PM_AGG) {
    if (!P.has_group) {
      cta256_sync();
      for (int w = (int)tid; w < P.acc_words; w += TILE) {
        const int op = agg_word_op(P, w);
        unsigned long long x = s_simple_acc[w];
        if (!x) continue;  // every state word starts at 0, the identity of its merge
        if (op == B2_MERGE_MAX) atomicMax(&A.tbl.acc[w], x);
        else if (op == B2_MERGE_OR) atomicOr(&A.tbl.acc[w], x);
        else if (op == B2_MERGE_XOR) atomicXor(&A.tbl.acc[w], x);
        else if (op == B2_MERGE_FIRST_KEY) first_agg_update(&A.tbl.acc[w], x, s_simple_acc[w + 1]);
        else if (op == B2_MERGE_ADD) atomicAdd(&A.tbl.acc[w], x);  // counts, integer limbs and the digits of exact Real sums are all additive
      }
    } else if (st.slots) {
      cta256_sync();
      for (unsigned int s = tid; s < st.slots; s += TILE) {
        if (st.keys[s] == SMEM_EMPTY_KEY) continue;
        unsigned int gslot = table_find_or_insert(A.tbl, st.keys[s], false);
        if (gslot == 0xffffffffu) { atomicExch(&A.ctr->agg_overflow, 1u); continue; }
        for (int a = 0; a < P.n_aggs; ++a) {
          const DevAgg g = P.aggs[a];
          const unsigned long long* src = st.acc + (size_t)s * P.acc_words + g.acc_off;
          unsigned long long* dst = A.tbl.acc + (size_t)gslot * P.acc_words + g.acc_off;
          if (src[0] == 0) continue;
          if (g.kind == AGG_FIRST) { first_agg_update(dst, src[0], src[1]); continue; }
          if (agg_is_bit(g.kind)) { if (g.kind == AGG_BIT_XOR) atomicXor(&dst[0], src[0]); else atomicOr(&dst[0], src[0]); continue; }
          atomicAdd(&dst[0], src[0]);
          if (g.kind == AGG_COUNT) continue;
          if (agg_is_extremum(g.kind)) atomicMax(&dst[1], src[1]);
          else if (g.arg_et == 1) { for (int d = 0; d < F64_ACC_DIGITS; ++d) if (src[1 + d]) atomicAdd(&dst[1 + d], src[1 + d]); }
          else { atomicAdd(&dst[1], src[1]); atomicAdd(&dst[2], src[2]); }
        }
      }
    }
  }
  // statistics
  for (int off = 16; off > 0; off >>= 1) {
    ts.keys += __shfl_xor_sync(0xffffffffu, ts.keys, off);
    ts.size += __shfl_xor_sync(0xffffffffu, ts.size, off);
    t_live += __shfl_xor_sync(0xffffffffu, t_live, off);
    ts.dflt += __shfl_xor_sync(0xffffffffu, ts.dflt, off);
    ts.newer |= __shfl_xor_sync(0xffffffffu, ts.newer, off);
    ts.last = max(ts.last, __shfl_xor_sync(0xffffffffu, ts.last, off));
    ts.warn += __shfl_xor_sync(0xffffffffu, ts.warn, off);
    t_first = min(t_first, __shfl_xor_sync(0xffffffffu, t_first, off));
  }
  if (lane == 0) {
    if (ts.keys) atomicAdd(&A.ctr->processed_keys, ts.keys);
    if (ts.keys && A.range_rows) atomicAdd(A.range_rows, ts.keys);
    if (ts.last) atomicMax(&A.ctr->last_row, A.entry_base + ts.last);
    if (ts.last) atomicMin(&A.ctr->first_row, A.entry_base + t_first);
    if (ts.size) atomicAdd(&A.ctr->processed_size, ts.size);
    if (t_live) atomicAdd(&A.ctr->live_rows, t_live);
    if (ts.dflt) atomicAdd(&A.ctr->default_lookups, ts.dflt);
    if (ts.newer) atomicOr(&A.ctr->met_newer, 1u);
    if (ts.warn) atomicAdd(&A.ctr->warn_div0, (unsigned long long)ts.warn);
  }
}

}  // namespace b2
