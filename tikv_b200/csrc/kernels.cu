// sm_90a kernels of the coprocessor hot path.
//
//   scan_kernel<PM_SCAN>  MVCC forward scan -> row decode -> RPN selection -> ordered compaction into columns
//                         (BatchTableScan + BatchSelection; table_scan_executor.rs, selection_executor.rs)
//   scan_kernel<PM_PROJ>  PM_SCAN whose output cells are expression values (BatchProjection; projection_executor.rs)
//   scan_kernel<PM_AGG>   same front end, then COUNT/SUM/AVG/MAX/MIN into a per-CTA shared-memory group table that is
//                         flushed into the HBM group table (BatchSimpleAggregation / BatchFastHashAggregation)
//   scan_kernel<PM_AGGM>  GROUP BY over 2..4 expressions: composite keys in a hash-tagged HBM table
//                         (BatchSlowHashAggregation; slow_hash_aggr_executor.rs)
//   scan_kernel<PM_TOPN>  per-CTA candidate buffers + threshold, merged by topn_rank_merge / gathered by topn_gather (BatchTopN);
//                         scan_topn_hbm_kernel: the same with the buffers in HBM (LIMIT above 2048)
//   scan_kernel<PM_CHECKSUM>  CRC-64/XZ per KV, XOR-folded (checksum.rs)
//   agg_finalize / agg_result, topn_*, pack_nulls, bounds: result materialisation; gen_*: synthetic region generator (tooling)
// The same device body (scan_kernel.cuh) is compiled per plan at run time by jit.cu.
//
// One thread owns one CF_WRITE entry; only the thread sitting on the first version of a user key does work for
// that key (walks its versions, decodes the row).  CTAs are persistent and pull 256-entry tiles.
#include <cuda_runtime.h>

#include "fast_kernel.cuh"

namespace b2 {

template <int MODE>
__global__ void __launch_bounds__(FK_THREADS, 2) fast_kernel(const __grid_constant__ DevPlan P, const __grid_constant__ ScanArgs A) {
  fast_body<MODE>(P, A);
}

template <int MODE>
__global__ void __launch_bounds__(TILE + 64, 2) scan_kernel(const __grid_constant__ DevPlan P, const __grid_constant__ ScanArgs A) {
  scan_body<MODE>(P, A);
}

// PM_TOPN above LIMIT 2048: the same body with the candidate buffer in HBM (one generic kernel serves every plan)
__global__ void __launch_bounds__(TILE + 64, 2) scan_topn_hbm_kernel(const __grid_constant__ DevPlan P, const __grid_constant__ ScanArgs A) {
  scan_body<PM_TOPN, true>(P, A);
}

static int g_num_sms = 0;
static int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;  // H100 SXM
  }
  return g_num_sms;
}

int scan_num_sms() { return num_sms(); }
size_t scan_stage_bytes(uint32_t key_cap, uint32_t val_cap) { return (size_t)N_STAGES * (key_cap + val_cap + 2 * STAGE_OFF_CAP); }
uint32_t scan_stage_entries() { return TILE + STAGE_LOOK + 1; }
size_t scan_out_stage_bytes() { return (size_t)N_OBUF * OBUF_BYTES + (size_t)N_OBUF * ONULL_WORDS * 4; }
size_t scan_crc_table_bytes() { return 8 * 256 * 8; }

template <int MODE>
static cudaError_t scan_occupancy(int* per_sm, size_t smem) {
  if (smem > 48 * 1024) cudaFuncSetAttribute(scan_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  return cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, scan_kernel<MODE>, TILE + 64, smem);
}
template <int MODE>
static void scan_launch_mode(const DevPlan& plan, const ScanArgs& a, int grid, size_t smem, cudaStream_t s) {
  if (smem > 48 * 1024) cudaFuncSetAttribute(scan_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  scan_kernel<MODE><<<grid, TILE + 64, smem, s>>>(plan, a);
}

// the kernel instantiation that serves a plan
int scan_kernel_mode(const DevPlan& plan) {
  if (plan.mode == PM_SCAN && plan.n_proj) return PM_PROJ;
  if (plan.mode == PM_AGG && plan.n_group > 1) return PM_AGGM;
  return plan.mode;
}

int scan_max_grid(int mode, size_t smem) {
  int per_sm = 0;
  cudaError_t e;
  switch (mode) {
    case PM_PROJ: e = scan_occupancy<PM_PROJ>(&per_sm, smem); break;
    case PM_SCAN: e = scan_occupancy<PM_SCAN>(&per_sm, smem); break;
    case PM_CHECKSUM: e = scan_occupancy<PM_CHECKSUM>(&per_sm, smem); break;
    case PM_TOPN: e = scan_occupancy<PM_TOPN>(&per_sm, smem); break;
    case PM_AGGM: e = scan_occupancy<PM_AGGM>(&per_sm, smem); break;
    default: e = scan_occupancy<PM_AGG>(&per_sm, smem); break;
  }
  if (e != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * num_sms();
}

cudaError_t launch_scan(const DevPlan& plan, const ScanArgs& a, int grid, size_t smem, cudaStream_t s) {
  if (a.c_hi <= a.c_lo) return cudaSuccess;
  uint32_t n_tiles = (a.c_hi - a.c_lo + TILE - 1) / TILE;
  if ((uint32_t)grid > n_tiles) grid = (int)n_tiles;
  switch (scan_kernel_mode(plan)) {
    case PM_PROJ: scan_launch_mode<PM_PROJ>(plan, a, grid, smem, s); break;
    case PM_SCAN: scan_launch_mode<PM_SCAN>(plan, a, grid, smem, s); break;
    case PM_CHECKSUM: scan_launch_mode<PM_CHECKSUM>(plan, a, grid, smem, s); break;
    case PM_TOPN: scan_launch_mode<PM_TOPN>(plan, a, grid, smem, s); break;
    case PM_AGGM: scan_launch_mode<PM_AGGM>(plan, a, grid, smem, s); break;
    default: scan_launch_mode<PM_AGG>(plan, a, grid, smem, s); break;
  }
  return cudaGetLastError();
}

int scan_topn_hbm_max_grid(size_t smem) {
  int per_sm = 0;
  if (smem > 48 * 1024) cudaFuncSetAttribute(scan_topn_hbm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, scan_topn_hbm_kernel, TILE + 64, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * num_sms();
}
cudaError_t launch_scan_topn_hbm(const DevPlan& plan, const ScanArgs& a, int grid, size_t smem, cudaStream_t s) {
  if (a.c_hi <= a.c_lo) return cudaSuccess;
  const uint32_t n_tiles = (a.c_hi - a.c_lo + TILE - 1) / TILE;
  if ((uint32_t)grid > n_tiles) grid = (int)n_tiles;
  if (smem > 48 * 1024) cudaFuncSetAttribute(scan_topn_hbm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  scan_topn_hbm_kernel<<<grid, TILE + 64, smem, s>>>(plan, a);
  return cudaGetLastError();
}

size_t fast_stage_bytes(uint32_t key_cap, uint32_t val_cap) { return (size_t)FK_STAGES * (key_cap + val_cap + 2 * STAGE_OFF_CAP); }
size_t fast_checksum_bytes() { return 8 * 256 * 8 + 256 * 8; }
template <int MODE>
static cudaError_t fast_occupancy(int* per_sm, size_t smem) {
  if (smem > 48 * 1024) cudaFuncSetAttribute(fast_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  return cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, fast_kernel<MODE>, FK_THREADS, smem);
}
int fast_max_grid(int mode, size_t smem) {
  int per_sm = 0;
  cudaError_t e = mode == PM_TOPN ? fast_occupancy<PM_TOPN>(&per_sm, smem) : (mode == PM_CHECKSUM ? fast_occupancy<PM_CHECKSUM>(&per_sm, smem) : fast_occupancy<PM_AGG>(&per_sm, smem));
  if (e != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * num_sms();
}
template <int MODE>
static void fast_launch_mode(const DevPlan& plan, const ScanArgs& a, int grid, size_t smem, cudaStream_t s) {
  if (smem > 48 * 1024) cudaFuncSetAttribute(fast_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  fast_kernel<MODE><<<grid, FK_THREADS, smem, s>>>(plan, a);
}
cudaError_t launch_fast(const DevPlan& plan, const ScanArgs& a, int grid, size_t smem, cudaStream_t s) {
  if (a.c_hi <= a.c_lo) return cudaSuccess;
  uint32_t n_tiles = (a.c_hi - a.c_lo + TILE - 1) / TILE;
  if ((uint32_t)grid > n_tiles) grid = (int)n_tiles;
  switch (plan.mode) {
    case PM_TOPN: fast_launch_mode<PM_TOPN>(plan, a, grid, smem, s); break;
    case PM_CHECKSUM: fast_launch_mode<PM_CHECKSUM>(plan, a, grid, smem, s); break;
    default: fast_launch_mode<PM_AGG>(plan, a, grid, smem, s); break;
  }
  return cudaGetLastError();
}

// ---- TopN: merge candidate lists, gather row payloads ------------------------------------------------------------
size_t topn_smem_bytes(uint32_t cap, int n_order) { return (((size_t)cap * ((size_t)n_order + 2) * 8 + (size_t)cap * 2) + 15) & ~(size_t)15; }

// The CTAs of blockIdx.x = b merge input lists [b * fan_in, (b + 1) * fan_in) into output list b: the best `limit` items,
// sorted.  The host applies it level by level (fan-in 16) down to a single list.  The input lists are sorted and the order
// is total (ids), so an item's output position is its own index + the number of items that come before it in each sibling list.  Every item is
// independent: blockIdx.y splits a group's items over as many CTAs as the occupied part needs, and a thread runs its
// (up to 15) binary searches in lockstep so that their L2 round trips overlap.  Only the first `limit - i` items of a
// sibling can keep item i inside the output, which bounds every search.  Cost follows the items present.
__global__ void __launch_bounds__(256) topn_rank_merge_kernel(const __grid_constant__ DevPlan P, TopNLists in, TopNLists out, unsigned int fan_in) {
  const unsigned int limit = (unsigned int)P.limit;
  const unsigned int l0 = blockIdx.x * fan_in;
  const unsigned int l1 = l0 + fan_in < in.n_lists ? l0 + fan_in : in.n_lists;
  const unsigned int clip = in.stride < limit ? in.stride : limit;
  unsigned int ends[16];
  unsigned int total = 0;
#pragma unroll
  for (unsigned int q = 0; q < 16; ++q) {
    if (l0 + q < l1) { const unsigned int c = in.counts[l0 + q]; total += c < clip ? c : clip; }
    ends[q] = total;
  }
  if (blockIdx.y == 0 && threadIdx.x == 0) out.counts[blockIdx.x] = total < limit ? total : limit;
  for (unsigned int f = blockIdx.y * blockDim.x + threadIdx.x; f < total; f += gridDim.y * blockDim.x) {
    unsigned int q = 0, first = 0;
#pragma unroll
    for (unsigned int z = 0; z < 15; ++z)
      if (f >= ends[z]) { q = z + 1; first = ends[z]; }
    const unsigned int i = f - first;
    TopItem me = in.items[(size_t)(l0 + q) * in.stride + i];
    const unsigned int room = limit - i;  // i < clip <= limit
    unsigned int lo[16], hi[16];
#pragma unroll
    for (unsigned int z = 0; z < 16; ++z) {
      const unsigned int cnt = ends[z] - (z ? ends[z - 1] : 0u);
      lo[z] = 0;
      hi[z] = z == q ? 0u : (cnt < room ? cnt : room);
    }
    bool more = true;
    while (more) {
      more = false;
#pragma unroll
      for (unsigned int z = 0; z < 16; ++z)
        if (lo[z] < hi[z]) {
          const unsigned int mid = (lo[z] + hi[z]) >> 1;
          if (item_less(in.items[(size_t)(l0 + z) * in.stride + mid], me, P)) lo[z] = mid + 1; else hi[z] = mid;
          more = true;
        }
    }
    unsigned int rank = i;
#pragma unroll
    for (unsigned int z = 0; z < 16; ++z) rank += lo[z];
    if (rank < limit) {
      me.slot = ((l0 + q) << 16) | i;
      out.items[(size_t)blockIdx.x * out.stride + rank] = me;
    }
  }
}

cudaError_t launch_topn_merge(const DevPlan& plan, const TopNLists& in, const TopNLists& out, uint32_t fan_in, cudaStream_t s) {
  const unsigned int groups = (in.n_lists + fan_in - 1) / fan_in;
  const unsigned int lists = fan_in < in.n_lists ? fan_in : in.n_lists;
  const unsigned int clip = in.stride < (unsigned int)plan.limit ? in.stride : (unsigned int)plan.limit;
  unsigned int y = (lists * clip + 255) / 256;
  if (y < 1) y = 1;
  if (y > 16) y = 16;  // (a full group then takes four rounds per thread; the usual, nearly empty lists cost the launch of fewer CTAs)
  topn_rank_merge_kernel<<<dim3(groups, y), 256, 0, s>>>(plan, in, out, fan_in);
  return cudaGetLastError();
}

// Two sorted lists (the running top-N, then one unit's) -> the best `limit` of both, sorted: every item finds its rank by
// a binary search in the other list (ids make the order total, so ranks are distinct).  slot = (source list << 16 | index),
// what topn_copy_kernel uses to pick the payload.
__global__ void __launch_bounds__(256) topn_merge2_kernel(const __grid_constant__ DevPlan P, const TopItem* a, const unsigned int* a_cnt, const TopItem* b,
                                                          const unsigned int* b_cnt, TopItem* out, unsigned int* out_cnt, unsigned int limit) {
  const unsigned int na = *a_cnt < limit ? *a_cnt : limit, nb = *b_cnt < limit ? *b_cnt : limit;
  for (unsigned int t = blockIdx.x * blockDim.x + threadIdx.x; t < na + nb; t += gridDim.x * blockDim.x) {
    const bool from_a = t < na;
    const unsigned int i = from_a ? t : t - na;
    TopItem it = from_a ? a[i] : b[i];
    const TopItem* o = from_a ? b : a;
    unsigned int lo = 0, hi = from_a ? nb : na;
    while (lo < hi) {  // items of the other list that come before `it`
      const unsigned int mid = (lo + hi) >> 1;
      if (item_less(o[mid], it, P)) lo = mid + 1; else hi = mid;
    }
    const unsigned int rank = i + lo;
    it.slot = ((from_a ? 0u : 1u) << 16) | i;
    if (rank < limit) out[rank] = it;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *out_cnt = na + nb < limit ? na + nb : limit;
}
cudaError_t launch_topn_merge2(const DevPlan& plan, const TopItem* a, const unsigned int* a_cnt, const TopItem* b, const unsigned int* b_cnt, TopItem* out,
                               unsigned int* out_cnt, uint32_t limit, cudaStream_t s) {
  const unsigned int grid = (2 * limit + 255) / 256 < 1 ? 1 : ((2 * limit + 255) / 256 > 16 ? 16 : (2 * limit + 255) / 256);  // one item per thread: the binary searches are L2 round trips
  topn_merge2_kernel<<<grid, 256, 0, s>>>(plan, a, a_cnt, b, b_cnt, out, out_cnt, limit);
  return cudaGetLastError();
}

// decode every scan column of the selected rows (take_all_append_to, top_n_heap.rs:56-133); one thread per row
__global__ void topn_gather_kernel(const __grid_constant__ DevPlan P, const __grid_constant__ ScanArgs A, const TopItem* items, const unsigned int* count,
                                   unsigned long long* pay, unsigned char* pay_null, unsigned int stride) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *count) return;
  const unsigned long long gid = A.desc ? ~items[i].id : items[i].id;
  uint32_t e = (uint32_t)(gid - A.entry_base);
  RunOut ro;
  resolve_run(A.blk, e, A.e_hi, A.e_hi, P.read_ts, P.isolation, A.dflt, &ro);
  Row row;
  Cells cells;
  uint8_t idx_buf[IDX_RAW_MAX];
  int err = ro.err ? ro.err : (ro.found ? DE_NONE : DE_BAD_WRITE);
  if (!err) {
    uint32_t ko = A.blk.koff[e], kl = A.blk.koff[e + 1] - ko;
    row.enc_key = A.blk.keys + ko; row.enc_key_len = kl - 8; row.commit_ts = ro.commit_ts; row.imms = A.imms;
    if (P.idx_cols > 0) err = index_row_split(P, row, cells, ro.val, ro.val_len, idx_buf);
    else {
      err = row_open(ro.val, ro.val_len, &row.rv);
      if (!err) err = row_split(P, row, cells);
    }
  }
  for (int k = 0; k < P.n_out; ++k) {
    Value v; v.null = true; v.bits = 0;
    if (!err) {
      int e2 = cell_value(P, row, cells, P.out_cols[k], &v);
      if (e2) { report_err(A.ctr, gid, e2); v.null = true; v.bits = 0; }
    }
    pay[(size_t)k * stride + i] = v.null ? 0ull : v.bits;
    pay_null[(size_t)k * stride + i] = v.null ? 1 : 0;
  }
  if (err) report_err(A.ctr, gid, err);
}

cudaError_t launch_topn_gather(const DevPlan& plan, const ScanArgs& a, const TopItem* items, const unsigned int* count, unsigned long long* pay,
                               unsigned char* pay_null, uint32_t stride, cudaStream_t s) {
  if (!stride) return cudaSuccess;
  topn_gather_kernel<<<(stride + 127) / 128, 128, 0, s>>>(plan, a, items, count, pay, pay_null, stride);
  return cudaGetLastError();
}

// payload of the merged list: row i comes from list (slot >> 16), index (slot & 0xffff)
__global__ void topn_copy_kernel(const TopItem* items, const unsigned int* count, unsigned int n_out, unsigned int stride, const unsigned long long* pay0,
                                 const unsigned char* null0, const unsigned long long* pay1, const unsigned char* null1, unsigned long long* pay_out,
                                 unsigned char* null_out) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *count) return;
  unsigned int l = items[i].slot >> 16, j = items[i].slot & 0xffffu;
  const unsigned long long* p = l ? pay1 : pay0;
  const unsigned char* q = l ? null1 : null0;
  for (unsigned int k = 0; k < n_out; ++k) {
    pay_out[(size_t)k * stride + i] = p[(size_t)k * stride + j];
    null_out[(size_t)k * stride + i] = q[(size_t)k * stride + j];
  }
}

cudaError_t launch_topn_copy(const TopItem* items, const unsigned int* count, uint32_t n_out, uint32_t stride, const unsigned long long* pay0,
                             const unsigned char* null0, const unsigned long long* pay1, const unsigned char* null1, unsigned long long* pay_out,
                             unsigned char* null_out, cudaStream_t s) {
  if (!stride) return cudaSuccess;
  topn_copy_kernel<<<(stride + 127) / 128, 128, 0, s>>>(items, count, n_out, stride, pay0, null0, pay1, null1, pay_out, null_out);
  return cudaGetLastError();
}

// byte-per-cell NULL flags -> BitVec words (bit = 1 means non-null)
__global__ void pack_nulls_kernel(const unsigned char* nulls, unsigned int n_cols, unsigned int stride, unsigned int n, unsigned long long* bitmaps,
                                  unsigned int words_per_col) {
  unsigned int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_cols * words_per_col) return;
  unsigned int k = t / words_per_col, w = t % words_per_col;
  unsigned long long bits = 0;
  for (unsigned int b = 0; b < 64; ++b) {
    unsigned int i = w * 64 + b;
    if (i >= n || !nulls[(size_t)k * stride + i]) bits |= 1ull << b;
  }
  bitmaps[(size_t)k * words_per_col + w] = bits;
}

cudaError_t launch_pack_nulls(const unsigned char* nulls, uint32_t n_cols, uint32_t stride, uint32_t n, unsigned long long* bitmaps, uint32_t words_per_col, cudaStream_t s) {
  unsigned int t = n_cols * words_per_col;
  if (!t) return cudaSuccess;
  pack_nulls_kernel<<<(t + 127) / 128, 128, 0, s>>>(nulls, n_cols, stride, n, bitmaps, words_per_col);
  return cudaGetLastError();
}

// ---- aggregation result materialisation ---------------------------------------------------------------------
__global__ void agg_finalize_kernel(const __grid_constant__ DevPlan P, AggTable t, Counters* ctr, unsigned long long* out_keys,
                                    unsigned char* out_key_null, unsigned long long* out_acc) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > t.cap + 1) return;
  if (P.n_group > 1) {
    if (i >= t.cap || t.keys[i] == AGG_EMPTY_KEY) return;
    unsigned int g = atomicAdd(&ctr->n_groups, 1u);
    const int K = P.n_group;
    for (int q = 0; q < K; ++q) out_keys[(size_t)g * K + q] = t.gkeys[(size_t)i * (K + 1) + q];
    out_key_null[g] = (unsigned char)t.gkeys[(size_t)i * (K + 1) + K];
    for (int w = 0; w < P.acc_words; ++w) out_acc[(size_t)g * P.acc_words + w] = t.acc[(size_t)i * P.acc_words + w];
    return;
  }
  if (i < t.cap ? t.keys[i] == AGG_EMPTY_KEY : t.special[i - t.cap] == 0) return;
  unsigned int g = atomicAdd(&ctr->n_groups, 1u);
  out_keys[g] = i == t.cap ? 0ull : (i == t.cap + 1 ? AGG_EMPTY_KEY : t.keys[i]);
  out_key_null[g] = i == t.cap;
  for (int w = 0; w < P.acc_words; ++w) out_acc[(size_t)g * P.acc_words + w] = t.acc[(size_t)i * P.acc_words + w];
}

cudaError_t launch_agg_finalize(const DevPlan& plan, const AggTable& t, Counters* ctr, unsigned long long* out_keys, unsigned char* out_key_null,
                                unsigned long long* out_acc, cudaStream_t s) {
  unsigned int n = t.cap + 2;
  agg_finalize_kernel<<<(n + 255) / 256, 256, 0, s>>>(plan, t, ctr, out_keys, out_key_null, out_acc);
  return cudaGetLastError();
}

// one thread per group: accumulators -> result columns [aggregates..., group key] (fast_hash_aggr_executor.rs:383-413)
__global__ void agg_result_kernel(const __grid_constant__ DevPlan P, unsigned int n_groups, const unsigned long long* g_keys, const unsigned char* g_null,
                                  const unsigned long long* g_acc, unsigned long long** col_data, unsigned long long** col_bitmap) {
  unsigned int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  int c = 0;
  const unsigned long long* acc = g_acc + (size_t)g * P.acc_words;
  for (int a = 0; a < P.n_aggs; ++a) {
    const DevAgg ag = P.aggs[a];
    unsigned long long cnt = acc[ag.acc_off];
    if (ag.kind == 0 || ag.kind == 2) { col_data[c][g] = cnt; ++c; }  // COUNT, or AVG's count column
    if (ag.kind == 1 || ag.kind == 2) {
      bool has = cnt != 0;
      if (ag.arg_et == 1) col_data[c][g] = has ? f64_acc_round(acc + ag.acc_off + 1) : 0ull;
      else {
        b2_decimal d;
        if (has) limbs_to_decimal(acc[ag.acc_off + 1], acc[ag.acc_off + 2], ag.arg_unsigned, &d);
        else { d.int_cnt = 1; d.frac_cnt = 0; d.result_frac_cnt = 0; d.negative = 0; for (int i = 0; i < 9; ++i) d.word_buf[i] = 0; }
        reinterpret_cast<b2_decimal*>(col_data[c])[g] = d;
      }
      if (!has) atomicAnd(&col_bitmap[c][g >> 6], ~(1ull << (g & 63)));
      ++c;
    }
    if (agg_is_extremum(ag.kind)) {  // MAX / MIN: NULL without a non-NULL input
      bool has = cnt != 0;
      col_data[c][g] = has ? extremum_value(acc[ag.acc_off + 1], ag.arg_et, ag.arg_unsigned, ag.kind == AGG_MIN) : 0ull;
      if (!has) atomicAnd(&col_bitmap[c][g >> 6], ~(1ull << (g & 63)));
      ++c;
    }
    // FIRST: NULL without a row or when the first row's value is NULL (impl_first.rs AggrFnStateFirst::push_result);
    // BIT_*: never NULL (impl_bit_op.rs AggrFnStateBitOp::push_result)
    if (ag.kind == AGG_FIRST || agg_is_bit(ag.kind)) {
      uint64_t v;
      if (!first_bit_result(ag.kind, (const uint64_t*)acc + ag.acc_off, &v)) atomicAnd(&col_bitmap[c][g >> 6], ~(1ull << (g & 63)));
      col_data[c][g] = v;
      ++c;
    }
  }
  if (P.n_group > 1) {
    for (int q = 0; q < P.n_group; ++q, ++c) {
      const bool isnull = (g_null[g] >> q) & 1;
      col_data[c][g] = isnull ? 0ull : g_keys[(size_t)g * P.n_group + q];
      if (isnull) atomicAnd(&col_bitmap[c][g >> 6], ~(1ull << (g & 63)));
    }
  } else if (P.has_group) {
    col_data[c][g] = g_null[g] ? 0ull : g_keys[g];
    if (g_null[g]) atomicAnd(&col_bitmap[c][g >> 6], ~(1ull << (g & 63)));
  }
}

cudaError_t launch_agg_result(const DevPlan& plan, unsigned int n_groups, const unsigned long long* g_keys, const unsigned char* g_null,
                              const unsigned long long* g_acc, unsigned long long** col_data, unsigned long long** col_bitmap, cudaStream_t s) {
  if (!n_groups) return cudaSuccess;
  agg_result_kernel<<<(n_groups + 127) / 128, 128, 0, s>>>(plan, n_groups, g_keys, g_null, g_acc, col_data, col_bitmap);
  return cudaGetLastError();
}


// ---- range bounds: lower_bound of each encoded key in each block -------------------------------------------
// One warp per (block, bound), 33-way: each round the 32 lanes compare 32 evenly spaced keys, so a 3e7-entry block takes
// 5 rounds of dependent HBM reads instead of 25 (the request waits for this search before its first unit starts).
// Invariant: every entry below lo is < the bound, every entry at or above hi is >= it.
__global__ void bounds_kernel(const BlockView* blocks, uint32_t n_blocks, const uint8_t* bounds, const uint32_t* bound_offs, uint32_t n_bounds, uint32_t* out) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n_blocks * n_bounds) return;  // (warp-uniform)
  const uint32_t bi = i / n_bounds, qi = i % n_bounds;
  const BlockView b = blocks[bi];
  const uint8_t* q = bounds + bound_offs[qi];
  const uint32_t qn = bound_offs[qi + 1] - bound_offs[qi];
  auto less = [&](uint32_t e) { return bytes_cmp(b.keys + b.koff[e], b.koff[e + 1] - b.koff[e], q, qn) < 0; };
  uint32_t lo = 0, hi = b.n;
  while (hi - lo > 32) {
    const uint32_t p = lo + (uint32_t)(((unsigned long long)(hi - lo) * (lane + 1)) / 33);  // strictly increasing in lane, < hi
    const uint32_t c = __popc(__ballot_sync(0xffffffffu, less(p)));                         // keys below the bound form a prefix
    const uint32_t p_below = __shfl_sync(0xffffffffu, p, c ? c - 1 : 0), p_at = __shfl_sync(0xffffffffu, p, c < 32 ? c : 31);
    if (c) lo = p_below + 1;
    if (c < 32) hi = p_at;
  }
  const uint32_t c = __popc(__ballot_sync(0xffffffffu, lo + lane < hi && less(lo + lane)));
  if (lane == 0) out[i] = lo + c;
}

// per (block, range) unit [lo, hi): do its first and last key share their first 12 bytes, and are those the start of a
// record key?  Keys are sorted, so every key in between shares them too: the clean-entry front end skips those bytes.
// out: 4 words per unit: ok flag, then the unit's first 12 key bytes (3 words, little-endian)
__global__ void unit_prefix_kernel(const BlockView* blocks, uint32_t n_blocks, uint32_t n_ranges, const uint32_t* bounds, uint32_t* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_blocks * n_ranges) return;
  const uint32_t bi = i / n_ranges, r = i % n_ranges;
  const BlockView b = blocks[bi];
  const uint32_t lo = bounds[(size_t)bi * n_ranges * 2 + 2 * r], hi = bounds[(size_t)bi * n_ranges * 2 + 2 * r + 1];
  uint32_t ok = 0;
  if (hi > lo) {
    const uint8_t* f = b.keys + b.koff[lo];
    const uint8_t* l = b.keys + b.koff[hi - 1];
    ok = b.koff[lo + 1] - b.koff[lo] >= 12 && b.koff[hi] - b.koff[hi - 1] >= 12 && record_key_prefix_ok(f);
    for (int j = 0; ok && j < 12; ++j) ok = f[j] == l[j];
    for (int w = 0; w < 3; ++w) out[4 * i + 1 + w] = ok ? ((uint32_t)f[4 * w] | ((uint32_t)f[4 * w + 1] << 8) | ((uint32_t)f[4 * w + 2] << 16) | ((uint32_t)f[4 * w + 3] << 24)) : 0u;
  }
  out[4 * i] = ok;
}

// ends: per block (the n_wblocks CF_WRITE blocks, then the CF_DEFAULT ones) its key and value heap sizes, key_offs[n] and
// val_offs[n].  sample: byte count, then up to 48 bytes of the first value of the first unit (ranges from first_range on,
// in the order the host builds units), which tells the host the row format.
__global__ void block_ends_kernel(const BlockView* blocks, uint32_t n_wblocks, uint32_t n_blocks, uint32_t n_ranges, uint32_t first_range,
                                  const uint32_t* bounds, uint32_t* ends, uint32_t* sample) {
  for (uint32_t b = threadIdx.x; b < n_blocks; b += blockDim.x) {
    const BlockView v = blocks[b];
    ends[2 * b] = v.n ? v.koff[v.n] : 0u;
    ends[2 * b + 1] = v.n ? v.voff[v.n] : 0u;
  }
  if (threadIdx.x) return;
  sample[0] = 0;
  for (uint32_t r = first_range; r < n_ranges; ++r)
    for (uint32_t b = 0; b < n_wblocks; ++b) {
      const uint32_t lo = bounds[(size_t)b * n_ranges * 2 + 2 * r], hi = bounds[(size_t)b * n_ranges * 2 + 2 * r + 1];
      if (hi <= lo) continue;
      const BlockView v = blocks[b];
      const uint32_t o = v.voff[lo], n = min(v.voff[lo + 1] - o, 48u);
      uint8_t* dst = reinterpret_cast<uint8_t*>(sample + 1);
      for (uint32_t j = 0; j < n; ++j) dst[j] = v.vals[o + j];
      sample[0] = n;
      return;
    }
}

cudaError_t launch_open_probe(const BlockView* blocks, uint32_t n_wblocks, uint32_t n_blocks, const uint8_t* bounds, const uint32_t* bound_offs, uint32_t n_ranges,
                              uint32_t first_range, uint32_t* out, uint32_t* unit_ok, uint32_t* ends, uint32_t* sample, cudaStream_t s) {
  const uint32_t n = n_wblocks * n_ranges * 2;
  if (n) {
    bounds_kernel<<<(n + 3) / 4, 128, 0, s>>>(blocks, n_wblocks, bounds, bound_offs, n_ranges * 2, out);
    unit_prefix_kernel<<<(n / 2 + 63) / 64, 64, 0, s>>>(blocks, n_wblocks, n_ranges, out, unit_ok);
  }
  block_ends_kernel<<<1, 128, 0, s>>>(blocks, n_wblocks, n_blocks, n ? n_ranges : 0, first_range, out, ends, sample);
  return cudaGetLastError();
}

__global__ void reverse_rows_kernel(const unsigned long long* in, const unsigned long long* bm_in, uint64_t in_cap, unsigned long long* out, unsigned long long* bm_out,
                                    uint64_t out_cap, uint64_t n_rows, uint64_t n_take, uint32_t n_cols) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_take) return;
  const uint64_t j = n_rows - 1 - i;
  for (uint32_t c = 0; c < n_cols; ++c) {
    out[(size_t)c * out_cap + i] = in[(size_t)c * in_cap + j];
    const bool nonnull = (bm_in[(size_t)c * (in_cap / 64) + (j >> 6)] >> (j & 63)) & 1ull;
    if (!nonnull) atomicAnd(&bm_out[(size_t)c * (out_cap / 64) + (i >> 6)], ~(1ull << (i & 63)));  // NULLs are rare: the bitmap starts as all ones
  }
}
cudaError_t launch_reverse_rows(const unsigned long long* in, const unsigned long long* bm_in, uint64_t in_cap, unsigned long long* out, unsigned long long* bm_out,
                                uint64_t out_cap, uint64_t n_rows, uint64_t n_take, uint32_t n_cols, cudaStream_t s) {
  if (!n_take || !n_cols) return cudaSuccess;
  reverse_rows_kernel<<<(unsigned)((n_take + 255) / 256), 256, 0, s>>>(in, bm_in, in_cap, out, bm_out, out_cap, n_rows, n_take, n_cols);
  return cudaGetLastError();
}

// ---- bytes / json / decimal output columns -----------------------------------------------------------------------
// The scan kernel leaves one cell reference per row (b2_device.h raw_ref_make: HBM address << 16 | length; NULL rows hold
// 0).  The rows a launch appended are [*row_lo, *row_hi) — device-resident counters, so these kernels chain on the stream
// without a host round trip.  Var-length columns: per-1024-row byte sums -> one CTA scans the sums (and moves the column's
// heap cursor) -> every 1024-row block writes its offsets (the chunk column's own i64 offsets, chunk/column.rs:1052-1072)
// and copies its cells into the heap.  Decimal columns: one thread parses one cell's (precision, frac, binary) payload
// into the 40-byte struct a chunk column stores (DecimalDecoder::read_decimal, mysql/decimal.rs:2204-2289).
enum { RAW_BLOCK = 1024 };
__global__ void __launch_bounds__(256) raw_block_sums_kernel(RawArgs R) {
  const RawCol& c = R.col[R.var_idx[blockIdx.y]];
  const unsigned long long lo = *R.row_lo, hi = *R.row_hi;
  const unsigned long long r0 = lo + (unsigned long long)blockIdx.x * RAW_BLOCK;
  if (r0 >= hi) return;
  unsigned int sum = 0;
  for (unsigned int i = threadIdx.x; i < RAW_BLOCK; i += 256)
    if (r0 + i < hi) sum += raw_ref_len(c.cells[r0 + i]);
  __shared__ unsigned int s_w[8];
  sum = __reduce_add_sync(0xffffffffu, sum);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < 8; ++w) t += s_w[w];
    R.sums[(size_t)blockIdx.y * R.sums_stride + blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(1024) raw_scan_sums_kernel(RawArgs R) {
  const int v = blockIdx.x;
  const RawCol& c = R.col[R.var_idx[v]];
  const unsigned long long lo = *R.row_lo, hi = *R.row_hi;
  const unsigned long long nblk = hi > lo ? (hi - lo + RAW_BLOCK - 1) / RAW_BLOCK : 0;
  unsigned long long* sums = R.sums + (size_t)v * R.sums_stride;
  __shared__ unsigned long long s_w[32];
  __shared__ unsigned long long s_carry;
  if (threadIdx.x == 0) s_carry = *c.heap_used;
  __syncthreads();
  for (unsigned long long base = 0; base < nblk; base += 1024) {
    const unsigned long long i = base + threadIdx.x;
    const unsigned long long x = i < nblk ? sums[i] : 0ull;
    unsigned long long incl = x;
    for (int off = 1; off < 32; off <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, off); if ((threadIdx.x & 31) >= off) incl += y; }
    if ((threadIdx.x & 31) == 31) s_w[threadIdx.x >> 5] = incl;
    __syncthreads();
    unsigned long long before = s_carry;
    for (unsigned int w = 0; w < (threadIdx.x >> 5); ++w) before += s_w[w];
    if (i < nblk) sums[i] = before + incl - x;  // the block's first heap offset
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = before + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (lo == 0) c.offsets[0] = 0;
    *c.heap_used = s_carry;
    if (s_carry > c.heap_cap) atomicExch(R.err, 2u);  // (cannot happen: the heap is sized for every value byte the pass can touch)
  }
}
__global__ void __launch_bounds__(256) raw_copy_kernel(RawArgs R) {
  const int v = blockIdx.y;
  const RawCol& c = R.col[R.var_idx[v]];
  const unsigned long long lo = *R.row_lo, hi = *R.row_hi;
  const unsigned long long r0 = lo + (unsigned long long)blockIdx.x * RAW_BLOCK;
  if (r0 >= hi || *R.err == 2u) return;
  __shared__ unsigned long long s_ref[RAW_BLOCK];
  __shared__ unsigned long long s_off[RAW_BLOCK];
  __shared__ unsigned int s_w[8];
  const unsigned int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // thread t owns rows 4t .. 4t+3 of the block
  unsigned long long ref[4];
  unsigned int len[4], mine = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const unsigned long long r = r0 + 4 * tid + j;
    ref[j] = r < hi ? c.cells[r] : 0ull;
    len[j] = raw_ref_len(ref[j]);
    mine += len[j];
  }
  unsigned int incl = mine;
  for (int off = 1; off < 32; off <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= (unsigned)off) incl += y; }
  if (lane == 31) s_w[wid] = incl;
  __syncthreads();
  unsigned long long at = R.sums[(size_t)v * R.sums_stride + blockIdx.x] + incl - mine;
  for (unsigned int w = 0; w < wid; ++w) at += s_w[w];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const unsigned long long r = r0 + 4 * tid + j;
    s_ref[4 * tid + j] = ref[j]; s_off[4 * tid + j] = at;
    at += len[j];
    if (r < hi) c.offsets[r + 1] = (long long)at;
  }
  __syncthreads();
  const unsigned int n = (unsigned int)(hi - r0 < RAW_BLOCK ? hi - r0 : RAW_BLOCK);
  for (unsigned int i = wid; i < n; i += 8) {  // one warp per cell, lanes stride over its bytes
    const unsigned char* src = raw_ref_addr(s_ref[i]);
    const unsigned int l = raw_ref_len(s_ref[i]);
    unsigned char* dst = c.heap + s_off[i];
    for (unsigned int b = lane; b < l; b += 32) dst[b] = src[b];
  }
}
__global__ void raw_decimal_kernel(RawArgs R) {
  const RawCol& c = R.col[R.dec_idx[blockIdx.y]];
  const unsigned long long lo = *R.row_lo, hi = *R.row_hi;
  const unsigned long long r = lo + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= hi) return;
  const unsigned long long ref = c.cells[r];
  b2_decimal d;
  memset(&d, 0, sizeof(d));
  if (ref != 0 && !raw_decimal_parse(raw_ref_addr(ref), raw_ref_len(ref), &d)) { atomicCAS(R.err, 0u, 1u); memset(&d, 0, sizeof(d)); }
  reinterpret_cast<b2_decimal*>(c.heap)[r] = d;
}
cudaError_t launch_raw_materialise(const RawArgs& R, uint64_t max_rows, cudaStream_t s) {
  if (!max_rows) return cudaSuccess;
  const unsigned int nblk = (unsigned int)((max_rows + RAW_BLOCK - 1) / RAW_BLOCK);
  if (R.n_var) {
    raw_block_sums_kernel<<<dim3(nblk, R.n_var), 256, 0, s>>>(R);
    raw_scan_sums_kernel<<<R.n_var, 1024, 0, s>>>(R);
    raw_copy_kernel<<<dim3(nblk, R.n_var), 256, 0, s>>>(R);
  }
  if (R.n_dec) raw_decimal_kernel<<<dim3((unsigned int)((max_rows + 255) / 256), R.n_dec), 256, 0, s>>>(R);
  return cudaGetLastError();
}

__global__ void fill_u64_kernel(unsigned long long* p, unsigned long long v, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}
cudaError_t launch_fill_u64(unsigned long long* p, unsigned long long v, size_t n, cudaStream_t s) {
  if (!n) return cudaSuccess;
  size_t blocks = (n + 255) / 256;
  if (blocks > 4096) blocks = 4096;
  fill_u64_kernel<<<(unsigned)blocks, 256, 0, s>>>(p, v, n);
  return cudaGetLastError();
}

// ---- synthetic region generator ---------------------------------------------------------------------------------
__host__ __device__ inline uint64_t gen_mix(uint64_t seed, uint64_t handle, uint64_t salt) {
  return mix64(seed ^ (handle * 0x9E3779B97F4A7C15ull) ^ ((salt + 1) * 0xBF58476D1CE4E5B9ull));
}
struct GenRow { int kind; /*0 plain,1 extra versions,2 delete,3 lock record*/ uint32_t entries; };
__device__ __forceinline__ GenRow gen_row_kind(const b2_gen_spec& s, uint64_t handle) {
  uint64_t r = gen_mix(s.seed, handle, 1000) % 1000000ull;
  GenRow g;
  if (r < s.extra_versions_per_million) { g.kind = 1; g.entries = 3; }
  else if (r < (uint64_t)s.extra_versions_per_million + s.delete_per_million) { g.kind = 2; g.entries = 2; }
  else if (r < (uint64_t)s.extra_versions_per_million + s.delete_per_million + s.lock_rec_per_million) { g.kind = 3; g.entries = 2; }
  else { g.kind = 0; g.entries = 1; }
  return g;
}
__device__ __forceinline__ bool gen_value(const b2_gen_spec& s, uint64_t handle, uint32_t c, uint64_t version_salt, int64_t* v) {
  if (s.null_per_million && s.null_per_million[c]) {
    if (gen_mix(s.seed, handle, 500 + c) % 1000000ull < s.null_per_million[c]) return false;
  }
  uint64_t x = gen_mix(s.seed + version_salt, handle, c);
  uint64_t range = s.col_range ? s.col_range[c] : 0;
  int64_t lo = s.col_lo ? s.col_lo[c] : 0;
  *v = range ? (int64_t)((uint64_t)lo + x % range) : (int64_t)x;
  return true;
}
__device__ __forceinline__ uint32_t int_width(int64_t v) {
  if (v >= -128 && v <= 127) return 1;
  if (v >= -32768 && v <= 32767) return 2;
  if (v >= -2147483648ll && v <= 2147483647ll) return 4;
  return 8;
}
__device__ __forceinline__ uint32_t varint_len(uint64_t v) { uint32_t n = 1; while (v >= 0x80) { v >>= 7; ++n; } return n; }
__device__ __forceinline__ uint32_t put_varint(uint8_t* p, uint64_t v) { uint32_t n = 0; while (v >= 0x80) { p[n++] = (uint8_t)(v | 0x80); v >>= 7; } p[n++] = (uint8_t)v; return n; }
__device__ __forceinline__ uint64_t zigzag(int64_t v) { uint64_t u = (uint64_t)v << 1; return v < 0 ? ~u : u; }

// size (write=false) or bytes (write=true) of the row value of `handle`
__device__ uint32_t gen_row_bytes(const b2_gen_spec& s, uint64_t handle, uint64_t version_salt, uint8_t* out, bool write) {
  uint32_t n = 0;
  if (s.row_format == 2) {
    uint32_t nn = 0, nul = 0, total = 0;
    for (uint32_t c = 0; c < s.n_cols; ++c) { int64_t v; if (gen_value(s, handle, c, version_salt, &v)) { ++nn; total += int_width(v); } else ++nul; }
    n = 6 + nn + nul + 2 * nn + total;
    if (!write) return n;
    out[0] = 128; out[1] = 0; out[2] = (uint8_t)nn; out[3] = (uint8_t)(nn >> 8); out[4] = (uint8_t)nul; out[5] = (uint8_t)(nul >> 8);
    uint32_t p_ids = 6, p_null = 6 + nn, p_off = 6 + nn + nul, p_val = p_off + 2 * nn, end = 0;
    for (uint32_t c = 0; c < s.n_cols; ++c) {
      int64_t v;
      if (gen_value(s, handle, c, version_salt, &v)) {
        uint32_t w = int_width(v);
        out[p_ids++] = (uint8_t)(c + 1);
        for (uint32_t i = 0; i < w; ++i) out[p_val + end + i] = (uint8_t)((uint64_t)v >> (8 * i));
        end += w;
        out[p_off] = (uint8_t)end; out[p_off + 1] = (uint8_t)(end >> 8); p_off += 2;
      } else out[p_null++] = (uint8_t)(c + 1);
    }
    return n;
  }
  // row format v1: [VAR_INT colid][VAR_INT zigzag | NIL]
  for (uint32_t c = 0; c < s.n_cols; ++c) {
    int64_t v;
    bool nonnull = gen_value(s, handle, c, version_salt, &v);
    if (write) { out[n] = 8; n += 1 + put_varint(out + n + 1, zigzag((int64_t)(c + 1))); }
    else n += 1 + varint_len(zigzag((int64_t)(c + 1)));
    if (nonnull) { if (write) { out[n] = 8; n += 1 + put_varint(out + n + 1, zigzag(v)); } else n += 1 + varint_len(zigzag(v)); }
    else { if (write) out[n] = 0; n += 1; }
  }
  return n;
}
// write record sizes: type + varint(start_ts) + ['v' len row] (+ 'l' u64 varint for lock records)
__device__ __forceinline__ uint32_t put_write_header(uint8_t* p, uint8_t type, uint64_t start_ts, bool write) {
  if (write) { p[0] = type; return 1 + put_varint(p + 1, start_ts); }
  return 1 + varint_len(start_ts);
}

__global__ void gen_sizes_kernel(const __grid_constant__ b2_gen_spec s, uint32_t* row_entries, uint32_t* row_val_bytes) {
  uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= s.n_rows) return;
  uint64_t handle = s.first_handle + r;
  GenRow g = gen_row_kind(s, handle);
  uint32_t row = gen_row_bytes(s, handle, 0, nullptr, false);
  uint32_t bytes = 0;
  if (g.kind == 0) bytes = put_write_header(nullptr, 'P', s.commit_ts - 1, false) + 2 + row;
  else if (g.kind == 1) {
    bytes = put_write_header(nullptr, 'P', s.newer_ts - 1, false) + 2 + gen_row_bytes(s, handle, 77, nullptr, false);
    bytes += put_write_header(nullptr, 'P', s.commit_ts - 1, false) + 2 + row;
    bytes += put_write_header(nullptr, 'P', s.commit_ts - 11, false) + 2 + gen_row_bytes(s, handle, 99, nullptr, false);
  } else if (g.kind == 2) {
    bytes = put_write_header(nullptr, 'D', s.commit_ts - 1, false);
    bytes += put_write_header(nullptr, 'P', s.commit_ts - 11, false) + 2 + gen_row_bytes(s, handle, 99, nullptr, false);
  } else {
    bytes = put_write_header(nullptr, 'L', s.commit_ts, false) + 1 + 8 + 1;
    bytes += put_write_header(nullptr, 'P', s.commit_ts - 1, false) + 2 + row;
  }
  row_entries[r] = g.entries;
  row_val_bytes[r] = bytes;
}

__device__ void gen_put_key(const b2_gen_spec& s, uint64_t handle, uint64_t commit_ts, uint8_t* k) {
  // memcomparable('t' ‖ i64cmp(table_id) ‖ "_r" ‖ i64cmp(handle)) ‖ !commit_ts  (35 bytes)
  uint8_t raw[19];
  raw[0] = 't';
  uint64_t t = (uint64_t)s.table_id ^ 0x8000000000000000ull, h = handle ^ 0x8000000000000000ull;
  for (int i = 0; i < 8; ++i) { raw[1 + i] = (uint8_t)(t >> (8 * (7 - i))); raw[11 + i] = (uint8_t)(h >> (8 * (7 - i))); }
  raw[9] = '_'; raw[10] = 'r';
  for (int i = 0; i < 8; ++i) { k[i] = raw[i]; k[9 + i] = raw[8 + i]; }
  k[8] = 0xff; k[17] = 0xff;
  k[18] = raw[16]; k[19] = raw[17]; k[20] = raw[18];
  for (int i = 21; i < 26; ++i) k[i] = 0;
  k[26] = 0xff - 5;
  uint64_t nts = ~commit_ts;
  for (int i = 0; i < 8; ++i) k[27 + i] = (uint8_t)(nts >> (8 * (7 - i)));
}

__device__ uint32_t gen_put_record(const b2_gen_spec& s, uint64_t handle, uint8_t type, uint64_t start_ts, uint64_t version_salt, bool with_row, uint8_t* v) {
  uint32_t n = put_write_header(v, type, start_ts, true);
  if (with_row) {
    uint32_t row = gen_row_bytes(s, handle, version_salt, v + n + 2, true);
    v[n] = 'v'; v[n + 1] = (uint8_t)row;
    n += 2 + row;
  }
  return n;
}

__global__ void gen_write_kernel(const __grid_constant__ GenArgs a) {
  const b2_gen_spec& s = a.spec;
  uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r > s.n_rows) return;
  if (r == s.n_rows) {  // terminal offsets
    uint32_t e = a.row_entry_off[r];
    a.koff[e] = e * 35u;
    a.voff[e] = a.row_val_off[r];
    return;
  }
  uint64_t handle = s.first_handle + r;
  GenRow g = gen_row_kind(s, handle);
  uint32_t e = a.row_entry_off[r];
  uint32_t vo = a.row_val_off[r];
  // versions are emitted newest first (descending commit_ts)
  uint64_t cts[3]; uint8_t typ[3]; uint64_t sts[3]; uint64_t salt[3]; bool with_row[3];
  int n = 0;
  if (g.kind == 1) { cts[n] = s.newer_ts; typ[n] = 'P'; sts[n] = s.newer_ts - 1; salt[n] = 77; with_row[n] = true; ++n; }
  if (g.kind == 3) { cts[n] = s.commit_ts + 1; typ[n] = 'L'; sts[n] = s.commit_ts; salt[n] = 0; with_row[n] = false; ++n; }
  if (g.kind == 2) { cts[n] = s.commit_ts; typ[n] = 'D'; sts[n] = s.commit_ts - 1; salt[n] = 0; with_row[n] = false; ++n; }
  else { cts[n] = s.commit_ts; typ[n] = 'P'; sts[n] = s.commit_ts - 1; salt[n] = 0; with_row[n] = true; ++n; }
  if (g.kind == 1 || g.kind == 2) { cts[n] = s.commit_ts - 10; typ[n] = 'P'; sts[n] = s.commit_ts - 11; salt[n] = 99; with_row[n] = true; ++n; }
  for (int i = 0; i < n; ++i) {
    a.koff[e + i] = (e + i) * 35u;
    gen_put_key(s, handle, cts[i], a.keys + (size_t)(e + i) * 35u);
    a.voff[e + i] = vo;
    uint32_t len = gen_put_record(s, handle, typ[i], sts[i], salt[i], with_row[i], a.vals + vo);
    if (typ[i] == 'L') {  // last_change -> the Put right below (commit_ts), 1 version away
      uint8_t* p = a.vals + vo + len;
      p[0] = 'l';
      for (int b = 0; b < 8; ++b) p[1 + b] = (uint8_t)(s.commit_ts >> (8 * (7 - b)));
      p[9] = 1;
      len += 10;
    }
    vo += len;
  }
}

cudaError_t launch_gen_sizes(const b2_gen_spec& spec, uint32_t* row_entries, uint32_t* row_val_bytes, cudaStream_t s) {
  if (!spec.n_rows) return cudaSuccess;
  gen_sizes_kernel<<<(unsigned)((spec.n_rows + 255) / 256), 256, 0, s>>>(spec, row_entries, row_val_bytes);
  return cudaGetLastError();
}
cudaError_t launch_gen_write(const GenArgs& a, cudaStream_t s) {
  gen_write_kernel<<<(unsigned)((a.spec.n_rows + 1 + 255) / 256), 256, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace b2
