// Host engine behind the C ABI (include/b2_copr.h): plan lowering, range/lock handling, block staging over two
// CUDA streams, kernel launches, result materialisation and error mapping.
//
// Reference counterparts: BatchExecutor trait (tidb_query_executors/src/interface.rs:36-97), BatchExecutorsRunner
// (runner.rs:606-851), TikvStorage/RangesScanner (src/coprocessor/dag/storage_impl.rs:39-123,
// tidb_query_common/src/storage/scanner.rs:122-221), lock checks of LatestKvPolicy::handle_lock
// (src/storage/mvcc/reader/scanner/forward.rs:384-431, txn_types/src/lock.rs:343-416, 520-611),
// ChecksumContext (src/coprocessor/checksum.rs:26-98).
#include <cuda_runtime.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <ctime>
#include <future>
#include <map>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include <cub/device/device_scan.cuh>

#include "encode.cuh"
#include "jit.h"
#include "kernels.cuh"
#include "plan_literal.h"
#include "plan_compile.h"

using namespace b2;

static thread_local std::string g_last_error;
namespace b2 { void set_last_error(const std::string& m) { g_last_error = m; } }  // for the other translation units (sst.cu)

#define CUDA_TRY(expr)                                                                                   \
  do {                                                                                                   \
    cudaError_t _e = (expr);                                                                             \
    if (_e != cudaSuccess) {                                                                             \
      fail(B2_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));                             \
      return B2_ERR_CUDA;                                                                                \
    }                                                                                                    \
  } while (0)

namespace {

// Request-scoped buffers come from a small caching pool (per process, per device): a coprocessor request is short and
// cudaMalloc / cudaMallocHost / cudaFree cost more than the request itself (and cudaFree synchronises the device).
struct BufPool {
  struct Blk { void* p; size_t cap; int device; };
  std::mutex mu;
  std::vector<Blk> free_list;
  size_t held = 0, limit;
  bool pinned;
  BufPool(bool pinned_, size_t limit_) : limit(limit_), pinned(pinned_) {}
  cudaError_t get(size_t n, void** p, size_t* cap) {
    int dev = 0;
    cudaGetDevice(&dev);
    {
      std::lock_guard<std::mutex> g(mu);
      size_t best = free_list.size();
      for (size_t i = 0; i < free_list.size(); ++i)
        if ((pinned || free_list[i].device == dev) && free_list[i].cap >= n && free_list[i].cap <= 2 * n + (1 << 20) && (best == free_list.size() || free_list[i].cap < free_list[best].cap)) best = i;
      if (best != free_list.size()) {
        *p = free_list[best].p; *cap = free_list[best].cap;
        held -= free_list[best].cap;
        free_list.erase(free_list.begin() + best);
        return cudaSuccess;
      }
    }
    size_t want = (n + 255) & ~(size_t)255;
    cudaError_t e = pinned ? cudaMallocHost(p, want) : cudaMalloc(p, want);
    if (e != cudaSuccess) {  // out of memory: drop the cache and retry once
      trim(0);
      cudaGetLastError();
      e = pinned ? cudaMallocHost(p, want) : cudaMalloc(p, want);
    }
    if (e == cudaSuccess) *cap = want;
    return e;
  }
  void put(void* p, size_t cap) {
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu);
    free_list.push_back(Blk{p, cap, dev});
    held += cap;
    while (held > limit && !free_list.empty()) {  // evict the largest
      size_t big = 0;
      for (size_t i = 1; i < free_list.size(); ++i) if (free_list[i].cap > free_list[big].cap) big = i;
      if (pinned) cudaFreeHost(free_list[big].p); else cudaFree(free_list[big].p);
      held -= free_list[big].cap;
      free_list.erase(free_list.begin() + big);
    }
  }
  void trim(size_t keep) {
    std::lock_guard<std::mutex> g(mu);
    while (held > keep && !free_list.empty()) {
      if (pinned) cudaFreeHost(free_list.back().p); else cudaFree(free_list.back().p);
      held -= free_list.back().cap;
      free_list.pop_back();
    }
  }
};
BufPool& dev_pool() { static BufPool p(false, 24ull << 30); return p; }
BufPool& host_pool() { static BufPool p(true, 8ull << 30); return p; }

// Timing events, reused across requests (per process, per device): creating and destroying them costs a driver call each,
// and a request times every launch.  An event taken from the pool has completed whatever it last recorded, because
// a request waits for its stream before giving its events back.
struct EventPool {
  std::mutex mu;
  std::vector<std::pair<int, cudaEvent_t>> free_list;
  cudaEvent_t get() {
    int dev = 0;
    cudaGetDevice(&dev);
    {
      std::lock_guard<std::mutex> g(mu);
      for (size_t i = free_list.size(); i-- > 0;)
        if (free_list[i].first == dev) { cudaEvent_t e = free_list[i].second; free_list.erase(free_list.begin() + i); return e; }
    }
    cudaEvent_t e = nullptr;
    return cudaEventCreate(&e) == cudaSuccess ? e : nullptr;
  }
  void put(cudaEvent_t e) {  // the event's device must be current
    if (!e) return;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu);
    free_list.push_back({dev, e});
  }
};
EventPool& event_pool() { static EventPool* p = new EventPool(); return *p; }

// A block taken from `Pool` and owned: it goes back to the pool when the buffer is destroyed or released, moving leaves the
// source empty.  The pool tags a returned block with the current device, so that device must be current then.
template <BufPool& (*Pool)()>
struct PooledBuf {
  void* p = nullptr;
  size_t cap = 0;
  PooledBuf() = default;
  PooledBuf(PooledBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  PooledBuf& operator=(PooledBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  ~PooledBuf() { release(); }
  void release() { if (p) Pool().put(p, cap); p = nullptr; cap = 0; }
};
struct DevBuf : PooledBuf<dev_pool> {  // growable device allocation
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaDeviceSynchronize();  // growing: in-flight work may still touch the old block before it goes back to the pool
    release();
    return dev_pool().get(n, &p, &cap);
  }
  // the same for a buffer only ever used on `s`: growing waits for that stream alone, not for the whole device
  cudaError_t reserve_on(cudaStream_t s, size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaStreamSynchronize(s);
    release();
    return dev_pool().get(n, &p, &cap);
  }
};
struct HostBuf : PooledBuf<host_pool> {  // growable pinned host allocation
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    release();
    return host_pool().get(n, &p, &cap);
  }
};

struct SrcBlock {  // caller's block descriptor + sizes
  b2_cf_block c;
  uint64_t key_bytes = 0, val_bytes = 0;
  uint64_t entry_base = 0;
};

struct Unit { uint32_t range_idx, block_idx, e_lo, e_hi, fast_ok; uint32_t prefix[3]; /* the unit's first 12 key bytes when fast_ok */ };

struct StageSlot {
  DevBuf keys, koff, vals, voff;
  int block = -1;
  bool done = false;  // every unit that reads `block` has been launched: the slot may be refilled (after free_ev)
  cudaEvent_t ready = nullptr, free_ev = nullptr;
  bool free_recorded = false;
};

// ---- lock records (host): the subset of Lock::parse that check_ts_conflict_si needs ----
struct HostLock { uint8_t type = 0; std::vector<uint8_t> primary; uint64_t ts = 0, min_commit_ts = 0; bool async_commit = false; };

bool parse_compact_bytes(const uint8_t*& p, size_t& n, std::vector<uint8_t>* out) {
  int64_t len;
  uint32_t c = dec_var_i64(p, (uint32_t)n, &len);
  if (!c || len < 0 || (uint64_t)len > n - c) return false;
  if (out) out->assign(p + c, p + c + len);
  p += c + len; n -= c + (size_t)len;
  return true;
}
bool parse_lock(const uint8_t* p, size_t n, HostLock* l) {
  if (n == 0) return false;
  uint8_t t = p[0];
  if (t != 'P' && t != 'D' && t != 'L' && t != 'S' && t != 'H') return false;
  l->type = t;
  if (t == 'H') return true;
  ++p; --n;
  if (!parse_compact_bytes(p, n, &l->primary)) return false;
  uint32_t c = dec_var_u64_tu(p, (uint32_t)n, &l->ts);
  if (!c) return false;
  p += c; n -= c;
  if (n == 0) return true;
  uint64_t ttl;
  c = dec_var_u64_tu(p, (uint32_t)n, &ttl);
  if (!c) return false;
  p += c; n -= c;
  while (n > 0) {
    uint8_t tag = *p++; --n;
    if (tag == 'v') { if (n < 1 || n - 1 < p[0]) return false; size_t k = 1 + p[0]; p += k; n -= k; }
    else if (tag == 'f' || tag == 't' || tag == 'c' || tag == 'g') { if (n < 8) return false; if (tag == 'c') l->min_commit_ts = ld_be64(p); p += 8; n -= 8; }
    else if (tag == 'a') {
      l->async_commit = true;
      uint64_t cnt; c = dec_var_u64_tu(p, (uint32_t)n, &cnt);
      if (!c) return false;
      p += c; n -= c;
      for (uint64_t i = 0; i < cnt; ++i) if (!parse_compact_bytes(p, n, nullptr)) return false;
    } else if (tag == 'r') {
      uint64_t cnt; c = dec_var_u64_tu(p, (uint32_t)n, &cnt);
      if (!c || n - c < cnt * 8) return false;
      p += c + cnt * 8; n -= c + cnt * 8;
    } else if (tag == 'l') {
      if (n < 8) return false;
      p += 8; n -= 8;
      uint64_t v; c = dec_var_u64_tu(p, (uint32_t)n, &v);
      if (!c) return false;
      p += c; n -= c;
    } else if (tag == 's') { uint64_t v; c = dec_var_u64_tu(p, (uint32_t)n, &v); if (!c) return false; p += c; n -= c; }
    else if (tag == 'F') {}
    else break;
  }
  return true;
}

int cmp_bytes_host(const uint8_t* a, size_t an, const uint8_t* b, size_t bn) {
  size_t m = std::min(an, bn);
  int c = m ? memcmp(a, b, m) : 0;
  if (c) return c;
  return an < bn ? -1 : (an > bn ? 1 : 0);
}

const char* dev_err_message(int code, int* status, int* mysql) {
  *mysql = 0;
  switch (code) {
    case DE_BAD_WRITE: *status = B2_ERR_STORAGE; return "bad format write";
    case DE_KEY_TOO_SHORT: *status = B2_ERR_STORAGE; return "key is too short to carry a timestamp";
    case DE_DEFAULT_NOT_FOUND: *status = B2_ERR_STORAGE; return "default not found";
    case DE_WRITE_CONFLICT: *status = B2_ERR_WRITE_CONFLICT; return "write conflict (RcCheckTs): a newer version exists";
    case DE_BAD_USER_KEY: *status = B2_ERR_STORAGE; return "invalid memcomparable user key";
    case DE_BAD_RECORD_KEY: *status = B2_ERR_CORRUPTED; return "record key expected";
    case DE_ROW_COLID_NOT_VARINT: *status = B2_ERR_CORRUPTED; return "Unable to decode row: column id must be VAR_INT";
    case DE_ROW_EOF: *status = B2_ERR_CORRUPTED; return "unexpected eof while decoding row";
    case DE_ROW_BAD_DATUM: *status = B2_ERR_CORRUPTED; return "unsupported or truncated datum in row";
    case DE_ROW_V2_BAD_INT: *status = B2_ERR_CORRUPTED; return "Failed to decode row v2 data as i64/u64";
    case DE_ROW_V2_RANGE: *status = B2_ERR_CORRUPTED; return "row v2 value slice out of range";
    case DE_MISSING_NOT_NULL: *status = B2_ERR_CORRUPTED; return "Data is corrupted, missing data for NOT NULL column";
    case DE_MISSING_COMMIT_TS: *status = B2_ERR_CORRUPTED; return "Query asks for _tidb_commit_ts, but the data is missing";
    case DE_DATUM_DECODE: *status = B2_ERR_CORRUPTED; return "Unsupported datum flag for the column's vector type";
    case DE_OVERFLOW_BIGINT: *status = B2_ERR_EVALUATE; *mysql = B2_MYSQL_ERR_DATA_OUT_OF_RANGE; return "BIGINT value is out of range";
    case DE_OVERFLOW_UBIGINT: *status = B2_ERR_EVALUATE; *mysql = B2_MYSQL_ERR_DATA_OUT_OF_RANGE; return "BIGINT UNSIGNED value is out of range";
    case DE_OVERFLOW_DOUBLE: *status = B2_ERR_EVALUATE; *mysql = B2_MYSQL_ERR_DATA_OUT_OF_RANGE; return "DOUBLE value is out of range";
    case DE_OVERFLOW_DIV: *status = B2_ERR_EVALUATE; *mysql = B2_MYSQL_ERR_DATA_OUT_OF_RANGE; return "UNSIGNED BIGINT value is out of range";
    case DE_IDX_BAD_KEY: *status = B2_ERR_CORRUPTED; return "record or index key expected";
    case DE_IDX_MISSING_COL: *status = B2_ERR_CORRUPTED; return "index column is missing value";
    case DE_IDX_BAD_HANDLE: *status = B2_ERR_CORRUPTED; return "Failed to decode handle of the index entry";
    case DE_IDX_NEW_LAYOUT: *status = B2_ERR_UNSUPPORTED; return "index value in the new (restored-data) layout is not on the device path";
    case DE_UNSUPPORTED_SIG: *status = B2_ERR_UNSUPPORTED; return "scalar function not supported on the device";
    case DE_UNSUPPORTED_TYPE: *status = B2_ERR_UNSUPPORTED; return "column type not supported on the device";
    default: *status = B2_ERR_CUDA; return "unknown device error";
  }
}

}  // namespace

struct b2_exec {
  CompiledPlan cp;
  int device = 0;
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  bool own_stream = false;
  int out_loc = B2_LOC_DEVICE;
  int src_loc = B2_LOC_DEVICE;
  uint64_t read_ts = 0;
  int isolation = B2_ISO_SI;
  bool check_newer = false;

  std::vector<SrcBlock> wblocks, dblocks;
  std::vector<std::vector<uint8_t>> range_lo, range_hi;  // encoded bounds per range (hi possibly cut by a lock)
  std::vector<std::vector<uint8_t>> range_raw_lo, range_raw_hi;  // the caller's raw bounds (take_scanned_range)
  std::vector<uint8_t> working_begin;                    // RangesScanner::working_range_begin_key (scanner.rs:204-229)
  uint64_t last_row_taken = 0;                           // Counters::last_row at the previous take
  uint64_t last_row_seen = 0, first_row_seen = ~0ull;    // Counters::last_row / first_row as of the last batch
  DevBuf range_rows;                                     // per range: rows returned by the MVCC scan
  std::vector<uint64_t> range_rows_taken;                // already handed out by collect_scanned_rows_per_range
  std::vector<int> range_lock_err;                      // 1 = range ends with KeyIsLocked
  std::vector<uint64_t> range_lock_ts;
  std::vector<Unit> units;
  uint32_t first_live_range = 0;                         // backward scans: ranges below a conflicting lock's range are never reached
  size_t cur_unit = 0;                                   // PM_SCAN cursor: the unit being consumed and what is left of it
  uint32_t cur_lo = 0, cur_hi = 0;
  bool started = false, drained = false, failed = false;
  bool saw_lock = false;
  uint64_t lock_keys_seen = 0;

  // device state
  DevBuf ctr_buf, status_buf, out_data, out_bitmap, dflt_views, dflt_store;
  DevBuf tbl_keys, tbl_occ, tbl_acc, tbl_gkeys, tbl_ready, grp_keys, grp_null, grp_acc, res_ptrs;
  std::vector<DevBuf> res_cols, res_bitmaps;
  unsigned int tbl_cap = 0;
  StageSlot slots[2];
  HostBuf h_out, h_ctr, h_res_ptrs;
  uint64_t out_cap = 0;

  // results exposed through b2_batch
  std::vector<b2_column> cols;
  b2_error_info last_err{};
  b2_exec_stats stats{};
  uint64_t entries_scanned = 0;

  // ---- deadline (runner.rs:974 `self.deadline.check()?` at the top of every batch; here also between unit launches) ----
  uint64_t deadline_ns = 0;
  static uint64_t now_ns() { timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return (uint64_t)t.tv_sec * 1000000000ull + (uint64_t)t.tv_nsec; }
  bool deadline_exceeded() {
    if (!deadline_ns || now_ns() < deadline_ns) return false;
    fail(B2_ERR_DEADLINE, "deadline is exceeded");
    drained = true;
    return true;
  }
  // ---- evaluation warnings (BatchExecuteResult::warnings; only "Division by 0" can be raised by the supported functions) ----
  uint64_t warnings_total = 0, warnings_reported = 0;
  // ---- b2_exec_next_batch_async ----
  std::future<int> async_fut;
  b2_batch async_batch{};
  bool async_running = false;
  uint64_t paging_size = 0;
  // B2_DEBUG_AGG_HASH_BITS (read when the request opens): keep only this many bits of the composite-key hash tag, so that
  // different keys collide in the group table on purpose (tests); 0 = all 64
  unsigned int debug_hash_bits = 0;

  int fail(int status, const std::string& msg, int mysql = 0, uint64_t entry = ~0ull) {
    last_err.status = status; last_err.mysql_code = mysql; last_err.entry_index = entry;
    snprintf(last_err.message, sizeof(last_err.message), "%s", msg.c_str());
    g_last_error = msg;
    failed = true;
    return status;
  }

  // The buffer members are destroyed after this body has run, so the device is still current (BufPool::put tags a block
  // with it) and both streams are drained when their blocks go back to the pool.
  ~b2_exec() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    if (copy_stream) { cudaStreamSynchronize(copy_stream); cudaStreamDestroy(copy_stream); }
    for (auto& s : slots) {
      if (s.ready) cudaEventDestroy(s.ready);
      if (s.free_ev) cudaEventDestroy(s.free_ev);
    }
    for (auto& e : kev) { event_pool().put(e.first); event_pool().put(e.second); }
    for (cudaEvent_t e : batch_ev) event_pool().put(e);
    if (own_stream && stream) cudaStreamDestroy(stream);
  }
  // the handle's streams: kernels run on the caller's stream (cfg->cuda_stream) or an own one; block staging of host
  // sources on an own one, created when the first block is staged
  cudaError_t open_streams(const b2_exec_config* cfg) {
    if (cfg && cfg->cuda_stream) { stream = (cudaStream_t)cfg->cuda_stream; return cudaSuccess; }
    cudaError_t e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) own_stream = true;
    return e;
  }

  Counters* ctr() { return (Counters*)ctr_buf.p; }

  // ---- plan-specialised kernel (jit.cu): used as soon as its compilation has finished, the generic kernel until then ----
  int jit_mode = B2_JIT_AUTO;
  bool jit_started = false;
  std::shared_future<JitKernel*> jit_fut;
  void jit_start() {
    if (jit_started || jit_mode == B2_JIT_OFF || cp.dev.mode == PM_CHECKSUM || !jit_available()) return;
    jit_fut = jit_get(device, cp.dev);
    jit_started = true;
  }
  const JitKernel* jit_ready() {
    if (!jit_started) return nullptr;
    if (jit_fut.wait_for(std::chrono::seconds(0)) != std::future_status::ready) return nullptr;
    const JitKernel* k = jit_fut.get();
    return k->ok ? k : nullptr;
  }
  // persistent grid = co-resident CTAs of whichever kernel the next launch uses
  int scan_grid_for(int mode, size_t smem) {
    if (const JitKernel* k = jit_ready()) return jit_max_blocks_per_sm(k, smem) * scan_num_sms();
    return scan_max_grid(mode, smem);
  }
  cudaError_t scan_launch(const ScanArgs& a, int grid, size_t smem) {
    if (const JitKernel* k = jit_ready()) { stats.jit_launches++; return jit_launch(k, a, grid, smem, stream); }
    return launch_scan(cp.dev, a, grid, smem, stream);
  }

  // Row format of the first row a unit will touch (TiDB tables are all-v1 or all-v2 in practice); decides whether the
  // v1 twin of the exact-layout path is part of the kernel.  A wrong guess only costs speed: every row is checked.
  // (A device source's first value was read by compute_units.)
  uint32_t v1_sample_len = 0;
  uint8_t v1_sample[48];
  bool sample_is_v1() {
    if (units.empty()) return false;
    uint8_t buf[64];
    memset(buf, 0, sizeof(buf));
    uint32_t n;
    if (src_loc == B2_LOC_HOST) {
      const Unit& u = units[0];
      const SrcBlock& b = wblocks[u.block_idx];
      if (u.e_lo >= b.c.n) return false;
      n = std::min<uint32_t>(b.c.val_offs[u.e_lo + 1] - b.c.val_offs[u.e_lo], 48);
      memcpy(buf, b.c.vals + b.c.val_offs[u.e_lo], n);
    } else {
      n = std::min<uint32_t>(v1_sample_len, 48);
      memcpy(buf, v1_sample, n);
    }
    // write record: type, varint start_ts, then 'v' len row... (write.rs:296-361); anything else: no opinion
    uint32_t pos = 1;
    while (pos < n && (buf[pos] & 0x80)) ++pos;
    ++pos;
    if (pos + 2 >= n || buf[pos] != 'v') return false;
    return buf[pos + 2] != 128 && buf[pos + 1] > 1;
  }

  // ---- source setup ----
  static void host_offs_end(const b2_cf_block& b, uint64_t* kb, uint64_t* vb) {
    *kb = b.n ? b.key_offs[b.n] : 0;
    *vb = b.n ? b.val_offs[b.n] : 0;
  }

  // A device-resident source is read once while the request opens (compute_units): heap sizes, range bounds, unit
  // prefixes and the row-format sample come back in one copy, behind one stream synchronise.
  int setup_source(const b2_region_source* src, const b2_key_range* ranges, uint32_t n_ranges) {
    src_loc = src->location;
    read_ts = src->read_ts; isolation = src->isolation_level; check_newer = src->check_has_newer_ts_data != 0;
    const bool host = src_loc == B2_LOC_HOST;
    uint64_t base = 0;
    for (uint32_t i = 0; i < src->n_write; ++i) {
      SrcBlock sb; sb.c = src->write[i]; sb.entry_base = base;
      if (host) host_offs_end(sb.c, &sb.key_bytes, &sb.val_bytes);
      base += sb.c.n;
      wblocks.push_back(sb);
    }
    for (uint32_t i = 0; src->dflt && i < src->n_dflt; ++i) {
      SrcBlock sb; sb.c = src->dflt[i];
      if (host) host_offs_end(sb.c, &sb.key_bytes, &sb.val_bytes);
      dblocks.push_back(sb);
    }
    // CF_DEFAULT views of a host source on the device: its blocks are copied once (long values are rare).  A device source's
    // views are written by compute_units.
    if (!dblocks.empty() && host) {
      std::vector<BlockView> views;
      {
        size_t total = 0;
        for (auto& d : dblocks) total += ((d.key_bytes + 31) & ~15ull) + ((d.val_bytes + 31) & ~15ull) + 2 * (((size_t)d.c.n + 1) * 4 + 16);
        CUDA_TRY(dflt_store.reserve(total));
        uint8_t* p = (uint8_t*)dflt_store.p;
        for (auto& d : dblocks) {
          BlockView v; v.n = d.c.n;
          auto put = [&](const void* srcp, size_t bytes) -> const void* {
            uint8_t* dst = p;
            if (bytes) cudaMemcpyAsync(dst, srcp, bytes, cudaMemcpyHostToDevice, stream);
            p += (bytes + 31) & ~15ull;
            return dst;
          };
          v.keys = (const uint8_t*)put(d.c.keys, d.key_bytes);
          v.vals = (const uint8_t*)put(d.c.vals, d.val_bytes);
          v.koff = (const uint32_t*)put(d.c.key_offs, ((size_t)d.c.n + 1) * 4);
          v.voff = (const uint32_t*)put(d.c.val_offs, ((size_t)d.c.n + 1) * 4);
          views.push_back(v);
        }
      }
      CUDA_TRY(dflt_views.reserve(views.size() * sizeof(BlockView)));
      CUDA_TRY(cudaMemcpyAsync(dflt_views.p, views.data(), views.size() * sizeof(BlockView), cudaMemcpyHostToDevice, stream));
      CUDA_TRY(cudaStreamSynchronize(stream));
    }
    // ranges -> encoded bounds (Range::from_pb_range + Key::from_raw)
    for (uint32_t i = 0; i < n_ranges; ++i) {
      range_lo.push_back(encode_memcomparable(ranges[i].start, ranges[i].start_len));
      range_hi.push_back(encode_memcomparable(ranges[i].end, ranges[i].end_len));
      range_lock_err.push_back(0);
      range_lock_ts.push_back(0);
      range_raw_lo.emplace_back(ranges[i].start, ranges[i].start + ranges[i].start_len);
      range_raw_hi.emplace_back(ranges[i].end, ranges[i].end + ranges[i].end_len);
    }
    // CF_LOCK (host memory): LatestKvPolicy::handle_lock for every lock inside a range, in key order
    if (src->lock && src->lock->n && isolation != B2_ISO_RC) {
      const b2_cf_block& L = *src->lock;
      // forward: ranges and locks in ascending order, the first conflict ends the scan; backward (TableScan.desc):
      // both in descending order, rows above the largest conflicting lock are produced first
      for (uint32_t rr = 0; rr < n_ranges; ++rr) {
        const uint32_t r = cp.desc ? n_ranges - 1 - rr : rr;
        for (uint32_t ii = 0; ii < L.n; ++ii) {
          const uint32_t i = cp.desc ? L.n - 1 - ii : ii;
          const uint8_t* k = L.keys + L.key_offs[i];
          size_t kn = L.key_offs[i + 1] - L.key_offs[i];
          if (cp.desc) {
            if (cmp_bytes_host(k, kn, range_hi[r].data(), range_hi[r].size()) >= 0) continue;
            if (cmp_bytes_host(k, kn, range_lo[r].data(), range_lo[r].size()) < 0) break;
          } else {
          if (cmp_bytes_host(k, kn, range_lo[r].data(), range_lo[r].size()) < 0) continue;
          if (cmp_bytes_host(k, kn, range_hi[r].data(), range_hi[r].size()) >= 0) break;
          }
          saw_lock = true;
          HostLock lk;
          if (!parse_lock(L.vals + L.val_offs[i], L.val_offs[i + 1] - L.val_offs[i], &lk)) return fail(B2_ERR_STORAGE, "bad format lock");
          bool conflict;
          if (isolation == B2_ISO_SI) {
            conflict = !(lk.type == 'H' || lk.ts > read_ts || lk.type == 'L' || lk.type == 'S' || lk.min_commit_ts > read_ts);
            for (uint32_t b = 0; conflict && b < src->n_bypass_locks; ++b) if (src->bypass_locks[b] == lk.ts) conflict = false;
            if (conflict && read_ts == ~0ull && !lk.async_commit) {
              // reading the latest committed version of the primary key ignores its own lock
              int rl = raw_key_len(k, (uint32_t)kn);
              if (rl >= 0 && (size_t)rl == lk.primary.size()) {
                bool same = true;
                for (int j = 0; j < rl && same; ++j) same = raw_at(k, j) == lk.primary[j];
                if (same) conflict = false;
              }
            }
          } else {  // RcCheckTs: lock.rs:418-455
            conflict = !(lk.type == 'H' || lk.type == 'L' || lk.type == 'S');
            for (uint32_t b = 0; conflict && b < src->n_bypass_locks; ++b) if (src->bypass_locks[b] == lk.ts) conflict = false;
          }
          if (!conflict) continue;
          for (uint32_t a = 0; a < src->n_access_locks; ++a)
            if (src->access_locks[a] == lk.ts) return fail(B2_ERR_UNSUPPORTED, "access_locks read-through is not supported on the device path");
          // rows before this key are produced, then the request fails (forward.rs:401-428; backward.rs:176-225: rows after it)
          if (cp.desc) { range_lo[r].assign(k, k + kn); range_lo[r].insert(range_lo[r].end(), 9, (uint8_t)0xff); }  // past every version of that key
          else range_hi[r].assign(k, k + kn);
          range_lock_err[r] = isolation == B2_ISO_SI ? B2_ERR_KEY_IS_LOCKED : B2_ERR_WRITE_CONFLICT;
          range_lock_ts[r] = lk.ts;
          lock_keys_seen++;
          break;
        }
        if (range_lock_err[r]) {
          if (cp.desc) first_live_range = r;  // ranges below it are never reached
          else { range_lo.resize(r + 1); range_hi.resize(r + 1); range_lock_err.resize(r + 1); range_lock_ts.resize(r + 1); }
          break;
        }
      }
    }
    return compute_units();
  }

  // Device source: one upload (block views, range bounds), the probe kernels, one download into pinned memory, one wait.
  // Fills res / unit_ok (compute_units' layout), the heap sizes of every block, the CF_DEFAULT views and the v1 sample.
  HostBuf h_open;
  int probe_device_source(uint32_t* res, uint32_t* unit_ok) {
    const uint32_t nr = (uint32_t)range_lo.size(), nb = (uint32_t)wblocks.size(), nd = (uint32_t)dblocks.size();
    if (!nb && !nd) return B2_OK;
    auto a16 = [](size_t n) { return (n + 15) & ~(size_t)15; };
    size_t flat_bytes = 0;
    for (uint32_t r = 0; r < nr; ++r) flat_bytes += range_lo[r].size() + range_hi[r].size();
    const size_t views_at = 0, flat_at = a16((size_t)(nb + nd) * sizeof(BlockView)), offs_at = flat_at + a16(flat_bytes + 16);
    const size_t in_bytes = a16(offs_at + ((size_t)nr * 2 + 1) * 4);
    const size_t n_ends = 2 * (size_t)(nb + nd), n_res = (size_t)nb * nr * 2, n_ok = (size_t)nb * nr * 4, n_sample = 1 + 12;
    const size_t out_bytes = (n_ends + n_res + n_ok + n_sample) * 4;
    CUDA_TRY(h_open.reserve(in_bytes + out_bytes));
    DevBuf d_open;
    CUDA_TRY(d_open.reserve(in_bytes + out_bytes));
    uint8_t* h = (uint8_t*)h_open.p;
    BlockView* views = (BlockView*)(h + views_at);
    for (uint32_t i = 0; i < nb + nd; ++i) {
      const b2_cf_block& c = i < nb ? wblocks[i].c : dblocks[i - nb].c;
      views[i].keys = c.keys; views[i].koff = c.key_offs; views[i].vals = c.vals; views[i].voff = c.val_offs; views[i].n = c.n;
    }
    uint8_t* flat = h + flat_at;
    uint32_t* offs = (uint32_t*)(h + offs_at);
    offs[0] = 0;
    size_t at = 0;
    for (uint32_t r = 0; r < nr; ++r) {
      memcpy(flat + at, range_lo[r].data(), range_lo[r].size()); at += range_lo[r].size(); offs[2 * r + 1] = (uint32_t)at;
      memcpy(flat + at, range_hi[r].data(), range_hi[r].size()); at += range_hi[r].size(); offs[2 * r + 2] = (uint32_t)at;
    }
    uint8_t* d = (uint8_t*)d_open.p;
    uint32_t* d_out = (uint32_t*)(d + in_bytes);
    cudaError_t e = cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess)
      e = launch_open_probe((const BlockView*)(d + views_at), nb, nb + nd, d + flat_at, (const uint32_t*)(d + offs_at), nr, first_live_range, d_out + n_ends,
                            d_out + n_ends + n_res, d_out, d_out + n_ends + n_res + n_ok, stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h + in_bytes, d_out, out_bytes, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess && nd) e = dflt_views.reserve((size_t)nd * sizeof(BlockView));
    if (e == cudaSuccess && nd) e = cudaMemcpyAsync(dflt_views.p, d + views_at + (size_t)nb * sizeof(BlockView), (size_t)nd * sizeof(BlockView), cudaMemcpyDeviceToDevice, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return fail(B2_ERR_CUDA, std::string("opening the request's blocks: ") + cudaGetErrorString(e));
    const uint32_t* out = (const uint32_t*)(h + in_bytes);
    for (uint32_t i = 0; i < nb + nd; ++i) {
      SrcBlock& sb = i < nb ? wblocks[i] : dblocks[i - nb];
      sb.key_bytes = out[2 * i]; sb.val_bytes = out[2 * i + 1];
    }
    memcpy(res, out + n_ends, n_res * 4);
    memcpy(unit_ok, out + n_ends + n_res, n_ok * 4);
    v1_sample_len = out[n_ends + n_res + n_ok];
    memcpy(v1_sample, out + n_ends + n_res + n_ok + 1, sizeof(v1_sample));
    return B2_OK;
  }

  // lower_bound of every range bound in every CF_WRITE block
  int compute_units() {
    uint32_t nr = (uint32_t)range_lo.size(), nb = (uint32_t)wblocks.size();
    std::vector<uint32_t> res((size_t)nb * nr * 2), unit_ok((size_t)nb * nr * 4, 0);  // unit_ok: [ok, 12 prefix bytes] per (block, range)
    if (src_loc != B2_LOC_HOST) {
      int rc = probe_device_source(res.data(), unit_ok.data());
      if (rc) return rc;
    } else if (nr && nb) {
      for (uint32_t b = 0; b < nb; ++b)
        for (uint32_t q = 0; q < nr * 2; ++q) {
          const std::vector<uint8_t>& key = (q & 1) ? range_hi[q / 2] : range_lo[q / 2];
          const b2_cf_block& B = wblocks[b].c;
          uint32_t lo = 0, hi = B.n;
          while (lo < hi) {
            uint32_t mid = lo + (hi - lo) / 2;
            if (cmp_bytes_host(B.keys + B.key_offs[mid], B.key_offs[mid + 1] - B.key_offs[mid], key.data(), key.size()) < 0) lo = mid + 1; else hi = mid;
          }
          res[(size_t)b * nr * 2 + q] = lo;
        }
      for (uint32_t b = 0; b < nb; ++b)
        for (uint32_t r = 0; r < nr; ++r) {  // (same test as unit_prefix_kernel)
          const b2_cf_block& B = wblocks[b].c;
          uint32_t lo = res[(size_t)b * nr * 2 + 2 * r], hi = res[(size_t)b * nr * 2 + 2 * r + 1];
          if (hi <= lo) continue;
          const uint8_t *f = B.keys + B.key_offs[lo], *l = B.keys + B.key_offs[hi - 1];
          const bool ok = B.key_offs[lo + 1] - B.key_offs[lo] >= 12 && B.key_offs[hi] - B.key_offs[hi - 1] >= 12 && record_key_prefix_ok(f) && memcmp(f, l, 12) == 0;
          unit_ok[((size_t)b * nr + r) * 4] = ok;
          if (ok) memcpy(&unit_ok[((size_t)b * nr + r) * 4 + 1], f, 12);
        }
    }
    for (uint32_t r = first_live_range; r < nr; ++r)
      for (uint32_t b = 0; b < nb; ++b) {
        uint32_t lo = res[(size_t)b * nr * 2 + 2 * r], hi = res[(size_t)b * nr * 2 + 2 * r + 1];
        if (hi > lo) {
          const uint32_t* uo = &unit_ok[((size_t)b * nr + r) * 4];
          units.push_back(Unit{r, b, lo, hi, uo[0], {uo[1], uo[2], uo[3]}});
        }
      }
    return B2_OK;
  }

  // ---- block residency ----
  int acquire_block(uint32_t bi, BlockView* v) {
    const SrcBlock& sb = wblocks[bi];
    if (src_loc == B2_LOC_DEVICE) { v->keys = sb.c.keys; v->koff = sb.c.key_offs; v->vals = sb.c.vals; v->voff = sb.c.val_offs; v->n = sb.c.n; return B2_OK; }
    StageSlot* s = nullptr;
    for (auto& x : slots) if (x.block == (int)bi) s = &x;
    if (!s) {
      int rc = stage_block(bi, &s);
      if (rc) return rc;
    }
    CUDA_TRY(cudaStreamWaitEvent(stream, s->ready, 0));
    v->keys = (const uint8_t*)s->keys.p; v->koff = (const uint32_t*)s->koff.p; v->vals = (const uint8_t*)s->vals.p; v->voff = (const uint32_t*)s->voff.p; v->n = sb.c.n;
    return B2_OK;
  }
  int stage_block(uint32_t bi, StageSlot** out) {
    const SrcBlock& sb = wblocks[bi];
    // pick the slot not holding the previous block (two slots alternate)
    StageSlot* s = &slots[bi & 1];
    if (!copy_stream) CUDA_TRY(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
    if (!s->ready) { CUDA_TRY(cudaEventCreateWithFlags(&s->ready, cudaEventDisableTiming)); CUDA_TRY(cudaEventCreateWithFlags(&s->free_ev, cudaEventDisableTiming)); }
    if (s->free_recorded) CUDA_TRY(cudaStreamWaitEvent(copy_stream, s->free_ev, 0));
    size_t kb = (sb.key_bytes + 31) & ~15ull, vb = (sb.val_bytes + 31) & ~15ull, ob = ((size_t)sb.c.n + 1) * 4;
    if (s->keys.cap < kb || s->vals.cap < vb || s->koff.cap < ob || s->voff.cap < ob) {
      CUDA_TRY(cudaStreamSynchronize(stream));  // buffers may still be in use
      CUDA_TRY(s->keys.reserve(kb)); CUDA_TRY(s->vals.reserve(vb)); CUDA_TRY(s->koff.reserve(ob)); CUDA_TRY(s->voff.reserve(ob));
    }
    CUDA_TRY(cudaMemcpyAsync(s->keys.p, sb.c.keys, sb.key_bytes, cudaMemcpyHostToDevice, copy_stream));
    CUDA_TRY(cudaMemcpyAsync(s->vals.p, sb.c.vals, sb.val_bytes, cudaMemcpyHostToDevice, copy_stream));
    // the readable bytes past the heaps (word-wide loads of the last entries land there) are zero, as the padding contract of
    // device-resident blocks has them: nothing may depend on what an earlier request left in a recycled buffer
    CUDA_TRY(cudaMemsetAsync((uint8_t*)s->keys.p + sb.key_bytes, 0, kb - sb.key_bytes, copy_stream));
    CUDA_TRY(cudaMemsetAsync((uint8_t*)s->vals.p + sb.val_bytes, 0, vb - sb.val_bytes, copy_stream));
    CUDA_TRY(cudaMemcpyAsync(s->koff.p, sb.c.key_offs, ob, cudaMemcpyHostToDevice, copy_stream));
    CUDA_TRY(cudaMemcpyAsync(s->voff.p, sb.c.val_offs, ob, cudaMemcpyHostToDevice, copy_stream));
    CUDA_TRY(cudaEventRecord(s->ready, copy_stream));
    s->block = (int)bi;
    s->done = false;
    h2d_bytes += sb.key_bytes + sb.val_bytes + 2 * ob;
    *out = s;
    return B2_OK;
  }
  void release_block(uint32_t bi) {
    if (src_loc == B2_LOC_DEVICE) return;
    for (auto& x : slots)
      if (x.block == (int)bi) { cudaEventRecord(x.free_ev, stream); x.free_recorded = true; }
  }
  // Called when unit `unit_idx` has been launched completely.  Keeps the H2D stream busy: the next two distinct blocks
  // are put in flight, the second one into the slot of the block that just finished (its copy waits on free_ev, i.e. on
  // the kernels that still read the old block, not on the host).
  void prefetch_after(size_t unit_idx) {
    if (src_loc == B2_LOC_DEVICE) return;
    const uint32_t cur = units[unit_idx].block_idx;
    bool cur_needed = unit_idx + 1 < units.size() && units[unit_idx + 1].block_idx == cur;
    if (!cur_needed)
      for (auto& x : slots) if (x.block == (int)cur) x.done = true;
    int ahead = 0;
    for (size_t u = unit_idx + 1; u < units.size() && ahead < 2; ++u) {
      const uint32_t b = units[u].block_idx;
      if (b == cur && cur_needed) continue;
      StageSlot& sl = slots[b & 1];
      if (sl.block == (int)b) { if (!sl.done) { ++ahead; } continue; }
      if (sl.block >= 0 && !sl.done) break;  // that slot still feeds launches to come
      StageSlot* s;
      if (stage_block(b, &s)) break;
      ++ahead;
    }
  }
  uint64_t h2d_bytes = 0;

  int init_device_state() {
    CUDA_TRY(ctr_buf.reserve(sizeof(Counters)));
    CUDA_TRY(h_ctr.reserve(2 * sizeof(Counters)));
    memset(&good_ctr, 0, sizeof(good_ctr));
    good_ctr.err = ~0ull; good_ctr.first_row = ~0ull;
    int rc = upload_counters(good_ctr);
    if (rc) return rc;
    CUDA_TRY(range_rows.reserve(std::max<size_t>(1, range_raw_lo.size()) * 8));
    CUDA_TRY(cudaMemsetAsync(range_rows.p, 0, std::max<size_t>(1, range_raw_lo.size()) * 8, stream));
    range_rows_taken.assign(range_raw_lo.size(), 0);
    return B2_OK;
  }
  // h_ctr holds two Counters: [0] receives read_counters, [1] is the pinned source of this upload.  The source may only be
  // rewritten once the previous upload has been waited for (read_counters), else the copy could read the new bytes:
  // a second upload before that is a bug in the engine and fails the request instead of racing.
  bool ctr_upload_in_flight = false;
  int upload_counters(const Counters& c) {
    if (ctr_upload_in_flight) return fail(B2_ERR_CUDA, "internal: counters uploaded again before the previous upload was waited for");
    Counters* src = (Counters*)h_ctr.p + 1;
    *src = c;
    CUDA_TRY(cudaMemcpyAsync(ctr_buf.p, src, sizeof(Counters), cudaMemcpyHostToDevice, stream));
    ctr_upload_in_flight = true;
    return B2_OK;
  }
  int read_counters(Counters* c) {
    CUDA_TRY(cudaMemcpyAsync(h_ctr.p, ctr_buf.p, sizeof(Counters), cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    ctr_upload_in_flight = false;
    memcpy(c, h_ctr.p, sizeof(Counters));
    harvest_kernel_times();
    return B2_OK;
  }
  // CUDA events bracketing every launch of the dominant kernel (roofline numerator / denominator in bench.py)
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> kev;
  size_t kev_used = 0;
  cudaEvent_t batch_ev[2] = {nullptr, nullptr};  // brackets each next_batch (time_processed_ns)
  void kernel_begin() {
    if (kev_used == kev.size()) kev.push_back({event_pool().get(), event_pool().get()});
    cudaEventRecord(kev[kev_used].first, stream);
  }
  void kernel_end() { cudaEventRecord(kev[kev_used].second, stream); ++kev_used; stats.kernel_launches++; }
  void harvest_kernel_times() {  // call after a stream synchronize
    for (size_t i = 0; i < kev_used; ++i) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, kev[i].first, kev[i].second) == cudaSuccess) stats.kernel_time_ns += (uint64_t)(ms * 1e6);
    }
    kev_used = 0;
  }
  void fill_stats(const Counters& c) {
    last_row_seen = c.last_row; first_row_seen = c.first_row;
    stats.write_entries_scanned = entries_scanned;
    stats.write_processed_keys = c.processed_keys;
    stats.processed_size = c.processed_size;
    stats.default_lookups = c.default_lookups;
    stats.lock_processed_keys = lock_keys_seen;
    stats.met_newer_ts_data = check_newer ? ((c.met_newer || saw_lock) ? 1 : 0) : -1;
    stats.h2d_bytes = h2d_bytes; stats.d2h_bytes = d2h_bytes;
    met_newer_any = c.met_newer || saw_lock;
    warnings_total = c.warn_div0;
  }
  bool met_newer_any = false;

  // the failing row a scan in this direction meets first
  unsigned long long first_error(const Counters& c) const { return cp.desc ? c.err_max : c.err; }
  int device_error(const Counters& c) {
    if (c.err == ~0ull) return B2_OK;
    const unsigned long long e = first_error(c);
    int status, mysql;
    const char* m = dev_err_message((int)(e & 0xff), &status, &mysql);
    return fail(status, m, mysql, e >> 8);
  }

  // shared-memory staging: capacities from the block's average entry size (+30 %), stages placed after `mode_bytes`
  size_t setup_staging(ScanArgs* a, const SrcBlock& sb, size_t mode_bytes) {
    uint32_t n = std::max<uint32_t>(1, sb.c.n), ents = scan_stage_entries();
    // stage capacity = average bytes of a tile's entries + slack; the slack shrinks (30 % .. 6 %) while that lets two
    // CTAs share an SM's shared memory.  A tile that does not fit is read from HBM directly.
    auto cap = [&](uint64_t total, uint64_t pct) { uint64_t c = (total * ents / n) * pct / 100 + 256; c = (c + 15) & ~15ull; return (uint32_t)std::min<uint64_t>(c, 72 * 1024); };
    a->stage_off = (uint32_t)((mode_bytes + 15) & ~15ull);
    const size_t two_per_sm = (233472 / 2) - 1024 - 512;  // H100 SM shared memory (228 KB) / 2 - per-CTA reserve - static
    size_t total = 0;
    for (uint64_t pct : {130, 120, 112, 106}) {
      a->stage_key_cap = cap(sb.key_bytes, pct); a->stage_val_cap = cap(sb.val_bytes, pct);
      total = a->stage_off + scan_stage_bytes(a->stage_key_cap, a->stage_val_cap);
      if (total <= two_per_sm) break;
    }
    if (total > two_per_sm) {
      a->stage_key_cap = cap(sb.key_bytes, 130); a->stage_val_cap = cap(sb.val_bytes, 130);
      total = a->stage_off + scan_stage_bytes(a->stage_key_cap, a->stage_val_cap);
    }
    if (total > 200 * 1024) { a->staging = 0; a->stage_key_cap = a->stage_val_cap = 0; return mode_bytes; }
    a->staging = 1;
    return total;
  }
  // ---- order-free pipelines: the lean kernel (fast_kernel.cuh) over a unit, then scan_body in list mode over the runs it
  // handed over (their first entries, appended on the device; the count never visits the host) ----
  DevBuf slow_list, slow_cnt;
  DevBuf const_pool;  // bytes constants of the plan (CompiledPlan::pool)
  bool fast_kernel_covers() const { return cp.dev.mode == PM_CHECKSUM || plan_has_fast_kernel(cp.dev); }
  // `a`: the unit's arguments (c_lo / c_hi set, mode pointers set).  general_smem_mode / fast_smem_mode: bytes of mode state
  // in front of the stages; fast_slots: CTA table slots of the lean aggregation kernel.
  int launch_unit(const ScanArgs& a0, const Unit& u, bool fast, size_t general_smem_mode, size_t fast_smem_mode, uint32_t fast_slots, int* general_grid_out,
                  int* fast_grid_out) {
    const int mode = scan_kernel_mode(cp.dev);
    if (!fast) {
      ScanArgs a = a0;
      size_t tot = setup_staging(&a, wblocks[u.block_idx], general_smem_mode);
      int grid = scan_grid_for(mode, tot);
      if (general_grid_out && *general_grid_out > 0) grid = std::min(grid, *general_grid_out);
      kernel_begin();
      CUDA_TRY(scan_launch(a, grid, tot));
      kernel_end();
      if (general_grid_out) *general_grid_out = grid;
      if (fast_grid_out) *fast_grid_out = 0;
      return B2_OK;
    }
    CUDA_TRY(slow_list.reserve_on(stream, (size_t)(u.e_hi - u.e_lo) * 4 + 16));
    CUDA_TRY(slow_cnt.reserve_on(stream, 16));
    CUDA_TRY(cudaMemsetAsync(slow_cnt.p, 0, 4, stream));
    ScanArgs f = a0;
    f.slow_list = (unsigned int*)slow_list.p; f.slow_count = (unsigned int*)slow_cnt.p;
    f.smem_slots = fast_slots;
    size_t ftot = setup_staging(&f, wblocks[u.block_idx], fast_smem_mode);
    const JitKernel* jk = jit_ready();
    if (jk && !jk->fn_fast) jk = nullptr;
    int fgrid = jk ? jit_max_blocks_per_sm(jk, ftot, true) * scan_num_sms() : fast_max_grid(cp.dev.mode, ftot);
    if (fast_grid_out && *fast_grid_out > 0) fgrid = std::min(fgrid, *fast_grid_out);
    kernel_begin();
    if (f.staging) {
      if (jk) { stats.jit_launches++; CUDA_TRY(jit_launch(jk, f, fgrid, ftot, stream, true)); }
      else CUDA_TRY(launch_fast(cp.dev, f, fgrid, ftot, stream));
    } else {  // no staging possible (huge entries): everything goes through the general kernel
      fast = false;
    }
    ScanArgs g = a0;
    size_t gtot = general_smem_mode;
    if (fast) {
      g.slow_list = f.slow_list; g.slow_count = f.slow_count; g.list_mode = 1;
      g.staging = 0; g.stage_off = 0; g.stage_key_cap = g.stage_val_cap = 0;
    } else {
      gtot = setup_staging(&g, wblocks[u.block_idx], general_smem_mode);
    }
    int ggrid = scan_grid_for(mode, gtot);
    if (general_grid_out && *general_grid_out > 0) ggrid = std::min(ggrid, *general_grid_out);
    if (cp.dev.mode == PM_TOPN && fast) {  // the two kernels leave their per-CTA lists side by side
      g.topn.items = a0.topn.items + (size_t)fgrid * a0.topn.stride; g.topn.counts = a0.topn.counts + fgrid;
    }
    CUDA_TRY(scan_launch(g, ggrid, gtot));
    kernel_end();
    stats.kernel_launches += fast ? 1 : 0;
    if (general_grid_out) *general_grid_out = ggrid;
    if (fast_grid_out) *fast_grid_out = fast ? fgrid : 0;
    return B2_OK;
  }

  ScanArgs base_args(const Unit& u, const BlockView& v) {
    ScanArgs a;
    memset(&a, 0, sizeof(a));
    a.blk = v;
    a.dflt.blocks = (const BlockView*)dflt_views.p; a.dflt.n_blocks = (uint32_t)dblocks.size();
    a.e_lo = u.e_lo; a.e_hi = u.e_hi;
    a.entry_base = wblocks[u.block_idx].entry_base;
    a.ctr = ctr();
    a.read_ts = cp.dev.read_ts; a.isolation = cp.dev.isolation;
    a.fast_ok = u.fast_ok;
    a.desc = cp.desc ? 1u : 0u;
    memcpy(a.imms, cp.imms, sizeof(a.imms));
    a.limit = cp.dev.limit;
    a.range_rows = range_rows.p ? (unsigned long long*)range_rows.p + u.range_idx : nullptr;
    return a;
  }

  // ---- PM_SCAN: up to `scan_rows` CF_WRITE entries per call, appended in key order into one set of columns ----
  // A forward scan consumes the units first to last, each from its lower end.  The rows of a backward scan (TableScan.desc;
  // scan_executor.rs:89-101, backward.rs:78-225) are the rows of the forward scan in reverse order (the MVCC rule per key
  // is the same), so it consumes the units last to first, each from its upper end, runs the forward kernel and reverses
  // the rows on the device.  A launch only emits runs that *start* inside it, and its walks may go past its upper end, so
  // a version run is never split.
  // output columns (8-byte cells) for `rows` rows in `data` / `bitmap`, their non-NULL bitmaps set to ones
  int reserve_out(DevBuf* data, DevBuf* bitmap, uint64_t* cap_now, uint64_t rows) {
    const size_t n_out = cp.dev.n_out;
    const uint64_t cap = std::max<uint64_t>(64, (rows + 63) & ~63ull);
    if (cap > *cap_now) {
      CUDA_TRY(cudaStreamSynchronize(stream));
      CUDA_TRY(data->reserve(cap * 8 * n_out)); CUDA_TRY(bitmap->reserve(cap / 8 * n_out));
      *cap_now = cap;
    }
    CUDA_TRY(cudaMemsetAsync(bitmap->p, 0xff, *cap_now / 8 * n_out, stream));
    return B2_OK;
  }
  // one launch over the entries [c_lo, c_hi) of unit `u`, appending to the output columns; the walks of the chunk's last
  // runs stop at e_hi
  int scan_chunk(const Unit& u, uint32_t c_lo, uint32_t c_hi, uint32_t e_hi) {
    const uint32_t n_tiles = (c_hi - c_lo + TILE - 1) / TILE;
    CUDA_TRY(status_buf.reserve_on(stream, ((size_t)n_tiles + 1) * 8));
    CUDA_TRY(cudaMemsetAsync(status_buf.p, 0, ((size_t)n_tiles + 1) * 8, stream));
    BlockView v;
    int rc = acquire_block(u.block_idx, &v);
    if (rc) return rc;
    ScanArgs a = base_args(u, v);
    a.c_lo = c_lo; a.c_hi = c_hi; a.e_hi = e_hi;
    a.tile_status = (unsigned long long*)status_buf.p;
    a.out_data = (unsigned long long*)out_data.p; a.out_bitmap = (unsigned long long*)out_bitmap.p;
    a.out_cap = out_cap;
    const size_t smem = setup_staging(&a, wblocks[u.block_idx], scan_out_stage_bytes());
    a.out_stage_off = 0;
    const int grid = scan_grid_for(scan_kernel_mode(cp.dev), smem);
    kernel_begin();
    CUDA_TRY(scan_launch(a, grid, smem));
    kernel_end();
    if (cp.dev.n_raw) { rc = raw_materialise(a, c_hi - c_lo); if (rc) return rc; }
    release_block(u.block_idx);
    stats.num_iterations++;
    return B2_OK;
  }
  // BatchLimitExecutor (limit_executor.rs:55-80): a plain scan needs at most `remaining` more rows, so do not read far
  // past them; with a selection in between the batch size is the caller's.  Returns the batch's entry budget.
  uint64_t begin_scan_batch(uint64_t scan_rows) {
    cols.clear();
    uint64_t budget = std::max<uint64_t>(1, std::min<uint64_t>(scan_rows, 1ull << 31));
    if (cp.scan_limit == ~0ull) return budget;
    if (limit_remaining == ~0ull) limit_remaining = cp.scan_limit;
    if (limit_remaining == 0) drained = true;
    if (cp.dev.n_conds == 0) budget = std::min<uint64_t>(budget, std::max<uint64_t>(4096, limit_remaining * 2));
    return budget;
  }
  // the rows of the batch that the Limit still takes
  uint64_t limit_take(uint64_t produced) {
    if (cp.scan_limit == ~0ull) return produced;
    if (produced < limit_remaining) { limit_remaining -= produced; return produced; }
    produced = limit_remaining;
    limit_remaining = 0;
    drained = true;
    return produced;
  }

  // the unit a scan consumes after unit `u`; units.size() = none
  size_t unit_after(size_t u) const { return !cp.desc ? u + 1 : u ? u - 1 : units.size(); }
  void enter_unit(size_t u) {
    cur_unit = u;
    if (u < units.size()) { cur_lo = units[u].e_lo; cur_hi = units[u].e_hi; }
  }
  // unit `u` is the last one of its range in scan order (the highest unit of a forward range, the lowest of a backward
  // one) and that range ends in a conflicting lock
  bool ends_locked_range(size_t u) const {
    const size_t next = unit_after(u);
    return (next >= units.size() || units[next].range_idx != units[u].range_idx) && range_lock_err[units[u].range_idx];
  }

  // one launch of a pass: the entries [c_lo, c_hi) of unit `unit`; the walks of its last runs stop at `walk_end`
  struct Piece { size_t unit; uint32_t c_lo, c_hi, walk_end; };
  // The pieces of the next pass, in ascending key order, taken from the cursor.  `bound` (a global entry index, ~0 = none)
  // is the failing row an earlier run of this pass met: a forward pass stops before it, a backward pass starts after it.
  std::vector<Piece> plan_pass(uint64_t budget, uint64_t bound) const {
    std::vector<Piece> ps;
    if (cp.desc) {  // one piece of at most `budget` entries from the top of the current unit
      const Unit& u = units[cur_unit];
      uint64_t c_lo = (uint64_t)cur_hi - cur_lo > budget ? cur_hi - budget : cur_lo;
      if (bound != ~0ull) c_lo = std::max<uint64_t>(c_lo, bound - wblocks[u.block_idx].entry_base + 1);
      if (c_lo < cur_hi) ps.push_back(Piece{cur_unit, (uint32_t)c_lo, cur_hi, u.e_hi});
      return ps;
    }
    // forward: across units up to the budget; a range that ends in a conflicting lock ends the pass
    for (size_t u = cur_unit; budget && u < units.size(); ++u) {
      const Unit& U = units[u];
      const uint64_t base = wblocks[U.block_idx].entry_base;
      const uint32_t c_lo = u == cur_unit ? cur_lo : U.e_lo;
      uint32_t c_hi = (uint32_t)std::min<uint64_t>(U.e_hi, (uint64_t)c_lo + budget);
      const bool cut = bound != ~0ull && base + c_hi > bound;
      if (cut) c_hi = bound > base + c_lo ? (uint32_t)(bound - base) : c_lo;
      // (the failing entry is a run start: nothing before it can reach past it)
      if (c_hi > c_lo) { ps.push_back(Piece{u, c_lo, c_hi, cut ? c_hi : U.e_hi}); budget -= c_hi - c_lo; }
      if (c_hi < U.e_hi || ends_locked_range(u)) break;
    }
    return ps;
  }

  // One pass: the pieces, each launch appending behind the rows of the launches before it (out_rows -> out_base on the
  // device), then a single host sync for the counters.  The cursor moves past every piece launched.  *lock_range: the
  // range whose conflicting lock the pass reached, or -1.
  int run_scan_pass(uint64_t budget, uint64_t bound, int* lock_range, Counters* c) {
    const std::vector<Piece> ps = plan_pass(budget, bound);
    uint64_t rows = 0, vb = 0;
    int last_blk = -1;
    for (const Piece& p : ps) {
      rows += p.c_hi - p.c_lo;
      const int b = (int)units[p.unit].block_idx;
      if (b != last_blk) { vb += wblocks[b].val_bytes; last_blk = b; }
    }
    int rc = reserve_out(&out_data, &out_bitmap, &out_cap, rows);
    if (rc) return rc;
    if (cp.dev.n_raw) {
      // every byte a cell reference of this pass can point at: the value heaps of the blocks it touches (+ CF_DEFAULT)
      for (const SrcBlock& d : dblocks) vb += d.val_bytes;
      CUDA_TRY(cudaStreamSynchronize(stream));
      rc = raw_prepare(out_cap, vb);
      if (rc) return rc;
    }
    // keep request-level statistics, reset the per-pass row counters
    CUDA_TRY(cudaMemsetAsync(&ctr()->out_rows, 0, 8, stream));
    CUDA_TRY(cudaMemsetAsync(&ctr()->out_base, 0, 8, stream));
    *lock_range = -1;
    for (const Piece& p : ps) {
      if (deadline_exceeded()) break;
      rc = scan_chunk(units[p.unit], p.c_lo, p.c_hi, p.walk_end);
      if (rc) return rc;
      CUDA_TRY(cudaMemcpyAsync(&ctr()->out_base, &ctr()->out_rows, 8, cudaMemcpyDeviceToDevice, stream));
      entries_scanned += p.c_hi - p.c_lo;
      if (cp.desc) cur_hi = p.c_lo; else cur_lo = p.c_hi;
      if (cur_lo < cur_hi) continue;
      // the unit is done.  prefetch_after stages the blocks of the units after it, which only a forward scan reads next.
      if (!cp.desc) prefetch_after(p.unit);
      if (ends_locked_range(p.unit)) *lock_range = (int)units[p.unit].range_idx;
      enter_unit(unit_after(p.unit));
    }
    return read_counters(c);
  }

  Counters good_ctr{};  // device counters after the last pass that met no failing row (first: what init_device_state uploads)
  DevBuf range_rows_prev;
  DevBuf rev_data, rev_bitmap;
  uint64_t rev_cap = 0;
  int next_scan_batch(uint64_t scan_rows, b2_batch* out) {
    const uint64_t budget = begin_scan_batch(scan_rows);
    const bool limited = cp.scan_limit != ~0ull;
    const size_t rr_bytes = std::max<size_t>(1, range_raw_lo.size()) * 8;
    Counters c = good_ctr;
    uint64_t written = 0;  // rows the last pass wrote
    while (!drained && !failed && written == 0) {
      if (cur_unit >= units.size()) { drained = true; break; }
      // what the pass starts from, restored if it meets a failing row
      const size_t save_unit = cur_unit;
      const uint32_t save_lo = cur_lo, save_hi = cur_hi;
      const uint64_t save_scanned = entries_scanned;
      CUDA_TRY(range_rows_prev.reserve_on(stream, rr_bytes));
      CUDA_TRY(cudaMemcpyAsync(range_rows_prev.p, range_rows.p, rr_bytes, cudaMemcpyDeviceToDevice, stream));
      int lock_r;
      int rc = run_scan_pass(budget, ~0ull, &lock_r, &c);
      if (rc) return rc;
      written = c.out_rows;
      if (c.err != ~0ull) {
        // the rows the scan meets before the failing row stay valid (interface.rs:229-235): redo the pass up to that row
        // from the state it started from, so nothing is counted twice and the statistics describe exactly the rows that
        // were returned (the reference's partial-result semantics)
        const Counters bad = c;
        cur_unit = save_unit; cur_lo = save_lo; cur_hi = save_hi; entries_scanned = save_scanned;
        rc = upload_counters(good_ctr);
        if (rc) return rc;
        CUDA_TRY(cudaMemcpyAsync(range_rows.p, range_rows_prev.p, rr_bytes, cudaMemcpyDeviceToDevice, stream));
        rc = run_scan_pass(budget, first_error(bad) >> 8, &lock_r, &c);
        if (rc) return rc;
        written = c.err == ~0ull ? c.out_rows : 0;
        // (the reference never reaches a failing row that lies beyond the rows a Limit still wants)
        if (!(limited && written >= limit_remaining)) device_error(bad);
        drained = true;
        break;
      }
      good_ctr = c;
      if (lock_r >= 0) {
        if (!(limited && written >= limit_remaining)) lock_failure((uint32_t)lock_r);
        drained = true;
        break;
      }
    }
    fill_stats(c);
    uint64_t produced = limit_take(written);
    if (!failed && cur_unit >= units.size()) {
      drained = true;
      if (!(limited && limit_remaining == 0)) check_trailing_lock();
    }
    if (cp.dev.n_raw && produced && !raw_outs.empty() && raw_collect() != B2_OK) produced = 0;
    if (!cp.desc) return publish_scan_columns(produced, out);
    // the kernel wrote the rows in ascending key order.  (A Limit may have cut them: the first `produced` rows of the
    // reversed order are the last ones the kernel wrote.)
    if (produced) {
      int rc = reserve_out(&rev_data, &rev_bitmap, &rev_cap, produced);
      if (rc) return rc;
      CUDA_TRY(launch_reverse_rows((const unsigned long long*)out_data.p, (const unsigned long long*)out_bitmap.p, out_cap, (unsigned long long*)rev_data.p,
                                   (unsigned long long*)rev_bitmap.p, rev_cap, written, produced, (uint32_t)cp.dev.n_out, stream));
      stats.kernel_launches++;
    }
    return publish_scan_columns(produced, out, &rev_data, &rev_bitmap, rev_cap);
  }

  // bytes / json / decimal output columns (kernels.cu raw_*): per column an offsets array + byte heap (or decimal structs),
  // a device-resident heap cursor, one error word
  struct RawOut { int out_idx; int kind; DevBuf offs, heap; uint64_t heap_cap = 0; uint64_t used = 0; };
  std::vector<RawOut> raw_outs;
  DevBuf raw_state, raw_sums;   // raw_state: [n_raw] heap cursors, then the error word
  HostBuf h_raw, h_raw_out;
  uint64_t raw_cap_rows = 0;
  int raw_prepare(uint64_t cap_rows, uint64_t value_bytes) {
    if (raw_outs.empty())
      for (int k = 0; k < cp.dev.n_out; ++k) {
        const int ck = cp.dev.cols[cp.dev.out_cols[k]].kind;
        if (!cp.dev.n_proj && ck_is_ref(ck)) { raw_outs.emplace_back(); raw_outs.back().out_idx = k; raw_outs.back().kind = ck; }
      }
    const size_t n = raw_outs.size();
    for (RawOut& r : raw_outs) {
      if (r.kind == CK_DEC) { CUDA_TRY(r.heap.reserve(cap_rows * 40)); r.heap_cap = cap_rows * 40; }
      else { CUDA_TRY(r.offs.reserve((cap_rows + 1) * 8)); CUDA_TRY(r.heap.reserve(std::max<uint64_t>(value_bytes, 16))); r.heap_cap = value_bytes; }
    }
    CUDA_TRY(raw_state.reserve_on(stream, (n + 1) * 8));
    CUDA_TRY(cudaMemsetAsync(raw_state.p, 0, (n + 1) * 8, stream));
    CUDA_TRY(raw_sums.reserve(std::max<size_t>(1, n) * ((cap_rows + 1023) / 1024 + 1) * 8));
    raw_cap_rows = cap_rows;
    return B2_OK;
  }
  // after a scan launch: resolve the cell references of the rows it appended ([out_base, out_rows) on the device)
  int raw_materialise(const ScanArgs& a, uint64_t max_rows) {
    RawArgs R;
    memset(&R, 0, sizeof(R));
    for (size_t i = 0; i < raw_outs.size(); ++i) {
      RawOut& r = raw_outs[i];
      R.col[i].cells = a.out_data + (size_t)r.out_idx * a.out_cap;
      R.col[i].offsets = (long long*)r.offs.p; R.col[i].heap = (unsigned char*)r.heap.p;
      R.col[i].heap_used = (unsigned long long*)raw_state.p + i; R.col[i].heap_cap = r.heap_cap;
      if (r.kind == CK_DEC) R.dec_idx[R.n_dec++] = (unsigned char)i; else R.var_idx[R.n_var++] = (unsigned char)i;
    }
    R.row_lo = &ctr()->out_base; R.row_hi = &ctr()->out_rows;
    R.sums = (unsigned long long*)raw_sums.p; R.sums_stride = (raw_cap_rows + 1023) / 1024 + 1;
    R.err = (unsigned int*)((unsigned long long*)raw_state.p + raw_outs.size());
    CUDA_TRY(launch_raw_materialise(R, max_rows, stream));
    stats.kernel_launches += (R.n_var ? 3 : 0) + (R.n_dec ? 1 : 0);
    return B2_OK;
  }
  // after the pass's counters are on the host: heap sizes and the error word
  int raw_collect() {
    const size_t n = raw_outs.size();
    CUDA_TRY(h_raw.reserve((n + 1) * 8));
    CUDA_TRY(cudaMemcpyAsync(h_raw.p, raw_state.p, (n + 1) * 8, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    const uint64_t* h = (const uint64_t*)h_raw.p;
    for (size_t i = 0; i < n; ++i) raw_outs[i].used = h[i];
    if ((uint32_t)h[n]) {
      failed = true;
      last_err.status = B2_ERR_CORRUPTED; last_err.mysql_code = 0; last_err.entry_index = ~0ull;
      snprintf(last_err.message, sizeof(last_err.message), "%s", (uint32_t)h[n] == 1 ? "decimal cell does not decode (decimal.rs read_decimal)" : "bytes column heap overflow");
      return last_err.status;
    }
    return B2_OK;
  }
  uint64_t limit_remaining = ~0ull;

  void lock_failure(uint32_t r) {
    fail(range_lock_err[r], "key is locked, lock_version=" + std::to_string(range_lock_ts[r]));
  }
  // a conflicting lock in a range that produced no unit still fails the request
  void check_trailing_lock() {
    if (failed) return;
    for (size_t r = 0; r < range_lock_err.size(); ++r)
      if (range_lock_err[r]) { lock_failure((uint32_t)r); return; }
  }

  // Fixed-width output columns (scan, aggregation and TopN results), one per output offset: fills `cols` and `last_dev`.
  // Host output copies each column's `n_rows` cells of `esz` bytes and `bm_bytes` of its bitmap into pinned memory.
  struct FixedCol { const void* data; const void* bitmap; size_t esz, bm_bytes; };
  int publish_fixed(const std::vector<FixedCol>& fc, uint64_t n_rows) {
    const bool to_host = out_loc == B2_LOC_HOST && n_rows;
    cols.assign(fc.size(), b2_column{});
    last_dev.assign(fc.size(), DevColRef{});
    last_rows = n_rows;
    if (to_host) {
      size_t total = 0;
      for (const FixedCol& f : fc) total += n_rows * f.esz + f.bm_bytes;
      CUDA_TRY(h_out.reserve(total));
    }
    uint8_t* hp = (uint8_t*)h_out.p;
    for (size_t i = 0; i < fc.size(); ++i) {
      const FixedCol& f = fc[i];
      const OutCol& oc = cp.schema[cp.output_offsets[i]];
      cols[i].kind = oc.kind; cols[i].field_tp = oc.field_tp; cols[i].field_flag = oc.field_flag; cols[i].len = n_rows;
      last_dev[i] = DevColRef{f.data, (const unsigned long long*)f.bitmap, oc.kind, oc.field_tp, oc.field_flag};
      if (to_host) {
        const size_t bytes = n_rows * f.esz;
        CUDA_TRY(cudaMemcpyAsync(hp, f.data, bytes, cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaMemcpyAsync(hp + bytes, f.bitmap, f.bm_bytes, cudaMemcpyDeviceToHost, stream));
        cols[i].data = hp; cols[i].null_bitmap = (const uint64_t*)(hp + bytes);
        hp += bytes + f.bm_bytes;
        d2h_bytes += bytes + f.bm_bytes;
      } else if (n_rows) {
        cols[i].data = f.data; cols[i].null_bitmap = (const uint64_t*)f.bitmap;
      }
    }
    if (to_host) CUDA_TRY(cudaStreamSynchronize(stream));
    return B2_OK;
  }

  int publish_scan_columns(uint64_t n_rows, b2_batch* out, const DevBuf* src_data = nullptr, const DevBuf* src_bitmap = nullptr, uint64_t src_cap = 0) {
    const size_t n_out = cp.dev.n_out;
    const uint8_t* data = (const uint8_t*)(src_data ? src_data->p : out_data.p);
    const uint8_t* bm = (const uint8_t*)(src_bitmap ? src_bitmap->p : out_bitmap.p);
    const uint64_t out_cap = src_data ? src_cap : this->out_cap;
    std::vector<FixedCol> fc(n_out);
    for (size_t k = 0; k < n_out; ++k) fc[k] = FixedCol{data + k * out_cap * 8, bm + k * (out_cap / 8), 8, ((n_rows + 63) / 64) * 8};
    int rc = publish_fixed(fc, n_rows);
    if (rc) return rc;
    // bytes / json / decimal columns: the 8-byte cells above are references; the column itself is the heap the raw_* kernels filled
    if (cp.dev.n_raw && n_rows) {
      size_t need = 0;
      for (RawOut& r : raw_outs) {
        if (r.kind != CK_DEC) r.used = 0;  // (rows beyond n_rows were materialised too: the heap in use ends at offsets[n_rows])
        need += r.kind == CK_DEC ? n_rows * 40 : (n_rows + 1) * 8;
      }
      std::vector<long long> ends(raw_outs.size(), 0);
      for (size_t i = 0; i < raw_outs.size(); ++i)
        if (raw_outs[i].kind != CK_DEC) CUDA_TRY(cudaMemcpyAsync(&ends[i], (const long long*)raw_outs[i].offs.p + n_rows, 8, cudaMemcpyDeviceToHost, stream));
      CUDA_TRY(cudaStreamSynchronize(stream));
      for (size_t i = 0; i < raw_outs.size(); ++i) if (raw_outs[i].kind != CK_DEC) { raw_outs[i].used = (uint64_t)ends[i]; need += (raw_outs[i].used + 15) & ~15ull; }
      uint8_t* hp = nullptr;
      if (out_loc == B2_LOC_HOST) { CUDA_TRY(h_raw_out.reserve(need + 64)); hp = (uint8_t*)h_raw_out.p; }
      for (RawOut& r : raw_outs) {
        const size_t k = (size_t)r.out_idx;
        DevColRef& d = last_dev[k];
        d.raw = true; d.data = r.heap.p;
        if (r.kind != CK_DEC) { d.offsets = (const long long*)r.offs.p; d.heap_len = r.used; }
        if (out_loc == B2_LOC_HOST) {
          if (r.kind == CK_DEC) {
            CUDA_TRY(cudaMemcpyAsync(hp, r.heap.p, n_rows * 40, cudaMemcpyDeviceToHost, stream));
            cols[k].data = hp; hp += (n_rows * 40 + 15) & ~15ull; d2h_bytes += n_rows * 40;
          } else {
            CUDA_TRY(cudaMemcpyAsync(hp, r.offs.p, (n_rows + 1) * 8, cudaMemcpyDeviceToHost, stream));
            cols[k].offsets = (const int64_t*)hp; hp += (n_rows + 1) * 8;
            if (r.used) CUDA_TRY(cudaMemcpyAsync(hp, r.heap.p, r.used, cudaMemcpyDeviceToHost, stream));
            cols[k].data = hp; hp += (r.used + 15) & ~15ull; d2h_bytes += (n_rows + 1) * 8 + r.used;
          }
        } else {
          cols[k].data = r.heap.p;
          cols[k].offsets = r.kind == CK_DEC ? nullptr : (const int64_t*)r.offs.p;
        }
      }
      if (out_loc == B2_LOC_HOST) CUDA_TRY(cudaStreamSynchronize(stream));
    }
    out->columns = cols.data(); out->n_columns = (uint32_t)n_out; out->n_rows = n_rows;
    out->is_drained = drained ? B2_DRAIN_DRAINED : B2_DRAIN_REMAIN;
    stats.num_produced_rows += n_rows;
    return failed ? last_err.status : B2_OK;
  }

  // ---- RangesScanner::take_scanned_range (tidb_query_common/src/storage/scanner.rs:204-229), forward scans ----
  // [lower, upper): lower = where the previous take ended (first take: the first range's start); upper = the last row
  // the MVCC scan returned so far + 0x00 (update_scanned_range_from_scanned_row :290-300), or the last range's end once
  // drained.  Raw keys, like b2_key_range.
  int entry_raw_key(uint64_t global_entry, std::vector<uint8_t>* raw) {
    for (const SrcBlock& b : wblocks) {
      if (global_entry < b.entry_base || global_entry >= b.entry_base + b.c.n) continue;
      uint32_t e = (uint32_t)(global_entry - b.entry_base), off[2];
      std::vector<uint8_t> enc;
      if (src_loc == B2_LOC_HOST) { off[0] = b.c.key_offs[e]; off[1] = b.c.key_offs[e + 1]; enc.assign(b.c.keys + off[0], b.c.keys + off[1]); }
      else {
        CUDA_TRY(cudaMemcpy(off, b.c.key_offs + e, 8, cudaMemcpyDeviceToHost));
        enc.resize(off[1] - off[0]);
        CUDA_TRY(cudaMemcpy(enc.data(), b.c.keys + off[0], enc.size(), cudaMemcpyDeviceToHost));
      }
      if (enc.size() < 8) return fail(B2_ERR_CORRUPTED, "CF_WRITE key without timestamp");
      int rl = raw_key_len(enc.data(), (uint32_t)enc.size() - 8);
      if (rl < 0) return fail(B2_ERR_CORRUPTED, "bad memcomparable key");
      raw->clear();
      for (int j = 0; j < rl; ++j) raw->push_back((uint8_t)raw_at(enc.data(), (uint32_t)j));
      return B2_OK;
    }
    return fail(B2_ERR_INVALID_ARG, "entry index outside every block");
  }
  std::vector<uint8_t> taken_lo, taken_hi;
  uint64_t first_row_taken = ~0ull;
  int take_scanned_range(const uint8_t** lo, uint32_t* lo_len, const uint8_t** hi, uint32_t* hi_len) {
    if (cp.desc) {
      // scanner.rs:204-229, scan_backward_in_range: [key of the last (smallest) row returned, where the previous take
      // ended); first take: up to the last range's end; once drained: down to the first range's start
      if (working_begin.empty() && !range_raw_hi.empty()) working_begin = range_raw_hi.back();
      taken_hi = working_begin;
      if (drained && !range_raw_lo.empty()) taken_lo = range_raw_lo[0];
      else if (first_row_seen != ~0ull && first_row_seen < first_row_taken) {
        int rc = entry_raw_key(first_row_seen, &taken_lo);
        if (rc) return rc;
      } else taken_lo = taken_hi;
      first_row_taken = first_row_seen;
      working_begin = taken_lo;
      *lo = taken_lo.data(); *lo_len = (uint32_t)taken_lo.size(); *hi = taken_hi.data(); *hi_len = (uint32_t)taken_hi.size();
      return B2_OK;
    }
    if (working_begin.empty() && !range_raw_lo.empty()) working_begin = range_raw_lo[0];
    taken_lo = working_begin;
    if (drained && !range_raw_hi.empty()) taken_hi = range_raw_hi.back();
    else if (last_row_seen > last_row_taken) {
      int rc = entry_raw_key(last_row_seen - 1, &taken_hi);
      if (rc) return rc;
      taken_hi.push_back(0);
    } else taken_hi = taken_lo;
    last_row_taken = last_row_seen;
    working_begin = taken_hi;
    *lo = taken_lo.data(); *lo_len = (uint32_t)taken_lo.size(); *hi = taken_hi.data(); *hi_len = (uint32_t)taken_hi.size();
    return B2_OK;
  }
  // RangesScanner::collect_scanned_rows_per_range (scanner.rs:196-201): rows per input range since the last call
  int collect_scanned_rows_per_range(uint64_t* out, uint32_t* n_inout) {
    uint32_t n = (uint32_t)range_rows_taken.size();
    if (out && n && range_rows.p) {
      std::vector<uint64_t> cur(n);
      CUDA_TRY(cudaStreamSynchronize(stream));
      CUDA_TRY(cudaMemcpy(cur.data(), range_rows.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
      for (uint32_t i = 0; i < n && i < *n_inout; ++i) { out[i] = cur[i] - range_rows_taken[i]; range_rows_taken[i] = cur[i]; }
    }
    *n_inout = n;
    return B2_OK;
  }

  // ---- response encoding of the batch just produced (runner.rs:1051-1088 encode_result_to_chunk) ----
  struct DevColRef { const void* data; const unsigned long long* bitmap; int kind; int field_tp; uint32_t field_flag; const long long* offsets = nullptr; uint64_t heap_len = 0; bool raw = false; };
  std::vector<DevColRef> last_dev;  // device-resident columns of the last batch, in output order
  uint64_t last_rows = 0;
  DevBuf enc_cols, enc_counts, enc_out, enc_lens, enc_offs, enc_tmp;
  HostBuf enc_host;

  int encode_batch(int32_t encode_type, int32_t location, b2_encoded_chunk* out) {
    memset(out, 0, sizeof(*out));
    out->encode_type = encode_type; out->location = location; out->n_rows = last_rows;
    const int nc = (int)last_dev.size();
    const uint64_t n = last_rows;
    if (encode_type != B2_ENCODE_TYPE_DEFAULT && encode_type != B2_ENCODE_TYPE_CHUNK) { g_last_error = "unknown encode type"; return B2_ERR_INVALID_ARG; }
    if (nc == 0 || (n == 0 && encode_type == B2_ENCODE_TYPE_DEFAULT)) return B2_OK;
    std::vector<EncCol> ec((size_t)nc);
    for (int k = 0; k < nc; ++k) {
      const DevColRef& d = last_dev[(size_t)k];
      ec[(size_t)k] = EncCol{d.data, d.bitmap, d.kind, d.field_tp == B2_TP_FLOAT ? 1 : 0, (d.field_flag & B2_FLAG_UNSIGNED) ? 1 : 0, 0u, 0ull, d.offsets, d.heap_len};
      if (encode_type == B2_ENCODE_TYPE_DEFAULT && (d.raw || d.kind == B2_COL_TIME || d.kind == B2_COL_DURATION)) {
        // the reference copies the stored datum of such a column (lazy_column.rs:242-257); the decoded cell does not determine it
        g_last_error = "TypeDefault encoding of bytes / json / decimal / time / duration scan columns is not on the device path (use TypeChunk)";
        return B2_ERR_UNSUPPORTED;
      }
    }
    CUDA_TRY(enc_cols.reserve((size_t)nc * sizeof(EncCol)));
    CUDA_TRY(enc_counts.reserve((size_t)nc * 4));
    std::vector<unsigned int> nulls((size_t)nc, 0);
    if (n) {
      CUDA_TRY(cudaMemcpyAsync(enc_cols.p, ec.data(), (size_t)nc * sizeof(EncCol), cudaMemcpyHostToDevice, stream));
      CUDA_TRY(launch_enc_null_count((const EncCol*)enc_cols.p, nc, n, (unsigned int*)enc_counts.p, stream));
      CUDA_TRY(cudaMemcpyAsync(nulls.data(), enc_counts.p, (size_t)nc * 4, cudaMemcpyDeviceToHost, stream));
      CUDA_TRY(cudaStreamSynchronize(stream));
      stats.kernel_launches++;
    }
    uint64_t total = 0;
    if (encode_type == B2_ENCODE_TYPE_CHUNK) {
      for (int k = 0; k < nc; ++k) {
        EncCol& c = ec[(size_t)k];
        c.null_cnt = nulls[(size_t)k]; c.chunk_off = total;
        uint64_t esz = c.kind == B2_COL_DECIMAL ? 40 : (c.is_f32 ? 4 : 8);
        if (c.kind == B2_COL_BYTES || c.kind == B2_COL_JSON) total += 8 + (c.null_cnt ? (n + 7) / 8 : 0) + (n + 1) * 8 + c.heap_len;
        else total += 8 + (c.null_cnt ? (n + 7) / 8 : 0) + n * esz;
      }
      CUDA_TRY(enc_out.reserve(total));
      CUDA_TRY(cudaMemcpyAsync(enc_cols.p, ec.data(), (size_t)nc * sizeof(EncCol), cudaMemcpyHostToDevice, stream));
      CUDA_TRY(launch_enc_chunk((const EncCol*)enc_cols.p, nc, n, (unsigned char*)enc_out.p, stream));
      stats.kernel_launches++;
    } else {
      bool fixed = true;
      for (int k = 0; k < nc; ++k) if (nulls[(size_t)k] || ec[(size_t)k].kind == B2_COL_DECIMAL) fixed = false;
      const unsigned long long* offs = nullptr;
      if (fixed) total = n * 9ull * (uint64_t)nc;
      else {
        CUDA_TRY(enc_lens.reserve(n * 4)); CUDA_TRY(enc_offs.reserve(n * 8));
        size_t tb = enc_scan_temp_bytes(n);
        CUDA_TRY(enc_tmp.reserve(tb));
        CUDA_TRY(launch_enc_row_len((const EncCol*)enc_cols.p, nc, n, (unsigned int*)enc_lens.p, stream));
        CUDA_TRY(launch_enc_scan((const unsigned int*)enc_lens.p, (unsigned long long*)enc_offs.p, n, enc_tmp.p, tb, stream));
        unsigned long long last_off = 0; unsigned int last_len = 0;
        CUDA_TRY(cudaMemcpyAsync(&last_off, (const unsigned long long*)enc_offs.p + (n - 1), 8, cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaMemcpyAsync(&last_len, (const unsigned int*)enc_lens.p + (n - 1), 4, cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        total = last_off + last_len;
        offs = (const unsigned long long*)enc_offs.p;
        stats.kernel_launches += 2;
      }
      CUDA_TRY(enc_out.reserve(total));
      CUDA_TRY(launch_enc_rows((const EncCol*)enc_cols.p, nc, n, offs, (unsigned int)(9 * nc), (unsigned char*)enc_out.p, stream));
      stats.kernel_launches++;
    }
    out->len = total;
    if (location == B2_LOC_HOST) {
      CUDA_TRY(enc_host.reserve(total));
      CUDA_TRY(cudaMemcpyAsync(enc_host.p, enc_out.p, total, cudaMemcpyDeviceToHost, stream));
      d2h_bytes += total;
      out->rows_data = (const uint8_t*)enc_host.p;
    } else out->rows_data = (const uint8_t*)enc_out.p;
    CUDA_TRY(cudaStreamSynchronize(stream));
    stats.d2h_bytes = d2h_bytes;
    return B2_OK;
  }

  uint64_t d2h_bytes = 0;

  // ---- PM_AGG: everything in one go ----
  int alloc_table(unsigned int cap) {
    size_t W = cp.dev.acc_words;
    CUDA_TRY(tbl_keys.reserve(((size_t)cap + 2) * 8));
    CUDA_TRY(tbl_occ.reserve(8));
    CUDA_TRY(tbl_acc.reserve(((size_t)cap + 2) * 8 * W));
    CUDA_TRY(cudaMemsetAsync(tbl_keys.p, 0xff, ((size_t)cap + 2) * 8, stream));  // AGG_EMPTY_KEY everywhere
    CUDA_TRY(cudaMemsetAsync(tbl_occ.p, 0, 8, stream));
    CUDA_TRY(cudaMemsetAsync(tbl_acc.p, 0, ((size_t)cap + 2) * 8 * W, stream));
    if (cp.dev.n_group > 1) {  // composite keys: key words per slot + a "key published" flag
      CUDA_TRY(tbl_gkeys.reserve((size_t)cap * 8 * (cp.dev.n_group + 1)));
      CUDA_TRY(tbl_ready.reserve((size_t)cap * 4));
      CUDA_TRY(cudaMemsetAsync(tbl_ready.p, 0, (size_t)cap * 4, stream));
    }
    tbl_cap = cap;
    return B2_OK;
  }

  int run_agg(b2_batch* out) {
    const DevPlan& P = cp.dev;
    uint64_t total_entries = 0;
    for (auto& u : units) total_entries += u.e_hi - u.e_lo;
    unsigned int cap = 1;
    if (P.has_group) {
      cap = 1u << 16;
      while (cap < (1u << 22) && (uint64_t)cap < total_entries * 2) cap <<= 1;
    }
    size_t smem = 0;
    uint32_t smem_slots = 0;
    if (P.has_group && P.n_group <= 1) {
      // small on purpose (192 resident groups per CTA): it absorbs the low-cardinality case, where global atomics would
      // serialise on a few addresses; beyond that the HBM table lives in L2 anyway and a big CTA table only costs
      // shared memory
      smem_slots = P.acc_words > 32 ? 0 : 256;  // (exact Real sums are 67 words per group: those plans use the HBM table only)
      while (smem_slots > 64 && (size_t)smem_slots * (8 + 8 * P.acc_words) > 64 * 1024) smem_slots >>= 1;
      smem = (size_t)smem_slots * (8 + 8 * P.acc_words);
    }
    // the lean kernel's CTA table: as many slots as 64 KB hold (2048 for COUNT + SUM), so that a thousand groups stay resident
    uint32_t fast_slots = 0;
    size_t fast_smem = 0;
    if (P.has_group && P.n_group <= 1) {
      // direct-addressed: accumulators of the group keys 0 .. slots-1 (+ 4 bytes of occupancy each); 1024 slots of COUNT + SUM
      // are 28 KB, which still lets three CTAs share an SM
      fast_slots = 1024;
      while (fast_slots > 64 && (size_t)fast_slots * (4 + 8 * P.acc_words) > 28 * 1024) fast_slots >>= 1;
      fast_smem = ((size_t)fast_slots * (4 + 8 * P.acc_words) + 15) & ~(size_t)15;
    }
    Counters c;
    for (;;) {
      int rc = alloc_table(cap);
      if (rc) return rc;
      rc = init_device_state();
      if (rc) return rc;
      int grid = 0;
      size_t grid_smem = ~(size_t)0;
      entries_scanned = 0;
      for (size_t ui = 0; ui < units.size(); ++ui) {
        const Unit& u = units[ui];
        if (deadline_exceeded()) { cudaStreamSynchronize(stream); return publish_agg(0, nullptr, nullptr, nullptr, out); }
        BlockView v;
        rc = acquire_block(u.block_idx, &v);
        if (rc) return rc;
        ScanArgs a = base_args(u, v);
        a.c_lo = u.e_lo; a.c_hi = u.e_hi;
        a.tbl.keys = (unsigned long long*)tbl_keys.p; a.tbl.special = (unsigned int*)tbl_occ.p; a.tbl.acc = (unsigned long long*)tbl_acc.p; a.tbl.cap = tbl_cap;
        a.tbl.gkeys = (unsigned long long*)tbl_gkeys.p; a.tbl.ready = (unsigned int*)tbl_ready.p; a.tbl.hash_mask_bits = debug_hash_bits;
        a.smem_slots = smem_slots;
        const bool fast = u.fast_ok && fast_kernel_covers();
        int gg = 0, fg = 0;
        rc = launch_unit(a, u, fast, smem, fast_smem, fast_slots, &gg, &fg);
        if (rc) return rc;
        grid = gg;
        release_block(u.block_idx);
        prefetch_after(ui);
        entries_scanned += u.e_hi - u.e_lo;
        stats.num_iterations++;
      }
      // the group table -> compact group list right behind the last unit, so that one read of the counters serves both;
      // the list of a table that overflowed is discarded with it
      if (P.has_group) {
        size_t W = P.acc_words;
        CUDA_TRY(grp_keys.reserve(((size_t)tbl_cap + 2) * 8 * std::max(1, P.n_group))); CUDA_TRY(grp_null.reserve((size_t)tbl_cap + 2)); CUDA_TRY(grp_acc.reserve(((size_t)tbl_cap + 2) * 8 * W));
        AggTable t; t.keys = (unsigned long long*)tbl_keys.p; t.special = (unsigned int*)tbl_occ.p; t.acc = (unsigned long long*)tbl_acc.p; t.cap = tbl_cap;
        t.gkeys = (unsigned long long*)tbl_gkeys.p; t.ready = (unsigned int*)tbl_ready.p; t.hash_mask_bits = 0;
        CUDA_TRY(launch_agg_finalize(P, t, ctr(), (unsigned long long*)grp_keys.p, (unsigned char*)grp_null.p, (unsigned long long*)grp_acc.p, stream));
      }
      rc = read_counters(&c);
      if (rc) return rc;
      if (c.agg_overflow && !c.agg_stuck && cap < (1u << 30)) {  // group table full: grow and redo (partial results are discarded)
        cap <<= 2;
        for (auto& s : slots) s.block = -1;
        continue;
      }
      break;
    }
    fill_stats(c);
    drained = true;
    if (c.agg_stuck)
      return fail(B2_ERR_UNSUPPORTED, "composite-key group table: " + std::to_string(c.agg_stuck) + " inserts gave up waiting for a claimed slot's key (longest probe run " +
                                          std::to_string(c.agg_probe_max) + " slots)");
    if (c.agg_overflow) return fail(B2_ERR_UNSUPPORTED, "group table exceeded the device capacity");
    if (c.err != ~0ull) { device_error(c); return publish_agg(0, nullptr, nullptr, nullptr, out); }
    check_trailing_lock();
    if (failed) return publish_agg(0, nullptr, nullptr, nullptr, out);
    unsigned int n_groups;
    const unsigned long long *gk = nullptr, *ga = nullptr;
    const unsigned char* gn = nullptr;
    if (!P.has_group) {
      n_groups = c.live_rows > 0 ? 1 : 0;  // simple_aggr_executor.rs:141-148, 233-248
      ga = (const unsigned long long*)tbl_acc.p;
    } else {
      n_groups = c.n_groups;
      gk = (const unsigned long long*)grp_keys.p; gn = (const unsigned char*)grp_null.p; ga = (const unsigned long long*)grp_acc.p;
    }
    part_n = n_groups; part_keys = gk; part_null = gn; part_acc = ga;
    return publish_agg(n_groups, gk, gn, ga, out);
  }
  unsigned int part_n = 0;
  const unsigned long long *part_keys = nullptr, *part_acc = nullptr;
  const unsigned char* part_null = nullptr;

  int publish_agg(unsigned int n_groups, const unsigned long long* gk, const unsigned char* gn, const unsigned long long* ga, b2_batch* out) {
    const DevPlan& P = cp.dev;
    size_t ncol = cp.schema.size();
    res_cols.resize(ncol); res_bitmaps.resize(ncol);
    std::vector<void*> ptrs(2 * ncol, nullptr);
    size_t bm_bytes = (((size_t)n_groups + 63) / 64) * 8;
    for (size_t k = 0; k < ncol; ++k) {
      size_t esz = cp.schema[k].kind == B2_COL_DECIMAL ? 40 : 8;
      CUDA_TRY(res_cols[k].reserve(std::max<size_t>(8, (size_t)n_groups * esz)));
      CUDA_TRY(res_bitmaps[k].reserve(std::max<size_t>(8, bm_bytes)));
      CUDA_TRY(cudaMemsetAsync(res_bitmaps[k].p, 0xff, std::max<size_t>(8, bm_bytes), stream));
      ptrs[k] = res_cols[k].p; ptrs[ncol + k] = res_bitmaps[k].p;
    }
    if (n_groups) {  // (one publish per request: the pinned source is written once)
      CUDA_TRY(res_ptrs.reserve(ptrs.size() * sizeof(void*)));
      CUDA_TRY(h_res_ptrs.reserve(ptrs.size() * sizeof(void*)));
      memcpy(h_res_ptrs.p, ptrs.data(), ptrs.size() * sizeof(void*));
      CUDA_TRY(cudaMemcpyAsync(res_ptrs.p, h_res_ptrs.p, ptrs.size() * sizeof(void*), cudaMemcpyHostToDevice, stream));
      CUDA_TRY(launch_agg_result(P, n_groups, gk, gn, ga, (unsigned long long**)res_ptrs.p, (unsigned long long**)res_ptrs.p + ncol, stream));
    }
    // deliver the requested output offsets
    const size_t n_out = cp.output_offsets.size();
    std::vector<FixedCol> fc(n_out);
    for (size_t i = 0; i < n_out; ++i) {
      const uint32_t k = cp.output_offsets[i];
      fc[i] = FixedCol{res_cols[k].p, res_bitmaps[k].p, (size_t)(cp.schema[k].kind == B2_COL_DECIMAL ? 40 : 8), bm_bytes};
    }
    int rc = publish_fixed(fc, n_groups);
    if (rc) return rc;
    // (next_batch waits for the stream before it returns the batch)
    out->columns = cols.data(); out->n_columns = (uint32_t)n_out; out->n_rows = n_groups; out->n_warnings = 0;
    out->is_drained = B2_DRAIN_DRAINED;
    stats.num_produced_rows += n_groups;
    return failed ? last_err.status : B2_OK;
  }

  // ---- PM_TOPN: per unit: per-CTA candidate lists -> unit top-N -> payload gather -> merge into the running top-N ----
  DevBuf tn_work, tn_lvl_a, tn_lvl_a_cnt, tn_lvl_b, tn_lvl_b_cnt, tn_lists, tn_counts, tn_pair, tn_pair_cnt, tn_tmp, tn_tmp_cnt, tn_blk_pay, tn_blk_null, tn_run_pay, tn_run_null, tn_tmp_pay, tn_tmp_null, tn_bitmap;

  int run_topn(b2_batch* out) {
    const DevPlan& P = cp.dev;
    drained = true;
    uint32_t limit = (uint32_t)P.limit, n_out = (uint32_t)P.n_out;
    int rc = init_device_state();
    if (rc) return rc;
    uint32_t n = 0;
    if (limit > 0 && !units.empty()) {  // top_n_executor.rs:304-312: n == 0 drains immediately
      uint32_t cap = 512;
      while (cap < limit + TILE) cap <<= 1;
      size_t smem = topn_smem_bytes(cap, P.n_order);
      ScanArgs probe; memset(&probe, 0, sizeof(probe));
      size_t tot0 = setup_staging(&probe, wblocks[units[0].block_idx], smem);
      int grid = scan_grid_for(PM_TOPN, std::max(tot0, smem));
      const bool any_fast = fast_kernel_covers();
      int fast_grid = 0;
      if (any_fast) {  // the lean kernel keeps its candidate buffers in HBM (ScanArgs::topn_work): shared memory holds the stages only
        const JitKernel* jk = jit_ready();
        ScanArgs fprobe; memset(&fprobe, 0, sizeof(fprobe));
        const size_t ftot0 = setup_staging(&fprobe, wblocks[units[0].block_idx], 0);
        fast_grid = jk && jk->fn_fast ? jit_max_blocks_per_sm(jk, ftot0, true) * scan_num_sms() : fast_max_grid(PM_TOPN, ftot0);
        CUDA_TRY(tn_work.reserve((size_t)fast_grid * smem));
      }
      const int lists_cap = grid + fast_grid;  // the lean and the general kernel leave their per-CTA lists side by side
      size_t isz = sizeof(TopItem);
      CUDA_TRY(tn_lists.reserve((size_t)lists_cap * limit * isz)); CUDA_TRY(tn_counts.reserve((size_t)lists_cap * 4));
      CUDA_TRY(tn_lvl_a.reserve((size_t)((lists_cap + 7) / 8) * limit * isz)); CUDA_TRY(tn_lvl_a_cnt.reserve((size_t)((lists_cap + 7) / 8) * 4));
      CUDA_TRY(tn_lvl_b.reserve((size_t)((lists_cap + 63) / 64) * limit * isz)); CUDA_TRY(tn_lvl_b_cnt.reserve((size_t)((lists_cap + 63) / 64) * 4));
      CUDA_TRY(tn_pair.reserve((size_t)2 * limit * isz)); CUDA_TRY(tn_pair_cnt.reserve(8));
      CUDA_TRY(tn_tmp.reserve((size_t)limit * isz)); CUDA_TRY(tn_tmp_cnt.reserve(8));
      size_t pay_bytes = (size_t)n_out * limit * 8, null_bytes = (size_t)n_out * limit;
      for (DevBuf* b : {&tn_blk_pay, &tn_run_pay, &tn_tmp_pay}) CUDA_TRY(b->reserve(pay_bytes));
      for (DevBuf* b : {&tn_blk_null, &tn_run_null, &tn_tmp_null}) CUDA_TRY(b->reserve(null_bytes));
      CUDA_TRY(cudaMemsetAsync(tn_pair_cnt.p, 0, 8, stream));
      CUDA_TRY(cudaMemsetAsync(tn_tmp_cnt.p, 0, 4, stream));
      // the running top-N and the buffer the next merge writes swap roles after every chunk (no copies back):
      // run_* = the running list, its count, payload columns, NULL flags; nxt_* = where merge2 / copy put the new one
      TopItem *run_items = (TopItem*)tn_pair.p, *nxt_items = (TopItem*)tn_tmp.p;
      unsigned int *run_cnt = (unsigned int*)tn_pair_cnt.p, *nxt_cnt = (unsigned int*)tn_tmp_cnt.p;
      DevBuf *run_pay = &tn_run_pay, *nxt_pay = &tn_tmp_pay, *run_null = &tn_run_null, *nxt_null = &tn_tmp_null;
      TopItem* const unit_items = (TopItem*)tn_pair.p + limit;  // the chunk's own top-N (second half of tn_pair)
      unsigned int* const unit_cnt = (unsigned int*)tn_pair_cnt.p + 1;
      // The running top-N seeds every later launch with its N-th item, and a CTA drops rows that cannot beat it after one
      // comparison.  The very first rows have no such bound, so the request starts with short chunks that grow 8x each:
      // after c rows the bound passes about limit / c of what follows, i.e. every chunk hands ~8 x limit candidates to
      // the merge below instead of one full list per CTA.
      uint64_t seeded_rows = 0;
      for (size_t ui = 0; ui < units.size(); ++ui) {
       const Unit& u = units[ui];
       BlockView v;
       rc = acquire_block(u.block_idx, &v);
       if (rc) return rc;
       for (uint32_t c_lo = u.e_lo; c_lo < u.e_hi;) {
        if (deadline_exceeded()) break;
        const uint64_t want = std::max<uint64_t>(16 * TILE, 7 * seeded_rows);
        const uint32_t c_hi = (uint64_t)(u.e_hi - c_lo) <= want + want / 2 ? u.e_hi : c_lo + (uint32_t)want;
        ScanArgs a = base_args(u, v);
        a.c_lo = c_lo; a.c_hi = c_hi;
        uint32_t n_tiles = (c_hi - c_lo + TILE - 1) / TILE;
        a.topn.items = (TopItem*)tn_lists.p; a.topn.counts = (unsigned int*)tn_counts.p; a.topn.stride = limit;
        a.topn_cap = cap;
        a.topn_seed = run_items; a.topn_seed_cnt = run_cnt;
        a.topn_work = (unsigned char*)tn_work.p; a.topn_work_stride = smem;
        CUDA_TRY(cudaMemsetAsync(tn_counts.p, 0, (size_t)lists_cap * 4, stream));
        const bool fast = any_fast && u.fast_ok;
        int gg = (int)std::min<uint32_t>((uint32_t)grid, n_tiles), fg = (int)std::min<uint32_t>((uint32_t)std::max(fast_grid, 1), n_tiles);
        rc = launch_unit(a, u, fast, smem, 0, 0, &gg, &fg);
        if (rc) return rc;
        a.topn.n_lists = (uint32_t)(gg + fg);
        // unit top-N (sorted) lands in the second half of `pair`
        TopNLists unit_out; unit_out.items = unit_items; unit_out.counts = unit_cnt; unit_out.n_lists = 1; unit_out.stride = limit;
        {  // per-CTA lists -> one list, fan-in 16 per level (after the first chunks the lists are nearly empty: fewer launches matter more than narrow merges)
          TopNLists cur = a.topn;
          int flip = 0;
          while (cur.n_lists > 16) {
            TopNLists nxt;
            nxt.n_lists = (cur.n_lists + 15) / 16; nxt.stride = limit;
            nxt.items = (TopItem*)(flip ? tn_lvl_b.p : tn_lvl_a.p); nxt.counts = (unsigned int*)(flip ? tn_lvl_b_cnt.p : tn_lvl_a_cnt.p);
            CUDA_TRY(launch_topn_merge(P, cur, nxt, 16, stream));
            stats.kernel_launches++;
            cur = nxt; flip ^= 1;
          }
          CUDA_TRY(launch_topn_merge(P, cur, unit_out, cur.n_lists, stream));
        }
        CUDA_TRY(launch_topn_gather(P, a, unit_items, unit_cnt, (unsigned long long*)tn_blk_pay.p, (unsigned char*)tn_blk_null.p, limit, stream));
        // running top-N + the chunk's top-N -> the other buffer set, which becomes the running one
        CUDA_TRY(launch_topn_merge2(P, run_items, run_cnt, unit_items, unit_cnt, nxt_items, nxt_cnt, limit, stream));
        CUDA_TRY(launch_topn_copy(nxt_items, nxt_cnt, n_out, limit, (const unsigned long long*)run_pay->p, (const unsigned char*)run_null->p,
                                  (const unsigned long long*)tn_blk_pay.p, (const unsigned char*)tn_blk_null.p, (unsigned long long*)nxt_pay->p, (unsigned char*)nxt_null->p, stream));
        std::swap(run_items, nxt_items); std::swap(run_cnt, nxt_cnt); std::swap(run_pay, nxt_pay); std::swap(run_null, nxt_null);
        entries_scanned += c_hi - c_lo;
        seeded_rows += c_hi - c_lo;
        stats.num_iterations++;
        stats.kernel_launches += 4;
        c_lo = c_hi;
       }
       release_block(u.block_idx);
       prefetch_after(ui);
      }
      if (run_pay != &tn_run_pay) { std::swap(tn_run_pay, tn_tmp_pay); std::swap(tn_run_null, tn_tmp_null); }  // the result is read from tn_run_* below
      CUDA_TRY(cudaMemcpyAsync(h_ctr.p, run_cnt, 4, cudaMemcpyDeviceToHost, stream));
      CUDA_TRY(cudaStreamSynchronize(stream));
      n = *(uint32_t*)h_ctr.p;
    }
    Counters c;
    rc = read_counters(&c);
    if (rc) return rc;
    fill_stats(c);
    if (failed) n = 0;  // (deadline)
    else if (c.err != ~0ull) { device_error(c); n = 0; }
    else { check_trailing_lock(); if (failed) n = 0; }
    // publish: payload columns of the running list, NULL flags packed into BitVec words
    uint32_t words = (std::max<uint32_t>(limit, 1) + 63) / 64;
    if (n) {
      CUDA_TRY(tn_bitmap.reserve((size_t)n_out * words * 8));
      CUDA_TRY(launch_pack_nulls((const unsigned char*)tn_run_null.p, n_out, limit, n, (unsigned long long*)tn_bitmap.p, words, stream));
    }
    const size_t n_sel = cp.output_offsets.size();
    std::vector<FixedCol> fc(n_sel, FixedCol{nullptr, nullptr, 8, (size_t)words * 8});
    for (size_t i = 0; i < n_sel && n; ++i) {
      const uint32_t k = cp.output_offsets[i];
      fc[i].data = (const uint8_t*)tn_run_pay.p + (size_t)k * limit * 8;
      fc[i].bitmap = (const uint8_t*)tn_bitmap.p + (size_t)k * words * 8;
    }
    rc = publish_fixed(fc, n);
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(stream));
    out->columns = cols.data(); out->n_columns = (uint32_t)n_sel; out->n_rows = n; out->n_warnings = 0;
    out->is_drained = B2_DRAIN_DRAINED;
    stats.num_produced_rows += n;
    return failed ? last_err.status : B2_OK;
  }

  int next_batch(uint64_t scan_rows, b2_batch* out) {
    memset(out, 0, sizeof(*out));
    cudaSetDevice(device);
    if (failed || drained) { out->is_drained = B2_DRAIN_DRAINED; return failed ? last_err.status : B2_OK; }
    if (deadline_exceeded()) { out->is_drained = B2_DRAIN_DRAINED; return last_err.status; }
    if (!started) {
      started = true;
      if (cp.dev.mode == PM_SCAN) {
        int rc = init_device_state();
        if (rc) return rc;
        enter_unit(cp.desc && !units.empty() ? units.size() - 1 : 0);
      }
    }
    if (!batch_ev[0]) { batch_ev[0] = event_pool().get(); batch_ev[1] = event_pool().get(); }
    cudaEvent_t t0 = batch_ev[0], t1 = batch_ev[1];
    cudaEventRecord(t0, stream);
    int rc;
    if (cp.dev.mode == PM_SCAN) rc = next_scan_batch(scan_rows, out);
    else if (cp.dev.mode == PM_AGG) rc = run_agg(out);
    else rc = run_topn(out);
    cudaEventRecord(t1, stream);
    cudaEventSynchronize(t1);
    float ms = 0;
    cudaEventElapsedTime(&ms, t0, t1);
    stats.time_processed_ns += (uint64_t)(ms * 1e6);
    out->n_warnings = (uint32_t)std::min<uint64_t>(warnings_total - warnings_reported, 0xffffffffull);
    warnings_reported = warnings_total;
    return rc;
  }
};

// ------------------------------------------------------------------------------------------------------------------
extern "C" {

uint32_t b2_abi_version(void) { return B2_ABI_VERSION; }
const char* b2_build_info(void) { return "tikv_b200 libb2copr sm_90a (CUDA " __DATE__ ")"; }
const char* b2_last_error_message(void) { return g_last_error.c_str(); }

int32_t b2_check_supported(const b2_dag_plan* plan) {
  CompiledPlan cp;
  std::string msg;
  int rc = compile_plan(plan, &cp, &msg);
  if (rc) g_last_error = msg;
  return rc;
}

// tooling: the compiled device plan as a C++ aggregate initialiser (plan-specialised kernel builds); returns its length
extern "C" int64_t b2_plan_literal(const b2_dag_plan* plan, char* buf, uint64_t cap) {
  CompiledPlan cp;
  std::string msg;
  int rc = compile_plan(plan, &cp, &msg);
  if (rc) { g_last_error = msg; return -rc; }
  std::string lit = plan_literal(cp.dev);
  if (buf && cap) { size_t n = std::min<size_t>(lit.size(), (size_t)cap - 1); memcpy(buf, lit.data(), n); buf[n] = 0; }
  return (int64_t)lit.size();
}

int32_t b2_exec_open(const b2_dag_plan* plan, const b2_key_range* ranges, uint32_t n_ranges, const b2_region_source* src,
                     const b2_exec_config* cfg, b2_exec** out) {
  if (!plan || !src || !out) { g_last_error = "null argument"; return B2_ERR_INVALID_ARG; }
  std::unique_ptr<b2_exec> h(new b2_exec());
  std::string msg;
  int rc = compile_plan(plan, &h->cp, &msg);
  if (rc) { g_last_error = msg; return rc; }
  h->device = src->device;
  cudaError_t e = cudaSetDevice(h->device);
  if (e != cudaSuccess) { g_last_error = std::string("cudaSetDevice: ") + cudaGetErrorString(e) + " (the CUDA device path is required; there is no CPU fallback)"; return B2_ERR_CUDA; }
  e = h->open_streams(cfg);
  if (e != cudaSuccess) { g_last_error = cudaGetErrorString(e); return B2_ERR_CUDA; }
  h->out_loc = cfg ? cfg->output_location : B2_LOC_DEVICE;
  h->deadline_ns = cfg ? cfg->deadline_ns : 0;
  h->paging_size = cfg ? cfg->paging_size : 0;
  if (const char* v = getenv("B2_DEBUG_AGG_HASH_BITS")) h->debug_hash_bits = (unsigned int)std::min(63, std::max(0, atoi(v)));
  if (h->paging_size && h->cp.dev.mode != PM_SCAN) {
    // Aggregation / TopN under paging depend on the reference's 1024-row batch boundaries (aggr_executor.rs:226-236,
    // top_n_executor.rs:304-318): the CPU executors keep those requests
    g_last_error = "paging is on the device path for scan / selection / projection pipelines only";
    return B2_ERR_UNSUPPORTED;
  }
  h->cp.dev.read_ts = src->read_ts;
  h->cp.dev.isolation = src->isolation_level;
  if (!h->cp.pool.empty()) {  // bytes constants (LIKE patterns): to HBM, their launch parameters become cell references into it
    e = h->const_pool.reserve(h->cp.pool.size() + 16);
    // (no wait: the source lives as long as the handle, and the kernels that read the copy run behind it on the same stream)
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->const_pool.p, h->cp.pool.data(), h->cp.pool.size(), cudaMemcpyHostToDevice, h->stream);
    if (e != cudaSuccess) { g_last_error = std::string("bytes constants: ") + cudaGetErrorString(e); return B2_ERR_CUDA; }
    patch_pool_imms(h->cp, (const uint8_t*)h->const_pool.p);
  }
  rc = h->setup_source(src, ranges, n_ranges);
  if (rc) { g_last_error = h->last_err.message; return rc; }
  // the exact-layout path for row-format-v1 rows is only compiled in / switched on when the data looks like v1
  if (h->cp.dev.fast_v1 && !h->sample_is_v1()) h->cp.dev.fast_v1 = 0;
  // plan-specialised kernel: B2_JIT=off|sync|auto (environment) overrides cfg->jit; `auto` compiles in the background
  // for requests big enough to matter and switches over when the kernel is ready
  h->jit_mode = cfg ? cfg->jit : B2_JIT_AUTO;
  if (const char* ev = getenv("B2_JIT")) h->jit_mode = !strcmp(ev, "off") ? B2_JIT_OFF : (!strcmp(ev, "sync") ? B2_JIT_SYNC : B2_JIT_AUTO);
  if (plan_uses_ext_sigs(h->cp.dev)) {  // DIV / MOD / IF / CASE ...: only compiled into specialised kernels (b2_device.h)
    if (!jit_available()) { g_last_error = "this plan's scalar functions need the run-time compiler (libnvrtc), which is not available"; return B2_ERR_UNSUPPORTED; }
    h->jit_mode = B2_JIT_SYNC;
  }
  uint64_t total_entries = 0;
  for (const Unit& u : h->units) total_entries += u.e_hi - u.e_lo;
  if (h->jit_mode == B2_JIT_SYNC || (h->jit_mode == B2_JIT_AUTO && total_entries >= (1u << 20))) h->jit_start();
  if (h->jit_mode == B2_JIT_SYNC && h->jit_started) {
    const JitKernel* k = h->jit_fut.get();
    if (!k->ok) { g_last_error = "plan-specialised kernel: " + k->error; return B2_ERR_CUDA; }
  }
  *out = h.release();
  return B2_OK;
}

// Prepared plan: compile the plan-specialised kernel for `device` now (blocking), so that later requests with this plan
// start on it.  B2_ERR_UNSUPPORTED when run-time compilation is not available in this process (the generic kernels work).
extern "C" int32_t b2_plan_prepare(const b2_dag_plan* plan, int32_t device) {
  CompiledPlan cp;
  std::string msg;
  int rc = compile_plan(plan, &cp, &msg);
  if (rc) { g_last_error = msg; return rc; }
  std::string why;
  if (!jit_available(&why)) { g_last_error = "run-time compilation unavailable: " + why; return B2_ERR_UNSUPPORTED; }
  // both data-dependent variants: without and (where the plan allows it) with the row-format-v1 exact-layout path
  std::shared_future<JitKernel*> with_v1;
  if (cp.dev.fast_v1) with_v1 = jit_get(device, cp.dev);
  cp.dev.fast_v1 = 0;
  const JitKernel* k = jit_get(device, cp.dev).get();
  if (k->ok && with_v1.valid()) k = with_v1.get();
  if (!k->ok) { g_last_error = "plan-specialised kernel: " + k->error; return B2_ERR_CUDA; }
  return B2_OK;
}

// Ahead-of-time: compile the plan-specialised kernel(s) of `plan` into the on-disk cache with NVRTC alone — no GPU, no
// CUDA context (build machines; `__graft_entry__.build()` warms the cache for the bench plans this way).  Returns B2_OK,
// *n_compiled (may be NULL) = kernels compiled now (0 = everything was cached already).
extern "C" int32_t b2_plan_precompile(const b2_dag_plan* plan, int32_t* n_compiled) {
  CompiledPlan cp;
  std::string msg;
  int rc = compile_plan(plan, &cp, &msg);
  if (rc) { g_last_error = msg; return rc; }
  int done = 0;
  for (int v1 = (cp.dev.fast_v1 ? 1 : 0); v1 >= 0; --v1) {  // both data-dependent variants, like b2_plan_prepare
    cp.dev.fast_v1 = v1;
    std::string err;
    int r = jit_precompile(cp.dev, &err);
    if (r < 0) { g_last_error = "plan-specialised kernel: " + err; return B2_ERR_UNSUPPORTED; }
    done += r == 0;
  }
  if (n_compiled) *n_compiled = done;
  return B2_OK;
}
extern "C" void b2_jit_counters(uint64_t* nvrtc_compiles, uint64_t* disk_cache_hits) {
  unsigned long long a = 0, b = 0;
  jit_counters(&a, &b);
  if (nvrtc_compiles) *nvrtc_compiles = a;
  if (disk_cache_hits) *disk_cache_hits = b;
}

int32_t b2_exec_schema(b2_exec* h, int32_t* field_tps, uint32_t* field_flags, uint32_t* n_inout) {
  uint32_t n = (uint32_t)h->cp.output_offsets.size();
  if (field_tps && field_flags)
    for (uint32_t i = 0; i < n && i < *n_inout; ++i) { field_tps[i] = h->cp.schema[h->cp.output_offsets[i]].field_tp; field_flags[i] = h->cp.schema[h->cp.output_offsets[i]].field_flag; }
  *n_inout = n;
  return B2_OK;
}

int32_t b2_exec_next_batch(b2_exec* h, uint64_t scan_rows, b2_batch* out) { return h->next_batch(scan_rows, out); }

int32_t b2_exec_collect_stats(b2_exec* h, b2_exec_stats* out) {
  h->stats.h2d_bytes = h->h2d_bytes; h->stats.d2h_bytes = h->d2h_bytes;  // (copies made after the last counter read-back included)
  *out = h->stats;
  return B2_OK;
}
int32_t b2_exec_last_error(b2_exec* h, b2_error_info* out) { *out = h->last_err; return B2_OK; }
int32_t b2_exec_can_be_cached(b2_exec* h) { return (h->check_newer && !h->met_newer_any && !h->saw_lock) ? 1 : 0; }
int32_t b2_exec_take_scanned_range(b2_exec* h, const uint8_t** lower, uint32_t* lower_len, const uint8_t** upper, uint32_t* upper_len) {
  if (!h || !lower || !lower_len || !upper || !upper_len) { g_last_error = "null argument"; return B2_ERR_INVALID_ARG; }
  return h->take_scanned_range(lower, lower_len, upper, upper_len);
}
int32_t b2_exec_collect_scanned_rows_per_range(b2_exec* h, uint64_t* rows, uint32_t* n_inout) {
  if (!h || !n_inout) { g_last_error = "null argument"; return B2_ERR_INVALID_ARG; }
  return h->collect_scanned_rows_per_range(rows, n_inout);
}
int32_t b2_exec_encode_batch(b2_exec* h, int32_t encode_type, int32_t location, b2_encoded_chunk* out) {
  if (!h || !out) { g_last_error = "null argument"; return B2_ERR_INVALID_ARG; }
  return h->encode_batch(encode_type, location, out);
}
void b2_exec_close(b2_exec* h) {
  if (h && h->async_running) h->async_fut.wait();  // a batch still in flight
  delete h;
}

int32_t b2_exec_agg_partials(b2_exec* h, b2_agg_partials* out) {
  if (h->cp.dev.mode != PM_AGG || !h->drained) { g_last_error = "no aggregation state: not an Aggregation pipeline or not drained yet"; return B2_ERR_INVALID_ARG; }
  out->n_groups = h->part_n; out->acc_words = (uint32_t)h->cp.dev.acc_words; out->location = B2_LOC_DEVICE; out->has_group = h->cp.dev.has_group;
  out->keys = (const uint64_t*)h->part_keys; out->key_null = (const uint8_t*)h->part_null; out->acc = (const uint64_t*)h->part_acc;
  out->max_word_mask = 0;
  out->key_words = (uint32_t)std::max(1, h->cp.dev.n_group); out->_pad = 0;
  for (int a = 0; a < h->cp.dev.n_aggs; ++a)
    if (agg_is_extremum(h->cp.dev.aggs[a].kind)) out->max_word_mask |= 1ull << (h->cp.dev.aggs[a].acc_off + 1);
  return B2_OK;
}
int32_t b2_exec_agg_word_ops(b2_exec* h, uint8_t* ops, uint32_t* n_inout) {
  if (!h || !ops || !n_inout) { g_last_error = "null argument"; return B2_ERR_INVALID_ARG; }
  if (h->cp.dev.mode != PM_AGG || !h->drained) { g_last_error = "no aggregation state: not an Aggregation pipeline or not drained yet"; return B2_ERR_INVALID_ARG; }
  const uint32_t n = (uint32_t)h->cp.dev.acc_words;
  if (*n_inout < n) { *n_inout = n; g_last_error = "ops buffer smaller than acc_words"; return B2_ERR_INVALID_ARG; }
  for (uint32_t w = 0; w < n; ++w) ops[w] = (uint8_t)agg_word_op(h->cp.dev, (int)w);
  *n_inout = n;
  return B2_OK;
}

int32_t b2_dag_handle(const b2_dag_plan* plan, const b2_key_range* ranges, uint32_t n_ranges, const b2_region_source* src,
                      const b2_exec_config* cfg, b2_batch* out, b2_exec** out_handle) {
  b2_exec* h = nullptr;
  int rc = b2_exec_open(plan, ranges, n_ranges, src, cfg, &h);
  if (rc) return rc;
  *out_handle = h;
  if (h->paging_size) {
    // runner.rs:790-806: a paging request stops after the batch in which `paging_size` rows have been produced and
    // hands back the scanned range.  One bounded batch here (rows come in key order, so any prefix is a valid page): the
    // batch covers enough entries for the page on an unselective plan; a selective one simply returns a shorter page.
    const uint64_t budget = std::min<uint64_t>(std::max<uint64_t>(h->paging_size * 2, 64), 1ull << 24);
    rc = h->next_batch(budget, out);
    if (rc == B2_OK && out->is_drained == B2_DRAIN_REMAIN) out->is_drained = B2_DRAIN_PAGING;
    return rc;
  }
  // run to drain in one batch: aggregations always do; scans process every unit in one go when the source is one chunk
  return h->next_batch(~0ull, out);
}

// ---- async next_batch: the batch runs on a worker thread of the handle, the caller polls ----
int32_t b2_exec_next_batch_async(b2_exec* h, uint64_t scan_rows) {
  if (!h) { g_last_error = "null argument"; return B2_ERR_INVALID_ARG; }
  if (h->async_running) { g_last_error = "a batch is already in flight on this handle"; return B2_ERR_INVALID_ARG; }
  h->async_running = true;
  h->async_fut = std::async(std::launch::async, [h, scan_rows] { return h->next_batch(scan_rows, &h->async_batch); });
  return B2_OK;
}
int32_t b2_exec_poll(b2_exec* h, b2_batch* out) {
  if (!h || !out) { g_last_error = "null argument"; return B2_ERR_INVALID_ARG; }
  if (!h->async_running) { g_last_error = "no batch in flight"; return B2_ERR_INVALID_ARG; }
  if (h->async_fut.wait_for(std::chrono::seconds(0)) != std::future_status::ready) return B2_PENDING;
  const int rc = h->async_fut.get();
  h->async_running = false;
  *out = h->async_batch;
  if (rc) g_last_error = h->last_err.message;
  return rc;
}

int32_t b2_exec_warnings(b2_exec* h, b2_warning* out, uint32_t cap, uint64_t* count_out) {
  if (!h || !count_out) { g_last_error = "null argument"; return B2_ERR_INVALID_ARG; }
  *count_out = h->warnings_total;
  const uint64_t n = std::min<uint64_t>(std::min<uint64_t>(h->warnings_total, cap), 64);  // DEFAULT_MAX_WARNING_CNT, expr/ctx.rs:62
  for (uint64_t i = 0; out && i < n; ++i) {
    out[i].mysql_code = B2_MYSQL_ERR_DIVISION_BY_ZERO; out[i]._pad = 0;
    snprintf(out[i].message, sizeof(out[i].message), "Division by 0");
  }
  return B2_OK;
}

// ---- HBM-resident block cache ----
namespace {
struct PinnedRegion {
  std::vector<DevBuf> bufs;
  std::vector<b2_cf_block> write, dflt;
  b2_cf_block lock{};
  std::vector<std::vector<uint8_t>> lock_host;  // CF_LOCK stays in host memory (the ABI reads it on the host)
  std::vector<uint32_t> lock_ko, lock_vo;
  bool has_lock = false;
  uint64_t bytes = 0;
  int refs = 0;
};
struct CacheKey { int device; uint64_t region, version; bool operator<(const CacheKey& o) const { return device != o.device ? device < o.device : (region != o.region ? region < o.region : version < o.version); } };
std::mutex g_cache_mu;
std::map<CacheKey, std::unique_ptr<PinnedRegion>>& region_cache() { static auto* m = new std::map<CacheKey, std::unique_ptr<PinnedRegion>>(); return *m; }
uint64_t g_cache_bytes[64] = {0}, g_cache_hits[64] = {0}, g_cache_misses[64] = {0};
uint64_t cache_budget() {  // B2_BLOCK_CACHE_BYTES, else three quarters of the current device's memory
  if (const char* v = getenv("B2_BLOCK_CACHE_BYTES")) return strtoull(v, nullptr, 10);
  size_t fr = 0, tot = 0;
  if (cudaMemGetInfo(&fr, &tot) != cudaSuccess || !tot) return 64ull << 30;
  return (uint64_t)tot / 4 * 3;
}
}  // namespace

int32_t b2_region_pin(int32_t device, uint64_t region_id, uint64_t data_version, const b2_region_source* src, b2_region_source* out) {
  if (!src || !out || src->location != B2_LOC_HOST || device < 0 || device >= 64) { g_last_error = "b2_region_pin: a host-resident source and a device ordinal below 64 are required"; return B2_ERR_INVALID_ARG; }
  if (cudaSetDevice(device) != cudaSuccess) { g_last_error = "cudaSetDevice failed"; return B2_ERR_CUDA; }
  std::lock_guard<std::mutex> g(g_cache_mu);
  const CacheKey key{device, region_id, data_version};
  auto it = region_cache().find(key);
  if (it == region_cache().end()) {
    g_cache_misses[device]++;
    std::unique_ptr<PinnedRegion> pr(new PinnedRegion());
    uint64_t need = 0;
    auto sizes = [&](const b2_cf_block& b, uint64_t* kb, uint64_t* vb) { *kb = b.n ? b.key_offs[b.n] : 0; *vb = b.n ? b.val_offs[b.n] : 0; };
    for (uint32_t i = 0; i < src->n_write; ++i) { uint64_t kb, vb; sizes(src->write[i], &kb, &vb); need += kb + vb + 8ull * (src->write[i].n + 1) + 128; }
    for (uint32_t i = 0; src->dflt && i < src->n_dflt; ++i) { uint64_t kb, vb; sizes(src->dflt[i], &kb, &vb); need += kb + vb + 8ull * (src->dflt[i].n + 1) + 128; }
    if (g_cache_bytes[device] + need > cache_budget()) { g_last_error = "block cache budget exceeded (B2_BLOCK_CACHE_BYTES)"; return B2_ERR_UNSUPPORTED; }
    cudaStream_t st;
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) { g_last_error = "cudaStreamCreate failed"; return B2_ERR_CUDA; }
    bool ok = true;
    auto up = [&](const void* p, size_t bytes) -> const void* {
      pr->bufs.emplace_back();
      DevBuf& d = pr->bufs.back();
      if (d.reserve(((bytes + 31) & ~(size_t)15) + 16) != cudaSuccess) { ok = false; return nullptr; }
      if (bytes && cudaMemcpyAsync(d.p, p, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) ok = false;
      return d.p;
    };
    auto copy_blocks = [&](const b2_cf_block* bs, uint32_t n, std::vector<b2_cf_block>* dst) {
      for (uint32_t i = 0; i < n && ok; ++i) {
        uint64_t kb, vb; sizes(bs[i], &kb, &vb);
        b2_cf_block d{};
        d.keys = (const uint8_t*)up(bs[i].keys, kb); d.key_offs = (const uint32_t*)up(bs[i].key_offs, 4ull * (bs[i].n + 1));
        d.vals = (const uint8_t*)up(bs[i].vals, vb); d.val_offs = (const uint32_t*)up(bs[i].val_offs, 4ull * (bs[i].n + 1));
        d.n = bs[i].n;
        dst->push_back(d);
      }
    };
    copy_blocks(src->write, src->n_write, &pr->write);
    if (src->dflt) copy_blocks(src->dflt, src->n_dflt, &pr->dflt);
    if (ok && cudaStreamSynchronize(st) != cudaSuccess) ok = false;
    cudaStreamDestroy(st);
    if (!ok) { g_last_error = "block cache: device allocation or copy failed"; return B2_ERR_CUDA; }
    if (src->lock && src->lock->n) {  // keep a private host copy of CF_LOCK
      const b2_cf_block& L = *src->lock;
      pr->lock_host.resize(2);
      pr->lock_host[0].assign(L.keys, L.keys + L.key_offs[L.n]); pr->lock_host[1].assign(L.vals, L.vals + L.val_offs[L.n]);
      pr->lock_ko.assign(L.key_offs, L.key_offs + L.n + 1); pr->lock_vo.assign(L.val_offs, L.val_offs + L.n + 1);
      pr->lock.keys = pr->lock_host[0].data(); pr->lock.key_offs = pr->lock_ko.data(); pr->lock.vals = pr->lock_host[1].data(); pr->lock.val_offs = pr->lock_vo.data(); pr->lock.n = L.n;
      pr->has_lock = true;
    }
    pr->bytes = need;
    g_cache_bytes[device] += need;
    it = region_cache().emplace(key, std::move(pr)).first;
  } else g_cache_hits[device]++;
  PinnedRegion& pr = *it->second;
  pr.refs++;
  *out = *src;
  out->location = B2_LOC_DEVICE; out->device = device;
  out->write = pr.write.data(); out->n_write = (uint32_t)pr.write.size();
  out->dflt = pr.dflt.empty() ? nullptr : pr.dflt.data(); out->n_dflt = (uint32_t)pr.dflt.size();
  out->lock = pr.has_lock ? &pr.lock : nullptr;
  return B2_OK;
}
int32_t b2_region_unpin(int32_t device, uint64_t region_id, uint64_t data_version) {
  std::lock_guard<std::mutex> g(g_cache_mu);
  auto it = region_cache().find(CacheKey{device, region_id, data_version});
  if (it == region_cache().end()) { g_last_error = "b2_region_unpin: not pinned"; return B2_ERR_INVALID_ARG; }
  if (--it->second->refs > 0) return B2_OK;
  cudaSetDevice(device);
  cudaDeviceSynchronize();  // requests still reading the cached blocks
  g_cache_bytes[device] -= it->second->bytes;
  region_cache().erase(it);
  return B2_OK;
}
void b2_region_cache_stats(int32_t device, uint64_t* bytes_cached, uint64_t* hits, uint64_t* misses) {
  std::lock_guard<std::mutex> g(g_cache_mu);
  const int d = device >= 0 && device < 64 ? device : 0;
  if (bytes_cached) *bytes_cached = g_cache_bytes[d];
  if (hits) *hits = g_cache_hits[d];
  if (misses) *misses = g_cache_misses[d];
}

int32_t b2_checksum_handle(const b2_key_range* ranges, uint32_t n_ranges, const uint8_t* old_prefix, uint32_t old_prefix_len,
                           const uint8_t* new_prefix, uint32_t new_prefix_len, const b2_region_source* src, const b2_exec_config* cfg,
                           b2_checksum_response* out, b2_exec_stats* stats) {
  std::unique_ptr<b2_exec> h(new b2_exec());
  h->device = src->device;
  cudaError_t e = cudaSetDevice(h->device);
  if (e != cudaSuccess) { g_last_error = std::string("cudaSetDevice: ") + cudaGetErrorString(e); return B2_ERR_CUDA; }
  if (h->open_streams(cfg) != cudaSuccess) return B2_ERR_CUDA;
  memset(&h->cp.dev, 0, sizeof(h->cp.dev));
  h->cp.dev.mode = PM_CHECKSUM;
  int rc = h->setup_source(src, ranges, n_ranges);
  if (rc) { g_last_error = h->last_err.message; return rc; }
  rc = h->init_device_state();
  if (rc) return rc;
  // crc register after the old prefix (checksum.rs:75-76 prefix_digest)
  uint64_t st = ~0ull;
  for (uint32_t i = 0; i < old_prefix_len; ++i) st = crc64_table_entry((uint8_t)(st ^ old_prefix[i])) ^ (st >> 8);
  if (new_prefix_len > 32) { g_last_error = "new_prefix longer than 32 bytes"; return B2_ERR_UNSUPPORTED; }
  h->cp.dev.read_ts = h->read_ts; h->cp.dev.isolation = h->isolation;
  for (size_t ui = 0; ui < h->units.size(); ++ui) {
    const Unit& u = h->units[ui];
    BlockView v;
    rc = h->acquire_block(u.block_idx, &v);
    if (rc) return rc;
    ScanArgs a = h->base_args(u, v);
    a.c_lo = u.e_lo; a.c_hi = u.e_hi;
    a.ck_init_state = st; a.ck_new_prefix_len = new_prefix_len; a.ck_old_prefix_len = old_prefix_len;
    memcpy(a.ck_new_prefix, new_prefix, new_prefix_len);
    // lean kernel: the unit's keys share their first 11 raw bytes ('t' table-id "_r"); the crc register after old_prefix and
    // raw[new_prefix_len .. 11) is the same for all of them.  (A new_prefix that reaches into the handle, or that the
    // unit's keys do not start with, is left to the general kernel, which also raises "Wrong prefix".)
    bool fast = u.fast_ok && h->fast_kernel_covers() && new_prefix_len <= 11;
    if (fast) {
      uint8_t raw[11];
      const uint8_t* enc = (const uint8_t*)u.prefix;
      for (int j = 0; j < 8; ++j) raw[j] = enc[j];
      for (int j = 8; j < 11; ++j) raw[j] = enc[j + 1];
      uint64_t ks = st;
      for (uint32_t j = 0; j < new_prefix_len && fast; ++j) fast = raw[j] == new_prefix[j];
      for (uint32_t j = new_prefix_len; j < 11; ++j) ks = crc64_table_entry((uint8_t)(ks ^ raw[j])) ^ (ks >> 8);
      a.ck_key_state = ks;
    }
    rc = h->launch_unit(a, u, fast, scan_crc_table_bytes(), fast_checksum_bytes(), 0, nullptr, nullptr);
    if (rc) return rc;
    h->release_block(u.block_idx);
    h->prefetch_after(ui);
    h->entries_scanned += u.e_hi - u.e_lo;
  }
  Counters c;
  rc = h->read_counters(&c);
  if (rc) return rc;
  h->fill_stats(c);
  if (stats) *stats = h->stats;
  if (c.err != ~0ull) {
    if (c.bad_prefix) { g_last_error = "Wrong prefix expect"; return B2_ERR_STORAGE; }
    h->device_error(c);
    return h->last_err.status;
  }
  h->check_trailing_lock();
  if (h->failed) return h->last_err.status;
  out->checksum = c.checksum; out->total_kvs = c.total_kvs; out->total_bytes = c.total_bytes;
  return B2_OK;
}

// ---- generator -----------------------------------------------------------------------------------------------
struct b2_gen {
  int device = 0;
  DevBuf keys, koff, vals, voff, row_entries, row_vals, scan_tmp, d_lo, d_range, d_null;
};

int32_t b2_gen_create(int32_t device, const b2_gen_spec* spec, b2_gen** out, b2_gen_block* out_block) {
  if (!spec || !out || !out_block) return B2_ERR_INVALID_ARG;
  if (spec->n_cols == 0 || spec->n_cols > 24 || (spec->row_format != 1 && spec->row_format != 2) || spec->commit_ts < 12 || spec->n_rows >= (1ull << 31)) {
    g_last_error = "generator spec out of range (1..24 columns, row format 1|2, commit_ts >= 12, < 2^31 rows)";
    return B2_ERR_INVALID_ARG;
  }
  if (cudaSetDevice(device) != cudaSuccess) { g_last_error = "cudaSetDevice failed"; return B2_ERR_CUDA; }
  std::unique_ptr<b2_gen> g(new b2_gen());
  g->device = device;
  b2_gen_spec s = *spec;
  size_t n = spec->n_rows, nc = spec->n_cols;
#define GEN_TRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { g_last_error = std::string(#x) + ": " + cudaGetErrorString(_e); return B2_ERR_CUDA; } } while (0)
  GEN_TRY(g->d_lo.reserve(nc * 8)); GEN_TRY(g->d_range.reserve(nc * 8)); GEN_TRY(g->d_null.reserve(nc * 4));
  std::vector<int64_t> lo(nc, 0); std::vector<uint64_t> range(nc, 0); std::vector<uint32_t> nul(nc, 0);
  for (size_t c = 0; c < nc; ++c) { if (spec->col_lo) lo[c] = spec->col_lo[c]; if (spec->col_range) range[c] = spec->col_range[c]; if (spec->null_per_million) nul[c] = spec->null_per_million[c]; }
  GEN_TRY(cudaMemcpy(g->d_lo.p, lo.data(), nc * 8, cudaMemcpyHostToDevice));
  GEN_TRY(cudaMemcpy(g->d_range.p, range.data(), nc * 8, cudaMemcpyHostToDevice));
  GEN_TRY(cudaMemcpy(g->d_null.p, nul.data(), nc * 4, cudaMemcpyHostToDevice));
  s.col_lo = (const int64_t*)g->d_lo.p; s.col_range = (const uint64_t*)g->d_range.p; s.null_per_million = (const uint32_t*)g->d_null.p;
  GEN_TRY(g->row_entries.reserve((n + 1) * 4)); GEN_TRY(g->row_vals.reserve((n + 1) * 4));
  GEN_TRY(cudaMemset(g->row_entries.p, 0, (n + 1) * 4)); GEN_TRY(cudaMemset(g->row_vals.p, 0, (n + 1) * 4));
  GEN_TRY(launch_gen_sizes(s, (uint32_t*)g->row_entries.p, (uint32_t*)g->row_vals.p, 0));
  size_t tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, (uint32_t*)g->row_entries.p, (uint32_t*)g->row_entries.p, (int)(n + 1));
  GEN_TRY(g->scan_tmp.reserve(tmp_bytes + 16));
  // 32-bit prefix sums: value heap must stay below 4 GiB (u32 offsets of the block format)
  GEN_TRY(cub::DeviceScan::ExclusiveSum(g->scan_tmp.p, tmp_bytes, (uint32_t*)g->row_entries.p, (uint32_t*)g->row_entries.p, (int)(n + 1)));
  GEN_TRY(cub::DeviceScan::ExclusiveSum(g->scan_tmp.p, tmp_bytes, (uint32_t*)g->row_vals.p, (uint32_t*)g->row_vals.p, (int)(n + 1)));
  uint32_t n_entries = 0, val_bytes = 0;
  GEN_TRY(cudaMemcpy(&n_entries, (uint32_t*)g->row_entries.p + n, 4, cudaMemcpyDeviceToHost));
  GEN_TRY(cudaMemcpy(&val_bytes, (uint32_t*)g->row_vals.p + n, 4, cudaMemcpyDeviceToHost));
  // guard against u32 wrap of the value heap (rows are < 300 bytes each)
  if ((uint64_t)n * 16 > 0xffffffffull && val_bytes < n) { g_last_error = "generated value heap exceeds 4 GiB; use more, smaller blocks"; return B2_ERR_INVALID_ARG; }
  uint64_t key_bytes = (uint64_t)n_entries * 35;
  if (key_bytes > 0xfffffff0ull) { g_last_error = "generated key heap exceeds 4 GiB; use more, smaller blocks"; return B2_ERR_INVALID_ARG; }
  GEN_TRY(g->keys.reserve(((size_t)key_bytes + 31) & ~15ull)); GEN_TRY(g->vals.reserve(((size_t)val_bytes + 31) & ~15ull));
  GEN_TRY(g->koff.reserve(((size_t)n_entries + 1) * 4)); GEN_TRY(g->voff.reserve(((size_t)n_entries + 1) * 4));
  GenArgs a;
  a.spec = s; a.keys = (uint8_t*)g->keys.p; a.koff = (uint32_t*)g->koff.p; a.vals = (uint8_t*)g->vals.p; a.voff = (uint32_t*)g->voff.p;
  a.row_entry_off = (const uint32_t*)g->row_entries.p; a.row_val_off = (const uint32_t*)g->row_vals.p;
  GEN_TRY(launch_gen_write(a, 0));
  GEN_TRY(cudaDeviceSynchronize());
  g->row_entries.release(); g->row_vals.release(); g->scan_tmp.release();
  memset(out_block, 0, sizeof(*out_block));
  out_block->block.keys = (const uint8_t*)g->keys.p; out_block->block.key_offs = (const uint32_t*)g->koff.p;
  out_block->block.vals = (const uint8_t*)g->vals.p; out_block->block.val_offs = (const uint32_t*)g->voff.p;
  out_block->block.n = n_entries;
  out_block->key_bytes = key_bytes; out_block->val_bytes = val_bytes; out_block->n_user_keys = n;
  *out = g.release();
  return B2_OK;
#undef GEN_TRY
}

void b2_gen_destroy(b2_gen* g) {
  if (!g) return;
  cudaSetDevice(g->device);  // (the buffers go back to this device's pool)
  delete g;
}

int32_t b2_copy_to_host(int32_t device, void* dst, const void* src_device, uint64_t bytes) {
  if (cudaSetDevice(device) != cudaSuccess) return B2_ERR_CUDA;
  cudaError_t e = cudaMemcpy(dst, src_device, bytes, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) { g_last_error = cudaGetErrorString(e); return B2_ERR_CUDA; }
  return B2_OK;
}
int32_t b2_copy_to_device(int32_t device, void* dst_device, const void* src, uint64_t bytes) {
  if (cudaSetDevice(device) != cudaSuccess) return B2_ERR_CUDA;
  cudaError_t e = cudaMemcpy(dst_device, src, bytes, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { g_last_error = cudaGetErrorString(e); return B2_ERR_CUDA; }
  return B2_OK;
}
int32_t b2_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0; return n; }
void* b2_host_alloc_pinned(uint64_t bytes) { void* p = nullptr; if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr; return p; }

// Pinned host memory on the NUMA node the GPU hangs off (staging buffers of host-resident sources: on a two-socket box a
// buffer on the far socket halves the H2D rate of GPUs 4-7).  The node comes from sysfs (PCI bus id of the device); the
// pages are bound with mbind(MPOL_BIND) before they are touched, then pinned with cudaHostRegister.  Falls back to
// cudaMallocHost when any step is unavailable.  Free with b2_host_free_pinned.
static std::mutex g_near_mu;
static std::vector<std::pair<void*, size_t>>& near_allocs() { static std::vector<std::pair<void*, size_t>> v; return v; }
static int gpu_numa_node(int device) {
  char bus[32];
  if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) return -1;
  for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
  std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
  FILE* f = fopen(path.c_str(), "r");
  if (!f) return -1;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  return node;
}
void* b2_host_alloc_pinned_near(int32_t device, uint64_t bytes) {
  const int node = gpu_numa_node(device);
  if (node >= 0 && node < 64 && bytes) {
    const size_t len = ((size_t)bytes + 4095) & ~(size_t)4095;
    void* p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (p != MAP_FAILED) {
      unsigned long mask = 1ul << node;
      long rc = syscall(SYS_mbind, p, len, 2 /* MPOL_BIND */, &mask, 65ul, 0u);
      if (rc == 0 && cudaSetDevice(device) == cudaSuccess && cudaHostRegister(p, len, cudaHostRegisterPortable) == cudaSuccess) {
        std::lock_guard<std::mutex> g(g_near_mu);
        near_allocs().push_back({p, len});
        return p;
      }
      cudaGetLastError();
      munmap(p, len);
    }
  }
  return b2_host_alloc_pinned(bytes);
}
int32_t b2_device_numa_node(int32_t device) { return gpu_numa_node(device); }
void b2_host_free_pinned(void* p) {
  if (!p) return;
  {
    std::lock_guard<std::mutex> g(g_near_mu);
    auto& v = near_allocs();
    for (size_t i = 0; i < v.size(); ++i)
      if (v[i].first == p) {
        cudaHostUnregister(p);
        munmap(p, v[i].second);
        v.erase(v.begin() + i);
        return;
      }
  }
  cudaFreeHost(p);
}

}  // extern "C"
