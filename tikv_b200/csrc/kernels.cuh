// Kernel-side structures and launch wrappers shared by kernels.cu (device) and engine.cu (host).
#pragma once
#ifndef B2_NVRTC
#include <cuda_runtime.h>
#endif

#include "b2_device.h"

namespace b2 {

enum { TILE = 256 };  // entries per tile = threads per CTA

// Counters accumulated across all launches of one request (device memory, zero-initialised except err).
struct Counters {
  unsigned long long err;              // min over failing rows of (global_entry << 8 | DevErr); ~0 = none
  unsigned long long out_rows;         // rows written by PM_SCAN launches (reset per batch by the host)
  unsigned long long out_base;         // rows written by earlier launches of the same batch (copied from out_rows between launches)
  unsigned long long live_rows;        // rows that passed MVCC + selection
  unsigned long long processed_keys;   // rows returned by the MVCC scan
  unsigned long long processed_size;   // sum(len(user_key) + len(value))
  unsigned long long entries_scanned;  // CF_WRITE entries covered
  unsigned long long default_lookups;
  unsigned long long checksum, total_kvs, total_bytes;  // checksum mode
  unsigned int met_newer;
  unsigned int agg_overflow;           // global group table full
  unsigned int n_groups;               // finalize: number of groups emitted
  unsigned int bad_prefix;             // checksum: key without new_prefix
  unsigned long long last_row;         // 1 + largest global CF_WRITE entry index the MVCC scan returned a row for (take_scanned_range)
  unsigned long long err_max;          // max over failing rows of (global_entry << 8 | DevErr): the first error of a backward scan; 0 = none
  unsigned long long warn_div0;        // "Division by 0" warnings (1365) raised on committed rows
  unsigned long long first_row;        // smallest global CF_WRITE entry index a row was returned for (take_scanned_range, backward); ~0 = none
  unsigned int agg_stuck;              // composite-key inserts that gave up waiting for a claimed slot's key (the request fails)
  unsigned int agg_probe_max;          // longest composite-key probe run above 64 slots (reported with agg_stuck)
};

// Open-addressing group table in HBM (fast_hash_aggr_executor.rs:216-229 `Groups`): slot = hash(key) & mask, linear
// probing on the key words themselves: a free slot holds AGG_EMPTY_KEY and is claimed with one 64-bit CAS (accumulators
// start at zero and are only added to, so a claimed slot needs no further initialisation).  Slot `cap` is the NULL-key
// group, slot `cap + 1` the group whose key equals AGG_EMPTY_KEY; `special[0..1]` say whether those two are in use.
#define AGG_EMPTY_KEY 0xffffffffffffffffull
#define AGG_MAX_PROBES 4096u  // longest probe run of a key; a longer one counts as a full table (grow and redo)
struct AggTable {
  unsigned long long* keys;  // cap + 2
  unsigned int* special;     // 2
  unsigned long long* acc;   // (cap + 2) * acc_words
  unsigned int cap;          // power of two
  // grouped by several expressions (PM_AGGM): `keys` holds a 64-bit hash tag of the composite key; the key itself is
  // gkeys[slot * (n_group + 1) ..] = n_group value words + the NULL mask, valid once ready[slot] != 0
  unsigned int hash_mask_bits;  // debug (B2_DEBUG_AGG_HASH_BITS): keep only this many hash bits, 0 = all 64
  unsigned long long* gkeys;
  unsigned int* ready;
};

struct TopNLists {
  TopItem* items;        // n_lists * stride
  unsigned int* counts;  // n_lists
  unsigned int n_lists, stride;
};

// One unit of a lean launch (fast_kernel.cuh): the launch walks the tiles of a table of these, claimed from one counter.
// Tiles never straddle units.
struct UnitDesc {
  BlockView blk;
  uint32_t e_lo;                    // first entry of the unit (the look-back of its first tile stops there)
  uint32_t c_lo, c_hi;              // the entries this launch covers (runs *starting* in [c_lo, c_hi))
  uint32_t tile_lo;                 // tiles of the units before this one in the table
  uint64_t entry_base;              // global index of blk entry 0
  unsigned long long* range_rows;   // the unit's scanned_rows_per_range slot, or nullptr
  uint64_t ck_key_state;            // checksum: see ScanArgs::ck_key_state
  uint64_t slow_off;                // the unit's segment of ScanArgs::slow_list
};

struct ScanArgs {
  BlockView blk;
  DefaultCf dflt;
  uint32_t e_lo, e_hi;  // entries of the block inside the key range
  uint32_t c_lo, c_hi;  // chunk handled by this launch (runs *starting* in [c_lo, c_hi))
  uint64_t entry_base;  // global index of blk entry 0
  uint64_t read_ts;     // snapshot timestamp of the request
  int32_t isolation;    // B2_ISO_* of the request
  int32_t _pad0;
  Counters* ctr;
  unsigned long long* range_rows;   // rows the MVCC scan returned inside this unit's key range (scanned_rows_per_range), or nullptr
  // PM_SCAN
  unsigned long long* tile_status;  // n_tiles + 1 words, zeroed per launch; last word = ticket
  unsigned long long* out_data;     // n_out columns, each `out_cap` u64 cells
  unsigned long long* out_bitmap;   // n_out columns, each out_cap/64 words pre-filled with 1s
  uint64_t out_cap;
  // PM_AGG
  AggTable tbl;
  uint32_t staging;                 // 1: stage tiles through shared memory with bulk copies
  uint32_t stage_off;               // byte offset of the stages inside dynamic shared memory (multiple of 16)
  uint32_t out_stage_off;           // PM_SCAN: byte offset of the output transpose buffer (multiple of 16)
  uint32_t stage_key_cap, stage_val_cap;  // bytes per stage for key / value heaps (multiples of 16)
  int64_t imms[MAX_IMMS];           // the request's constants (DevNode::sig / FastCond::imm_slot index them)
  uint64_t limit;                   // TopN limit (not part of the compiled plan shape)
  // hand-over between the lean kernel (fast_kernel.cuh) and the general one: first entries of the runs the lean kernel left alone
  unsigned int* slow_list;          // capacity >= c_hi - c_lo
  unsigned int* slow_count;
  uint32_t list_mode;               // scan_body: 1 = process the entries of slow_list (count read on the device) instead of [c_lo, c_hi)
  uint32_t smem_slots;              // PM_AGG: per-CTA table slots (power of two), 0 = disabled.  Kept in this padding slot: every
                                    //    other field keeps its alignment, which decides how the kernels load their parameters
  uint64_t ck_key_state;            // lean checksum: crc register after old_prefix and the unit's common raw key bytes [new_prefix_len, 11)
  uint32_t desc;                    // backward scan (TableScan.desc): TopN ties go to the larger key (item ids are complemented)
  uint32_t _pad3;
  uint32_t fast_ok;                 // 1: every key of [e_lo, e_hi) starts with the same 12 bytes 't' tid "_r" (first and last key of the
                                    //    sorted unit agree): the clean-entry front end may skip them
  uint32_t _pad1;
  // PM_CHECKSUM
  uint64_t ck_init_state;           // crc register after old_prefix
  uint32_t ck_new_prefix_len, ck_old_prefix_len;
  uint8_t ck_new_prefix[32];
  // PM_TOPN
  TopNLists topn;                   // per-CTA result lists (stride = limit)
  uint32_t topn_cap;                // candidate capacity of a CTA (engine.cu run_topn: power of two >= limit + TILE, 8192 above LIMIT 2048)
  const TopItem* topn_seed;         // running top-N of the units already merged (sorted), or nullptr:
  const unsigned int* topn_seed_cnt;  //   once it holds `limit` rows its last one is every CTA's initial threshold
  unsigned char* topn_work;           // lean TopN kernel: the CTAs' candidate buffers live in HBM / L2 (topn_work + blockIdx.x * stride): a
  unsigned long long topn_work_stride;//   seeded CTA touches its buffer for a handful of rows per launch, and shared memory buys a third CTA per SM.
                                      //   Above LIMIT 2048 the general kernel's buffers live there too (scan_topn_hbm_kernel)
  // the lean kernel: its units (it reads none of blk, e_lo, c_lo, c_hi, entry_base, range_rows, ck_key_state above), the
  // counter its CTAs claim tiles from (zeroed before the launch), and per unit a hand-over count (slow_count[u]) and segment
  // (slow_list + units[u].slow_off)
  const UnitDesc* units;
  unsigned int* tile_ctr;
  uint32_t n_units, n_unit_tiles;
};

struct GenArgs {
  b2_gen_spec spec;  // pointers inside are device pointers
  uint8_t* keys; uint32_t* koff; uint8_t* vals; uint32_t* voff;
  const uint32_t* row_entry_off;   // exclusive scan of entries per row (n_rows + 1)
  const uint32_t* row_val_off;     // exclusive scan of value bytes per row (n_rows + 1)
};

#ifndef B2_NVRTC
// launchers (kernels.cu)
cudaError_t launch_scan(const DevPlan& plan, const ScanArgs& a, int grid, size_t smem, cudaStream_t s);
// the lean kernels (fast_kernel.cuh): PM_AGG (at most one group-by expression, no Real sums), PM_TOPN, PM_CHECKSUM
cudaError_t launch_fast(const DevPlan& plan, const ScanArgs& a, int grid, size_t smem, cudaStream_t s);
int fast_max_grid(int mode, size_t smem);
size_t fast_stage_bytes(uint32_t key_cap, uint32_t val_cap);
size_t fast_checksum_bytes();             // PM_CHECKSUM tables + per-length key states
int scan_max_grid(int mode, size_t smem);  // occupancy-based persistent grid size
// the general TopN kernel with its candidate buffers in HBM (a.topn_work; LIMIT above 2048): grid size, launch
int scan_topn_hbm_max_grid(size_t smem);
cudaError_t launch_scan_topn_hbm(const DevPlan& plan, const ScanArgs& a, int grid, size_t smem, cudaStream_t s);
int scan_num_sms();
size_t scan_stage_bytes(uint32_t key_cap, uint32_t val_cap);  // dynamic shared memory needed by the tile stages
size_t scan_crc_table_bytes();             // PM_CHECKSUM replicated CRC table
int scan_kernel_mode(const DevPlan& plan);  // PM_* instantiation that serves `plan`
size_t scan_out_stage_bytes();             // PM_SCAN output transpose buffer
uint32_t scan_stage_entries();             // entries a stage must hold (tile + look-behind/ahead)
// n_group >= 2: out_keys holds n_group words per group, out_key_null the group's NULL mask (bit q = q-th expression)
cudaError_t launch_agg_finalize(const DevPlan& plan, const AggTable& t, Counters* ctr, unsigned long long* out_keys, unsigned char* out_key_null,
                                unsigned long long* out_acc, cudaStream_t s);
cudaError_t launch_agg_result(const DevPlan& plan, unsigned int n_groups, const unsigned long long* g_keys, const unsigned char* g_null,
                              const unsigned long long* g_acc, unsigned long long** col_data, unsigned long long** col_bitmap, cudaStream_t s);
// TopN: merge every `fan_in` (<= 16) lists of `in` into the best `limit` items (sorted) -> one list of `out`; gather decodes
// the rows of a list
cudaError_t launch_topn_merge(const DevPlan& plan, const TopNLists& in, const TopNLists& out, uint32_t fan_in, cudaStream_t s);
cudaError_t launch_topn_gather(const DevPlan& plan, const ScanArgs& a, const TopItem* items, const unsigned int* count, unsigned long long* pay,
                               unsigned char* pay_null, uint32_t stride, cudaStream_t s);
cudaError_t launch_topn_copy(const TopItem* items, const unsigned int* count, uint32_t n_out, uint32_t stride, const unsigned long long* pay0,
                             const unsigned char* null0, const unsigned long long* pay1, const unsigned char* null1, unsigned long long* pay_out,
                             unsigned char* null_out, cudaStream_t s);
cudaError_t launch_topn_merge2(const DevPlan& plan, const TopItem* a, const unsigned int* a_cnt, const TopItem* b, const unsigned int* b_cnt, TopItem* out,
                               unsigned int* out_cnt, uint32_t limit, cudaStream_t s);
cudaError_t launch_pack_nulls(const unsigned char* nulls, uint32_t n_cols, uint32_t stride, uint32_t n, unsigned long long* bitmaps, uint32_t words_per_col, cudaStream_t s);
size_t topn_smem_bytes(uint32_t cap, int n_order);
// What opening a request over device-resident blocks reads from them.  blocks: the n_wblocks CF_WRITE blocks, then the
// CF_DEFAULT ones (n_blocks in all).  out: lower_bound of every range bound (lo, hi per range) in every CF_WRITE block;
// unit_ok[block * n_ranges + range]: that unit's keys share a record-key prefix; ends: key_offs[n], val_offs[n] per block;
// sample: the byte count and first bytes of the first value of the first unit of the ranges from first_range on
cudaError_t launch_open_probe(const BlockView* blocks, uint32_t n_wblocks, uint32_t n_blocks, const uint8_t* bounds, const uint32_t* bound_offs, uint32_t n_ranges,
                              uint32_t first_range, uint32_t* out, uint32_t* unit_ok, uint32_t* ends, uint32_t* sample, cudaStream_t s);
cudaError_t launch_gen_sizes(const b2_gen_spec& spec, uint32_t* row_entries, uint32_t* row_val_bytes, cudaStream_t s);
cudaError_t launch_gen_write(const GenArgs& a, cudaStream_t s);
cudaError_t launch_fill_u64(unsigned long long* p, unsigned long long v, size_t n, cudaStream_t s);
// backward scans: out row i = in row (n_rows - 1 - i) for i < n_take, every column and its non-NULL bitmap; out bitmaps pre-filled with ones
// bytes / json / decimal output columns of the rows one scan launch appended (kernels.cu raw_*)
enum { MAX_RAW = 16 };
struct RawCol {
  unsigned long long* cells;      // the column's cell references (ScanArgs::out_data + column * out_cap)
  long long* offsets;             // var-length: out_cap + 1 offsets
  unsigned char* heap;            // var-length: byte heap; decimal: out_cap b2_decimal structs
  unsigned long long* heap_used;  // var-length: the heap cursor (device-resident, carried from launch to launch)
  unsigned long long heap_cap;
};
struct RawArgs {
  RawCol col[MAX_RAW];
  unsigned char var_idx[MAX_RAW], dec_idx[MAX_RAW];  // indices into col
  unsigned int n_var, n_dec;
  const unsigned long long* row_lo; const unsigned long long* row_hi;  // the launch's rows (device counters)
  unsigned long long* sums; unsigned long long sums_stride;            // scratch: n_var x ceil(max_rows / 1024)
  unsigned int* err;              // 1 = a decimal cell does not decode, 2 = heap overflow
};
cudaError_t launch_raw_materialise(const RawArgs& R, uint64_t max_rows, cudaStream_t s);
// Final merge of gathered partial tables (agg_merge.cu, b2_agg_merge): row r = keys[r * keys_stride ..] (key_words
// words), key_null[r] (NULL mask), acc[r * acc_stride ..] (acc_words state words); ops (acc_words B2_MERGE_*) and
// part_offs (n_parts + 1 row offsets) are device pointers.  Outputs have room for n groups; *n_groups (device) receives
// their number.
struct AggMergeArgs {
  const long long* keys;
  const unsigned char* key_null;
  const long long* acc;
  uint64_t keys_stride, acc_stride;
  uint32_t n, key_words, acc_words, n_parts;
  const unsigned char* ops;
  const unsigned long long* part_offs;
  int32_t desc;
  long long* out_keys;         // n_groups * key_words
  unsigned char* out_null;     // n_groups
  long long* out_acc;          // n_groups * acc_words
  unsigned int* n_groups;
};
// cub-style: tmp == nullptr stores the scratch bytes the merge needs in *tmp_bytes and launches nothing
cudaError_t launch_agg_merge(const AggMergeArgs& a, void* tmp, size_t* tmp_bytes, cudaStream_t s);
cudaError_t launch_reverse_rows(const unsigned long long* in, const unsigned long long* bm_in, uint64_t in_cap, unsigned long long* out, unsigned long long* bm_out,
                                uint64_t out_cap, uint64_t n_rows, uint64_t n_take, uint32_t n_cols, cudaStream_t s);

#endif  // !B2_NVRTC

}  // namespace b2
