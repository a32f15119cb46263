// Per-entry / per-row device logic of the coprocessor hot path (MVCC visibility, row decode, RPN).
// Every function is __host__ __device__ so tests/host_emul.cpp can drive exactly this code on the CPU
// (a debug harness; the product only ever runs it inside the sm_90a kernels in kernels.cu).
//
// Reference semantics being reproduced (tikv/tikv paths):
//   src/storage/mvcc/reader/scanner/forward.rs:172-515     latest-version forward scan
//   components/txn_types/src/write.rs:296-361, 425-442     write record
//   components/tidb_query_executors/src/table_scan_executor.rs:200-281, 365-475
//   components/tidb_query_datatype/src/codec/row/v2/{row_slice.rs:74-166,330-357, compat_v1.rs:13-129}
//   components/tidb_query_datatype/src/codec/{datum.rs:1117-1155, datum_codec.rs:401-446}
//   components/tidb_query_expr/src/{impl_compare.rs:63-240, impl_op.rs:8-127, impl_arithmetic.rs:42-398}
#pragma once
#ifndef B2_NVRTC
#include <stdint.h>
#include <math.h>
#endif

#include "../../include/b2_copr.h"

#if defined(__CUDACC__)
#define B2_HD __host__ __device__ __forceinline__
#define B2_HD_NOINLINE __host__ __device__ __noinline__
#else
#define B2_HD inline
#define B2_HD_NOINLINE inline
#endif
// Decoders that only the general (dirty-data / v1 / odd-row) paths call: out of line when jit.cu sets B2_COLD_OUTLINE (plans
// with the rarer scalar functions, whose unrolled evaluators make NVRTC slow), inlined everywhere else: the scan kernel's
// register allocation is sensitive to it.  The clean-entry paths have their own branch-free decoders.
#if defined(B2_COLD_OUTLINE) && defined(__CUDACC__)
#define B2_COLD __device__ __noinline__
#else
#define B2_COLD B2_HD
#endif

namespace b2 {

// ---- limits of the device plan ----
enum { MAX_GROUP = 4, MAX_PROJ = 16, MAX_COLS = 64, MAX_NODES = 96, MAX_CONDS = 8, MAX_AGGS = 8, MAX_ORDER = 4, MAX_STACK = 16, MAX_ACC_WORDS = 144,
       MAX_IMMS = 48 /* constants of a plan that travel as launch parameters instead of being part of the (compiled) plan */,
       MAX_TOPN_LIMIT = 4096 /* per-CTA candidate lists cost CTAs x limit x sizeof(TopItem) of HBM (engine.cu run_topn) */ };

// ---- device error codes (mapped to B2_ERR_* + message in engine.cu) ----
enum DevErr {
  DE_NONE = 0,
  DE_BAD_WRITE = 1,          // WriteRef::parse failure                     -> STORAGE
  DE_KEY_TOO_SHORT = 2,      // key shorter than the 8-byte ts suffix       -> STORAGE
  DE_DEFAULT_NOT_FOUND = 3,  // near_load_data_by_write miss                -> STORAGE
  DE_WRITE_CONFLICT = 4,     // RcCheckTs newer version                     -> WRITE_CONFLICT
  DE_BAD_USER_KEY = 5,       // memcomparable decode of user key failed     -> STORAGE
  DE_BAD_RECORD_KEY = 6,     // check_record_key / decode_int_handle        -> CORRUPTED
  DE_ROW_COLID_NOT_VARINT = 7,   // "Unable to decode row: column id must be VAR_INT"
  DE_ROW_EOF = 8,            // unexpected eof while splitting the row
  DE_ROW_BAD_DATUM = 9,      // split_datum: unsupported flag / too short
  DE_ROW_V2_BAD_INT = 10,    // "Failed to decode row v2 data as i64/u64"
  DE_ROW_V2_RANGE = 11,      // value slice / checksum cut out of range (reference panics)
  DE_MISSING_NOT_NULL = 12,  // "Data is corrupted, missing data for NOT NULL column"
  DE_MISSING_COMMIT_TS = 13,
  DE_DATUM_DECODE = 14,      // ensure_decoded: flag not decodable as the column's eval type
  DE_OVERFLOW_BIGINT = 20,   // 1690 BIGINT value is out of range
  DE_OVERFLOW_UBIGINT = 21,  // 1690 BIGINT UNSIGNED
  DE_OVERFLOW_DOUBLE = 22,   // 1690 DOUBLE
  DE_OVERFLOW_DIV = 23,      // 1690 "UNSIGNED BIGINT" (codec/overflow.rs:9-58: every integer-division overflow says so)
  DE_UNSUPPORTED_SIG = 30,
  DE_UNSUPPORTED_TYPE = 31,  // row holds a type the device path does not materialise
  DE_RAW_TOO_LONG = 32,      // bytes / json / decimal cell of 64 KiB or more (cell references carry 16 length bits)
  DE_IDX_BAD_KEY = 40,       // check_index_key (table.rs:114-140): not 't' tid "_i" idx ...
  DE_IDX_MISSING_COL = 41,   // "{i}th column is missing value" (index_scan_executor.rs:493-506)
  DE_IDX_BAD_HANDLE = 42,    // handle flag / length (index_scan_executor.rs:406-412, 451-471)
  DE_IDX_NEW_LAYOUT = 43,    // index value in the new (restored-data) layout: left to the CPU executor
};

// ---- plan as seen by the kernels ----
enum ColKind { CK_INT = 0, CK_REAL = 1, CK_OTHER = 2,
               // never evaluated, only materialised (they stay LazyBatchColumn::Raw in the reference until the response is encoded):
               CK_TIME = 3,   // DATE / DATETIME -> u64 CoreTime bits (Time::from_packed_u64, mysql/time/mod.rs:2002-2043)
               CK_DUR = 4,    // DURATION -> i64 nanoseconds
               CK_BYTES = 5, CK_JSON = 6, CK_DEC = 7 };  // cell reference (address << 16 | length) resolved after the scan kernel
B2_HD bool ck_is_ref(int k) { return k >= CK_BYTES; }
enum ColRole { CR_NORMAL = 0, CR_HANDLE = 1, CR_TABLE_ID = 2, CR_COMMIT_TS = 3, CR_SHADOWED = 4 /* duplicate col id: never filled */,
               CR_IDX_HANDLE = 5 /* BatchIndexScan: the int handle, from the key tail (non-unique index) or the value (unique) */ };
enum V2Class { V2_INT = 0, V2_UINT = 1, V2_COPY = 2, V2_BYTES = 3, V2_NIL = 4, V2_UNSUPPORTED = 5 };  // write_v2_as_datum arms
enum DefState { DS_NONE = 0, DS_VALUE = 1, DS_NULL = 2, DS_ERROR = 3 };

struct DevCol {
  int64_t col_id;
  int64_t default_bits;
  uint8_t kind, role, is_unsigned, not_null, tp, v2_class, def_state, v2_hint;
  uint8_t fsp, _p[7];  // CK_TIME: fractional-second digits of the column (tipb ColumnInfo.decimal, -1 -> 0)
};
struct DevNode {
  int32_t sig;   // FN: tipb ScalarFuncSig.  Constant: 0 = the value is `imm`; s > 0 = the value is launch parameter imms[s - 1]
                 // (plan_compile.h hoists constants so that `col < 5` and `col < 7` are one plan shape: one compiled kernel)
  uint8_t kind, n_args, et /*0 int 1 real*/, is_unsigned;
  int64_t imm;  // const bits (i64 or f64 bits) or column offset
};
struct DevExpr { uint16_t start, n; };
enum AggKind { AGG_COUNT = 0, AGG_SUM = 1, AGG_AVG = 2, AGG_MAX = 3, AGG_MIN = 4, AGG_FIRST = 5, AGG_BIT_AND = 6, AGG_BIT_OR = 7, AGG_BIT_XOR = 8 };
struct DevAgg { DevExpr arg; uint8_t kind /*AggKind*/, arg_et, arg_unsigned, acc_off; };
struct DevOrder { DevExpr e; uint8_t desc, et, is_unsigned, _pad; };

enum PlanMode { PM_SCAN = 0, PM_AGG = 1, PM_TOPN = 2, PM_CHECKSUM = 3,
                PM_PROJ = 4 /* kernel instantiation only: PM_SCAN whose output cells are projection expressions (DevPlan::mode stays PM_SCAN) */,
                PM_AGGM = 5 /* kernel instantiation only: PM_AGG grouped by 2..MAX_GROUP expressions (DevPlan::mode stays PM_AGG) */ };

// A selection condition of the shape `column <cmp> constant` over an integer column of the exact-layout fast path
struct FastCond {
  int64_t imm;
  uint8_t h;         // stored position of the column
  uint8_t op;        // 0 <  1 <=  2 >  3 >=  4 ==  5 !=   (column on the left; plan_compile flips `const <cmp> column`)
  uint8_t col_uns;   // compare the column as unsigned (field flag)
  uint8_t imm_uns;   // the constant is unsigned
  uint8_t zero_ext;  // decode: zero-extend (v2 UINT class)
  uint8_t imm_slot;  // s > 0: the constant is launch parameter imms[s - 1] (`imm` is 0 then)
  uint8_t _p[2];
};

struct DevPlan {
  int32_t mode;
  int32_t n_cols;
  int32_t n_nodes, n_conds;
  int32_t n_aggs, has_group, acc_words;
  int32_t n_order;
  int32_t n_out;
  int32_t isolation;  // B2_ISO_*
  int32_t need_value;  // 0 when no column is read from the row value (key-only)
  int32_t has_handle_cols;
  int32_t fast_n;      // > 0: rows holding exactly these `fast_n` non-null column ids (and no NULL ids) take the register fast path
  int32_t idx_cols;    // BatchIndexScan (index_scan_executor.rs): > 0 = the first `idx_cols` columns are index columns decoded from the
                       //   key's datums, then optionally the int handle (role CR_IDX_HANDLE) and the physical table id column; 0 = table scan
  uint64_t fast_filled;  // `filled` mask of such a row (every row-stored plan column)
  uint32_t fast_cls;     // bit h: stored column h (id order) is integer-class (width must be 1/2/4/8)
  uint32_t fast_uns;     // bit h: stored column h is zero-extended (unsigned)
  int8_t fast_out[8];    // PM_SCAN: output column fed by stored column h (first occurrence), or -1
  int32_t n_out_slow;    // PM_SCAN: outputs of a fast row that still go through cell_value (handle, Real, repeats ...)
  uint32_t fast_need;    // bit h: stored column h (id order) is read by some expression of the plan (conditions, group keys,
                         //   aggregate arguments, sort keys): the lean kernels decode those once per row
  int32_t fast_v1;       // 1: the fast path also covers row-format-v1 rows (all stored columns integer-class, ids <= 63)
                         //    and the request's data looked like v1 when it was opened (engine samples the first row)
  uint64_t fast_ids;   // the expected sorted non-null id bytes of such a row, packed little-endian (fast_n <= 8)
  uint64_t read_ts;
  uint64_t limit;
  DevExpr conds[MAX_CONDS];
  DevExpr group;
  uint8_t group_et, group_unsigned;
  uint8_t topn_all_keys;       // PM_TOPN: 1 = a sort key after the first can fail or warn (it is not a plain column or constant):
                               //   the lean kernel evaluates every sort key of every row, as the reference does, instead of
                               //   only those of the rows whose first key can still beat the CTA's bound
  uint8_t _p1;
  DevAgg aggs[MAX_AGGS];
  DevOrder order[MAX_ORDER];
  uint8_t out_cols[MAX_COLS];
  uint8_t out_slow[MAX_COLS];  // indices into out_cols
  int32_t n_fconds;            // == n_conds when every condition is a FastCond (else 0)
  int32_t n_raw;               // PM_SCAN: output columns that are cell references (bytes / json / decimal), resolved by the raw_* kernels
  FastCond fconds[MAX_CONDS];
  int32_t n_proj;              // BatchProjectionExecutor on top: out_cols index `proj`, every output is an expression value
  int32_t expr_refs;           // 1: some expression reads a cell reference (bytes / DECIMAL leaf: LIKE, Decimal comparisons): rows carry the HBM
                               //    address of their value (Row::gv) in every mode, and the lean kernels (which do not) stay out
  DevExpr proj[MAX_PROJ];
  int32_t n_group;             // >= 2: BatchSlowHashAggregation, grouped by `groups` (has_group is 1, `group` unused)
  int32_t _gpad;
  DevExpr groups[MAX_GROUP];
  uint8_t groups_et[MAX_GROUP];  // 0 Int, 1 Real
  DevCol cols[MAX_COLS];
  DevNode nodes[MAX_NODES];
};

// One CF block on the device.
struct BlockView {
  const uint8_t* keys;
  const uint32_t* koff;
  const uint8_t* vals;
  const uint32_t* voff;
  uint32_t n;
  static constexpr bool kWholeBlock = true;
  // entry accessors: the MVCC walk is written against these so that a shared-memory staged window of the block
  // (kernels.cu SmemView) can stand in for the HBM arrays
  B2_HD const uint8_t* kptr(uint32_t i) const { return keys + koff[i]; }
  B2_HD uint32_t klen(uint32_t i) const { return koff[i + 1] - koff[i]; }
  B2_HD const uint8_t* vptr(uint32_t i) const { return vals + voff[i]; }
  B2_HD uint32_t vlen(uint32_t i) const { return voff[i + 1] - voff[i]; }
  B2_HD const uint8_t* gval(const uint8_t* p) const { return p; }  // a value byte's address in HBM (the view is the HBM heap itself)
};

// ---- byte access -------------------------------------------------------------------------------
// Unaligned 8-byte little-endian load built from aligned 32-bit words + funnel shifts (3 word loads instead of 8
// byte loads).  It may touch up to 3 bytes before and 11 bytes after `p`, always inside the same 16-byte-padded
// heap (ABI contract in b2_copr.h) or the padded shared-memory stage.
B2_HD uint64_t ld64(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
  // (pointer arithmetic instead of integer masking keeps the address space visible to the compiler: LDS for staged bytes)
  uint32_t mis = (uint32_t)(unsigned long long)p & 3u;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p - mis);
  uint32_t s = mis * 8u;
  uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
  uint32_t lo = __funnelshift_r(w0, w1, s), hi = __funnelshift_r(w1, w2, s);
  return ((uint64_t)hi << 32) | lo;
#else
  uint64_t v;
  __builtin_memcpy(&v, p, 8);
  return v;
#endif
}
B2_HD uint32_t ld32(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
  uint32_t mis = (uint32_t)(unsigned long long)p & 3u;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p - mis);
  return __funnelshift_r(w[0], w[1], mis * 8u);
#else
  uint32_t v;
  __builtin_memcpy(&v, p, 4);
  return v;
#endif
}
B2_HD uint64_t bswap64(uint64_t v) {
#if defined(__CUDA_ARCH__)
  uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
  return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
#else
  return __builtin_bswap64(v);
#endif
}
B2_HD uint32_t ld8(const uint8_t* p) { return *p; }
B2_HD uint64_t ld_be64(const uint8_t* p) { return bswap64(ld64(p)); }
B2_HD uint64_t ld_le(const uint8_t* p, int n) {  // n in {1,2,4,8}
  uint64_t v = ld64(p);
  return n >= 8 ? v : (v & ((1ull << (8 * n)) - 1));
}
B2_HD bool bytes_eq(const uint8_t* a, const uint8_t* b, uint32_t n) {
  // 8 bytes at a time from the tail: record keys share their table prefix and differ in the handle
  while (n >= 8) {
    n -= 8;
    if (ld64(a + n) != ld64(b + n)) return false;
  }
  if (n == 0) return true;
  return ((ld64(a) ^ ld64(b)) & ((1ull << (8 * n)) - 1)) == 0;
}
B2_HD int bytes_cmp(const uint8_t* a, uint32_t an, const uint8_t* b, uint32_t bn) {
  uint32_t m = an < bn ? an : bn;
  for (uint32_t i = 0; i < m; ++i) {
    if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
  }
  return an < bn ? -1 : (an > bn ? 1 : 0);
}

B2_HD uint32_t ctz32(uint32_t v) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__ffs((int)v) - 1u;  // BREV + FLO
#else
  return (uint32_t)__builtin_ctz(v);
#endif
}
B2_HD uint32_t ctz64(uint64_t v) {
#if defined(__CUDA_ARCH__)
  const uint32_t lo = (uint32_t)v;  // (the 64-bit __ffsll costs three times the 32-bit one)
  return lo ? ctz32(lo) : 32u + ctz32((uint32_t)(v >> 32));
#else
  return (uint32_t)__builtin_ctzll(v);
#endif
}
// eight 7-bit groups, one per byte (bit 7 of every byte clear) -> one 56-bit value
B2_HD uint64_t compress7(uint64_t x) {
  x = ((x & 0x7f007f007f007f00ull) >> 1) | (x & 0x007f007f007f007full);
  x = ((x & 0x3fff00003fff0000ull) >> 2) | (x & 0x00003fff00003fffull);
  x = ((x & 0x0fffffff00000000ull) >> 4) | (x & 0x000000000fffffffull);
  return x;
}
// components/codec/src/number.rs:445-483 try_decode_var_u64. returns bytes consumed, 0 = eof.
// Word-wise: one unaligned 8-byte load finds the terminating byte (first byte with bit 7 clear) and the payload bits
// are gathered with three mask-and-shift steps; bytes 9 and 10 of the longest encodings are looked at separately.
// (With n >= 10 the reference takes the 10th byte unconditionally and keeps only its lowest bit.)
B2_COLD uint32_t dec_var_u64(const uint8_t* p, uint32_t n, uint64_t* out) {
  if (n == 0) return 0;
  const uint64_t w = ld64(p);
  if ((w & 0x80u) == 0) { *out = w & 0x7fu; return 1; }
  const uint64_t stop = ~w & 0x8080808080808080ull;
  if (stop) {
    const uint32_t len = (ctz64(stop) >> 3) + 1;  // 2..8
    if (len > n) return 0;
    const uint64_t x = len == 8 ? w : (w & ((1ull << (8 * len)) - 1));
    *out = compress7(x & 0x7f7f7f7f7f7f7f7full);
    return len;
  }
  if (n < 9) return 0;  // every available byte asks for more
  const uint64_t x = compress7(w & 0x7f7f7f7f7f7f7f7full);
  const uint64_t b8 = p[8];
  if (b8 < 0x80) { *out = x | (b8 << 56); return 9; }
  if (n < 10) return 0;
  *out = x | ((b8 & 0x7f) << 56) | (((uint64_t)p[9] & 1) << 63);
  return 10;
}
// components/tikv_util/src/codec/number.rs:224-275 (overflow error on a 10th byte > 1)
B2_HD uint32_t dec_var_u64_tu(const uint8_t* p, uint32_t n, uint64_t* out) {
  uint64_t v = 0;
  for (uint32_t i = 0; i < n && i < 10; ++i) {
    uint64_t b = p[i];
    if (i == 9) {
      if (b > 1) return 0;
      *out = v | (b << 63);
      return 10;
    }
    v |= (b & 0x7f) << (7 * i);
    if (b < 0x80) { *out = v; return i + 1; }
  }
  return 0;
}
B2_COLD uint32_t dec_var_i64(const uint8_t* p, uint32_t n, int64_t* out) {
  uint64_t uv;
  uint32_t c = dec_var_u64(p, n, &uv);
  if (!c) return 0;
  int64_t v = (int64_t)(uv >> 1);
  if (uv & 1) v = ~v;
  *out = v;
  return c;
}
B2_HD uint32_t first_var_int_len(const uint8_t* p, uint32_t n) {  // number.rs:530-567
  const uint32_t lim = n >= 10 ? 9 : n;
  if (lim == 0) return n;
  const uint64_t stop = ~ld64(p) & 0x8080808080808080ull;
  if (stop) {
    const uint32_t len = (ctz64(stop) >> 3) + 1;
    if (len <= lim) return len;
  } else if (lim >= 9 && p[8] < 0x80) return 9;
  return n >= 10 ? 10 : n;
}

B2_HD double cmp_u64_to_f64(uint64_t u) {  // tikv_util/src/codec/number.rs:36-42
  const uint64_t S = 0x8000000000000000ull;
  if (u & S) u &= ~S; else u = ~u;
#if defined(__CUDA_ARCH__)
  return __longlong_as_double((long long)u);
#else
  double f;
  __builtin_memcpy(&f, &u, 8);
  return f;
#endif
}
B2_HD uint64_t f64_bits(double f) {
#if defined(__CUDA_ARCH__)
  return (uint64_t)__double_as_longlong(f);
#else
  uint64_t u;
  __builtin_memcpy(&u, &f, 8);
  return u;
#endif
}
B2_HD double bits_f64(uint64_t u) {
#if defined(__CUDA_ARCH__)
  return __longlong_as_double((long long)u);
#else
  double f;
  __builtin_memcpy(&f, &u, 8);
  return f;
#endif
}

// ---- keys --------------------------------------------------------------------------------------
B2_HD uint64_t key_commit_ts(const uint8_t* k, uint32_t klen) { return ~ld_be64(k + klen - 8); }

// entries i and j of the same block share their user key? (types.rs:249-267 is_user_key_eq)
template <class V>
B2_HD bool same_user_key(const V& b, uint32_t i, uint32_t j) {
  uint32_t al = b.klen(i), bl = b.klen(j);
  if (al != bl) return false;
  const uint8_t* a = b.kptr(i);
  const uint8_t* c = b.kptr(j);
  if (al < 8) return al == 0 ? true : bytes_eq(a, c, al);
  return bytes_eq(a, c, al - 8);
}

// Memcomparable user key -> raw key view (bytes.rs:178-228).  We never materialise the raw key: raw byte j
// lives at enc[j + j/8].  Returns raw length, or -1 if the encoding is invalid.
B2_HD int raw_key_len(const uint8_t* enc, uint32_t enc_len) {
  uint32_t off = 0;
  int raw = 0;
  if (enc_len == 27) {  // int-handle record key: two full groups + a 3-byte tail (markers FF FF FA, 5 zero pad bytes)
    uint64_t tail = ld64(enc + 19);  // enc[19..26]
    if (enc[8] == 0xff && enc[17] == 0xff && (tail >> 16) == 0xfa0000000000ull) return 19;
  }
  for (;;) {
    if (off + 9 > enc_len) return -1;
    uint32_t marker = enc[off + 8];
    uint32_t pad = 0xffu - marker;
    if (pad == 0) { raw += 8; off += 9; continue; }
    if (pad > 8) return -1;
    for (uint32_t i = 8 - pad; i < 8; ++i)
      if (enc[off + i] != 0) return -1;
    raw += 8 - pad;
    return raw;  // trailing bytes after the terminal group are ignored (decode_bytes leaves them to the caller)
  }
}
B2_HD uint32_t raw_at(const uint8_t* enc, uint32_t j) { return enc[j + (j >> 3)]; }
B2_HD uint64_t raw_be64(const uint8_t* enc, uint32_t j) {
  if (j == 11) {  // int handle: raw[11..15] = enc[12..16], raw[16..18] = enc[18..20]
    uint64_t a = bswap64(ld64(enc + 12)), b = bswap64(ld64(enc + 18));
    return (a & 0xffffffffff000000ull) | (b >> 40);
  }
  if (j == 1) {  // table id: raw[1..7] = enc[1..7], raw[8] = enc[9]
    uint64_t a = bswap64(ld64(enc + 1));
    return (a & 0xffffffffffffff00ull) | enc[9];
  }
  uint64_t v = 0;
  for (uint32_t i = 0; i < 8; ++i) v = (v << 8) | raw_at(enc, j + i);
  return v;
}

// ---- write record --------------------------------------------------------------------------------
struct WriteRec {
  uint8_t type;  // 'P','D','L','R'
  uint8_t has_short, has_gc_fence, lc_kind;  // lc_kind: 0 unknown 1 exist 2 not-exist
  uint32_t short_off, short_len;
  uint64_t start_ts, gc_fence, lc_ts, lc_versions;
};

B2_HD int parse_write(const uint8_t* p, uint32_t n, WriteRec* w) {
  if (n == 0) return DE_BAD_WRITE;
  uint8_t t = p[0];
  if (t != 'P' && t != 'D' && t != 'L' && t != 'R') return DE_BAD_WRITE;
  w->type = t;
  w->has_short = 0; w->has_gc_fence = 0; w->lc_kind = 0; w->gc_fence = 0; w->short_off = 0; w->short_len = 0;
  uint32_t pos = 1;
  uint32_t c = dec_var_u64(p + pos, n - pos, &w->start_ts);
  if (!c) return DE_BAD_WRITE;
  pos += c;
  uint64_t lc_ts = 0, lc_ver = 0;
  // the overwhelmingly common record: Put/.. + start_ts + 'v' len row, nothing after it
  if (pos + 2 <= n && p[pos] == 'v' && pos + 2 + p[pos + 1] == n) {
    w->has_short = 1; w->short_off = pos + 2; w->short_len = p[pos + 1];
    w->lc_ts = 0; w->lc_versions = 0;
    return DE_NONE;
  }
  while (pos < n) {
    uint8_t tag = p[pos++];
    if (tag == 'v') {
      if (pos >= n) return DE_BAD_WRITE;
      uint32_t len = p[pos++];
      if (n - pos < len) return DE_BAD_WRITE;  // reference panics
      w->has_short = 1; w->short_off = pos; w->short_len = len;
      pos += len;
    } else if (tag == 'R') {
    } else if (tag == 'F') {
      if (n - pos < 8) return DE_BAD_WRITE;
      w->has_gc_fence = 1; w->gc_fence = ld_be64(p + pos);
      pos += 8;
    } else if (tag == 'l') {
      if (n - pos < 8) return DE_BAD_WRITE;
      lc_ts = ld_be64(p + pos);
      pos += 8;
      uint32_t m = dec_var_u64_tu(p + pos, n - pos, &lc_ver);
      if (!m) return DE_BAD_WRITE;
      pos += m;
    } else if (tag == 'S') {
      uint64_t src;
      uint32_t m = dec_var_u64_tu(p + pos, n - pos, &src);
      if (!m) return DE_BAD_WRITE;
      pos += m;
    } else {
      break;
    }
  }
  if (lc_ts == 0) w->lc_kind = lc_ver > 0 ? 2 : 0;
  else {
    if (lc_ver == 0) return DE_BAD_WRITE;  // LastChange::make_exist assert
    w->lc_kind = 1;
  }
  w->lc_ts = lc_ts; w->lc_versions = lc_ver;
  return DE_NONE;
}

// ---- MVCC: resolve the run of versions that starts at entry `e0` -------------------------------------
struct DefaultCf {  // CF_DEFAULT blocks (global order) for long values
  const BlockView* blocks;
  uint32_t n_blocks;
};

struct RunOut {
  int err;            // DevErr
  int found;          // 1 = a visible Put
  uint32_t entry;     // index of the chosen CF_WRITE entry
  const uint8_t* val; // row value bytes (inside CF_WRITE value or CF_DEFAULT)
  uint32_t val_len;
  uint64_t commit_ts;
  uint32_t met_newer; // saw a version newer than read_ts
  uint32_t dflt_lookup;
  uint32_t steps;     // entries visited
  uint32_t truncated; // the walk needed an entry at or beyond `walk_hi` (not resident in this view): redo on the whole block
};

// near_load_data_by_write (scanner/mod.rs:371-402): exact-match lookup of user_key ‖ !start_ts in CF_DEFAULT
B2_HD bool default_lookup(const DefaultCf& d, const uint8_t* ukey, uint32_t uklen, uint64_t start_ts, const uint8_t** val, uint32_t* vlen) {
  uint8_t ts[8];
  uint64_t nts = ~start_ts;
  for (int i = 0; i < 8; ++i) ts[i] = (uint8_t)(nts >> (8 * (7 - i)));
  for (uint32_t bi = 0; bi < d.n_blocks; ++bi) {
    const BlockView& b = d.blocks[bi];
    uint32_t lo = 0, hi = b.n;
    while (lo < hi) {
      uint32_t mid = lo + (hi - lo) / 2;
      const uint8_t* k = b.keys + b.koff[mid];
      uint32_t kl = b.koff[mid + 1] - b.koff[mid];
      // compare k with ukey‖ts
      uint32_t m = kl < uklen ? kl : uklen;
      int c = bytes_cmp(k, m, ukey, m);
      if (c == 0) {
        if (kl < uklen) c = -1;
        else c = bytes_cmp(k + uklen, kl - uklen, ts, 8);
      }
      if (c < 0) lo = mid + 1; else hi = mid;
    }
    if (lo < b.n) {
      const uint8_t* k = b.keys + b.koff[lo];
      uint32_t kl = b.koff[lo + 1] - b.koff[lo];
      if (kl == uklen + 8 && bytes_eq(k, ukey, uklen) && ld_be64(k + uklen) == nts) {
        *val = b.vals + b.voff[lo];
        *vlen = b.voff[lo + 1] - b.voff[lo];
        return true;
      }
    }
  }
  return false;
}

// forward.rs:310-375 (move_write_cursor_to_ts) + :433-515 (LatestKvPolicy::handle_write), restated as a walk over
// the contiguous run of versions [e0, e_hi) of one user key.  `e_hi` is the range's upper bound entry; the view `b`
// only holds entries below `walk_hi` (<= e_hi; the whole block: walk_hi == e_hi).
template <class V>
B2_HD void resolve_run(const V& b, uint32_t e0, uint32_t e_hi, uint32_t walk_hi, uint64_t read_ts, int isolation, const DefaultCf& dflt, RunOut* o) {
  o->err = DE_NONE; o->found = 0; o->met_newer = 0; o->dflt_lookup = 0; o->steps = 1; o->truncated = 0;
  uint32_t i = e0;
  const uint8_t* k0 = b.kptr(e0);
  uint32_t kl0 = b.klen(e0);
  if (kl0 < 8) { o->err = DE_KEY_TOO_SHORT; o->entry = e0; return; }
  // move to the first version with commit_ts <= read_ts
  for (;;) {
    uint64_t cts = key_commit_ts(b.kptr(i), b.klen(i));
    if (cts <= read_ts) break;
    o->met_newer = 1;
    if (isolation == B2_ISO_RC_CHECK_TS) { o->err = DE_WRITE_CONFLICT; o->entry = i; return; }
    ++i; o->steps++;
    if (i >= e_hi) return;
    if (i >= walk_hi) { o->truncated = 1; return; }
    if (!same_user_key(b, e0, i)) return;
  }
  for (;;) {
    const uint8_t* vp = b.vptr(i);
    uint32_t vl = b.vlen(i);
    WriteRec w;
    int e = parse_write(vp, vl, &w);
    if (e) { o->err = e; o->entry = i; return; }
    if (w.has_gc_fence && w.gc_fence != 0 && w.gc_fence <= read_ts) return;  // write.rs:425-442
    if (w.type == 'P') {
      o->commit_ts = key_commit_ts(b.kptr(i), b.klen(i));
      o->entry = i;
      if (w.has_short) { o->val = vp + w.short_off; o->val_len = w.short_len; o->found = 1; return; }
      if constexpr (!V::kWholeBlock) {
        o->truncated = 1;  // the value lives in CF_DEFAULT (HBM): such rows are resolved through the block view
        return;
      } else {
        o->dflt_lookup = 1;
        if (!default_lookup(dflt, k0, kl0 - 8, w.start_ts, &o->val, &o->val_len)) { o->err = DE_DEFAULT_NOT_FOUND; return; }
        o->found = 1;
        return;
      }
    }
    if (w.type == 'D') return;
    // Lock / Rollback
    if (w.lc_kind == 2) return;
    if (w.lc_kind == 1 && w.lc_versions >= 8 /* SEEK_BOUND */) {
      // seek to user_key ‖ last_change_ts: first later version with commit_ts <= last_change_ts
      for (;;) {
        ++i; o->steps++;
        if (i >= e_hi) return;
        if (i >= walk_hi) { o->truncated = 1; return; }
        if (!same_user_key(b, e0, i)) return;
        if (key_commit_ts(b.kptr(i), b.klen(i)) <= w.lc_ts) break;
      }
    } else {
      ++i; o->steps++;
      if (i >= e_hi) return;
      if (i >= walk_hi) { o->truncated = 1; return; }
      if (!same_user_key(b, e0, i)) return;
    }
  }
}

// ---- row access ----------------------------------------------------------------------------------
enum CellKind { CELL_MISSING = 0, CELL_V1 = 1, CELL_V2 = 2, CELL_NULL = 3 };

struct RowView {
  const uint8_t* v;
  uint32_t n;
  uint8_t fmt;  // 0 = no columns, 1 = v1, 2 = v2
  // v2 header
  uint8_t big;
  uint16_t nn_cnt, null_cnt;
  uint32_t ids_off, null_ids_off, offs_off, vals_off, vals_len;
};

struct Cells {  // per-column cell location for v1 rows (filled by row_split)
  uint32_t off[MAX_COLS];
  uint32_t len_kind[MAX_COLS];  // len << 2 | kind
};

// split_datum (datum.rs:1117-1155, desc = false): length of the first datum or 0 + err
B2_COLD uint32_t split_datum(const uint8_t* p, uint32_t n, int* err) {
  if (n == 0) { *err = DE_ROW_BAD_DATUM; return 0; }
  uint32_t pos;
  const uint8_t* r = p + 1;
  uint32_t rn = n - 1;
  switch (p[0]) {
    case 3: case 4: case 5: case 7: pos = 8; break;  // INT, UINT, FLOAT, DURATION
    case 1: {  // BYTES: memcomparable groups
      uint32_t idx = 8;
      for (;;) {
        if (rn < idx + 1) { pos = rn; break; }
        if (r[idx] != 0xff) { pos = idx + 1; break; }
        idx += 9;
      }
      break;
    }
    case 2: {  // COMPACT_BYTES
      int64_t len;
      uint32_t c = dec_var_i64(r, rn, &len);
      if (!c) pos = rn;
      else {
        uint64_t t = (uint64_t)len + c;
        pos = t < rn ? (uint32_t)t : rn;
      }
      break;
    }
    case 0: pos = 0; break;  // NIL
    case 6: {  // DECIMAL: prec, frac, bin
      if (rn < 2) { *err = DE_ROW_BAD_DATUM; return 0; }
      uint32_t prec = r[0], frac = r[1];
      if (prec < frac) { *err = DE_ROW_BAD_DATUM; return 0; }
      const uint8_t d2b[10] = {0, 1, 1, 2, 2, 3, 3, 4, 4, 4};
      uint32_t ic = prec - frac;
      pos = (ic / 9) * 4 + d2b[ic % 9] + (frac / 9) * 4 + d2b[frac % 9] + 2;
      break;
    }
    case 8: case 9: pos = first_var_int_len(r, rn); break;  // VAR_INT / VAR_UINT
    default: *err = DE_ROW_BAD_DATUM; return 0;  // JSON / vector / unknown: not handled on the device
  }
  if (n < pos + 1) { *err = DE_ROW_BAD_DATUM; return 0; }
  return pos + 1;
}

B2_HD uint32_t v2_id(const RowView& r, uint32_t base, uint32_t i) {
  return r.big ? (uint32_t)ld_le(r.v + base + 4 * i, 4) : r.v[base + i];
}
B2_HD uint32_t v2_off(const RowView& r, uint32_t i) {
  return r.big ? (uint32_t)ld_le(r.v + r.offs_off + 4 * i, 4) : (uint32_t)ld_le(r.v + r.offs_off + 2 * i, 2);
}
// LeBytes::binary_search (row_slice.rs:330-357)
B2_HD bool v2_search(const RowView& r, uint32_t base, uint32_t cnt, uint32_t id, uint32_t* idx) {
  if (cnt == 0) return false;
  uint32_t size = cnt, lo = 0, steps = 20;
  while (steps > 0 && size > 1) {
    uint32_t half = size / 2, mid = lo + half;
    if (!(v2_id(r, base, mid) > id)) lo = mid;
    size -= half;
    --steps;
  }
  if (v2_id(r, base, lo) == id) { *idx = lo; return true; }
  return false;
}

// RowSlice::from_bytes (row_slice.rs:74-115)
B2_HD int row_open(const uint8_t* v, uint32_t n, RowView* r) {
  r->v = v; r->n = n;
  if (n == 0 || (n == 1 && v[0] == 0)) { r->fmt = 0; return DE_NONE; }  // table_scan_executor.rs:377-378
  if (v[0] != 128) { r->fmt = 1; return DE_NONE; }
  r->fmt = 2;
  if (n < 6) return DE_ROW_EOF;
  uint64_t hdr = ld64(v);  // 0x80, flags, u16 non-null count, u16 null count
  uint32_t flags = (uint32_t)(hdr >> 8) & 0xffu;
  r->big = flags & 1;
  r->nn_cnt = (uint16_t)(hdr >> 16);
  r->null_cnt = (uint16_t)(hdr >> 32);
  uint32_t idw = r->big ? 4 : 1, ofw = r->big ? 4 : 2;
  uint64_t pos = 6;
  r->ids_off = (uint32_t)pos; pos += (uint64_t)r->nn_cnt * idw;
  if (pos > n) return DE_ROW_EOF;
  r->null_ids_off = (uint32_t)pos; pos += (uint64_t)r->null_cnt * idw;
  if (pos > n) return DE_ROW_EOF;
  r->offs_off = (uint32_t)pos; pos += (uint64_t)r->nn_cnt * ofw;
  if (pos > n) return DE_ROW_EOF;
  r->vals_off = (uint32_t)pos; r->vals_len = n - (uint32_t)pos;
  if (flags & 2) {  // WITH_CHECKSUM: cut_checksum_bytes :231-259 + assert len 5 or 9
    uint32_t last = r->nn_cnt == 0 ? 0 : v2_off(*r, r->nn_cnt - 1u);
    if (last > r->vals_len) return DE_ROW_V2_RANGE;
    uint32_t ck = r->vals_len - last;
    if (ck != 5 && ck != 9) return DE_ROW_V2_RANGE;
    r->vals_len = last;
  }
  return DE_NONE;
}

// Locate column `c` of the plan in a v2 row (process_v2 :261-279).
// `hint` = position the column would have if the row held exactly the plan's columns (the common case): one id
// compare replaces the binary search.
B2_HD int v2_locate(const RowView& r, int64_t col_id, uint32_t hint, uint32_t* off, uint32_t* len, int* err) {
  int64_t upper = r.big ? 0xffffffffll : 0xffll;
  if (!(col_id > 0 && col_id <= upper)) return CELL_MISSING;
  uint32_t idx = hint;
  bool hit = hint < r.nn_cnt && v2_id(r, r.ids_off, hint) == (uint32_t)col_id;
  if (hit || v2_search(r, r.ids_off, r.nn_cnt, (uint32_t)col_id, &idx)) {
    uint32_t end, start;
    if (!r.big && idx > 0) { uint32_t w = ld32(r.v + r.offs_off + 2 * idx - 2); start = w & 0xffffu; end = w >> 16; }
    else { end = v2_off(r, idx); start = idx > 0 ? v2_off(r, idx - 1) : 0; }
    if (start > end || end > r.vals_len) { *err = DE_ROW_V2_RANGE; return CELL_MISSING; }
    *off = r.vals_off + start; *len = end - start;
    return CELL_V2;
  }
  if (v2_search(r, r.null_ids_off, r.null_cnt, (uint32_t)col_id, &idx)) return CELL_NULL;
  return CELL_MISSING;
}

struct Row {
  RowView rv;
  const uint8_t* enc_key;  // encoded user key (memcomparable), without ts
  uint32_t enc_key_len;
  uint64_t commit_ts;
  uint64_t filled;  // bitmask of plan columns present in the row (bit c)
  uint32_t fast;    // 1 (v2) / 2 (v1): the row holds exactly the plan's columns, all non-null: cells come from the two offset words below
  uint64_t o_lo, o_hi;  // the row's u16 end-offsets 0..3 / 4..7
  uint64_t idx_handle;  // BatchIndexScan: the row's int handle (bits)
  const int64_t* imms;  // the request's hoisted constants (ScanArgs::imms: kernel parameter space on the device)
  uint64_t* cv = nullptr;  // lean kernels, plan-specialised builds: the integer cells of the stored columns the plan's expressions
                        //   (a caller-owned array of 8 words: kept out of the row so that indexing it never forces the row into local memory)
  uint32_t cv_mask = 0; //   read (DevPlan::fast_need), decoded once per row; bit h set = cv[h] is valid
  const uint8_t* gv = nullptr;  // address of rv.v[0] in the block's HBM heap (rv.v may be a shared-memory copy): what the cell
                                //   references of bytes / json / decimal columns are made of (set only when the plan has such columns)
  mutable uint32_t warn = 0;  // EvalWarnings raised while evaluating expressions on this row ("Division by 0", expr/ctx.rs:267-286);
                              // counted into the request only when the row's tile is committed
};
B2_HD int64_t node_imm(const Row& row, const DevNode& nd) { return nd.sig > 0 ? row.imms[nd.sig - 1] : nd.imm; }

B2_HD uint32_t shr_clamp(uint32_t v, uint32_t sh) {  // v >> sh, 0 for sh >= 32
#if defined(__CUDA_ARCH__)
  return __funnelshift_rc(v, 0u, sh);
#else
  return sh >= 32 ? 0u : v >> sh;
#endif
}
// end offset of stored column h of a fast row (h is a compile-time constant after unrolling)
B2_HD uint32_t fast_end(const Row& row, int h) { return (uint32_t)((h < 4 ? row.o_lo : row.o_hi) >> ((h & 3) * 16)) & 0xffffu; }
// integer cell of a fast v1 row: the datum of stored column h starts two bytes (VAR_INT flag + one-byte column id)
// after the end of the previous datum; decode_int_datum (datum_codec.rs:401-421) by flag, lengths validated by the probe
B2_HD uint64_t fast_int_cell_v1(const Row& row, uint32_t prev_end) {
  const uint8_t* p = row.rv.v + prev_end + 2;
  const uint32_t flag = p[0];
  if (flag == 8) { int64_t v = 0; dec_var_i64(p + 1, 10, &v); return (uint64_t)v; }
  if (flag == 9) { uint64_t v = 0; dec_var_u64(p + 1, 10, &v); return v; }
  const uint64_t u = ld_be64(p + 1);
  return flag == 3 ? u ^ 0x8000000000000000ull : u;
}
// integer cell of a fast row: stored column h spans [start, end) of the value area (compat_v1.rs:13-38)
B2_HD uint64_t fast_int_cell(const Row& row, uint32_t start, uint32_t end, bool zero_extend) {
  uint64_t u = ld64(row.rv.v + row.rv.vals_off + start);
  const uint32_t sh = (64u - 8u * (end - start)) & 63u;  // width 8 -> 0: branch-free, so neighbouring cells overlap
  u <<= sh;
  return zero_extend ? (u >> sh) : (uint64_t)((int64_t)u >> sh);
}
// Every stored column of this fast v2 row is 8 bytes wide (full-range BIGINTs: the common table of wide integers)?
B2_HD bool fast_all8(const DevPlan& P, const Row& row) {
  const uint64_t m_lo = P.fast_n >= 4 ? ~0ull : ((1ull << (16 * P.fast_n)) - 1);
  const uint64_t m_hi = P.fast_n >= 8 ? ~0ull : (P.fast_n <= 4 ? 0ull : ((1ull << (16 * (P.fast_n - 4))) - 1));
  return row.fast == 1 && ((row.o_lo ^ 0x0020001800100008ull) & m_lo) == 0 && ((row.o_hi ^ 0x0040003800300028ull) & m_hi) == 0;
}
// ... then the cells of the stored columns in `need` (bit h) come out of one run of aligned words with one shift amount
// (2 word loads + 2 funnel shifts per cell instead of an unaligned load each); width 8 needs no sign / zero extension
B2_HD void fast_cells8(const Row& row, uint32_t need, uint64_t (&out)[8]) {
  const uint8_t* p = row.rv.v + row.rv.vals_off;
#if defined(__CUDA_ARCH__)
  const uint32_t mis = (uint32_t)(unsigned long long)p & 3u;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p - mis);
  const uint32_t s = mis * 8u;
#pragma unroll
  for (int h = 0; h < 8; ++h) {
    out[h] = 0;
    if ((need >> h) & 1u) {
      const uint32_t a = w[2 * h], b = w[2 * h + 1], c = w[2 * h + 2];
      out[h] = ((uint64_t)__funnelshift_r(b, c, s) << 32) | __funnelshift_r(a, b, s);
    }
  }
#else
  for (int h = 0; h < 8; ++h) {
    out[h] = 0;
    if ((need >> h) & 1u) __builtin_memcpy(&out[h], p + 8 * h, 8);
  }
#endif
}

// decode the stored integer columns in `need` (bit h) of a fast v2 row into row.cv (compile-time positions when unrolled)
B2_HD void fast_fill_cells(const DevPlan& P, Row& row, uint32_t need) {
  uint32_t prev = 0;
#pragma unroll
  for (int h = 0; h < 8; ++h) {
    if (h < P.fast_n) {
      const uint32_t end = fast_end(row, h);
      if ((need >> h) & 1u) row.cv[h] = fast_int_cell(row, prev, end, (P.fast_uns >> h) & 1u);
      prev = end;
    }
  }
  row.cv_mask = need;
}

// stored column h of a fast row of either format, h known only at run time (conditions, cell_value).  The v1 decoder
// is kept out of the unrolled per-position loops on purpose: inlined there it tripled the size of the hot loop.
B2_HD uint64_t fast_cell_dyn(const Row& row, uint32_t h, bool zero_extend, bool v1_enabled) {
  const uint32_t end = (uint32_t)((h < 4 ? row.o_lo : row.o_hi) >> ((h & 3) * 16)) & 0xffffu;
  const uint32_t start = h == 0 ? 0u : ((uint32_t)((h - 1 < 4 ? row.o_lo : row.o_hi) >> (((h - 1) & 3) * 16)) & 0xffffu);
  return v1_enabled && row.fast == 2 ? fast_int_cell_v1(row, start) : fast_int_cell(row, start, end, zero_extend);
}
// Row format v1 twin of fast_row_probe: the row is exactly `08 id datum` for the plan's columns in id order, every datum
// an INT / UINT / VAR_INT / VAR_UINT that fits the buffer.  The end offsets of the datums go into the same two
// registers as for v2 rows.  Anything else (NIL, other flags, more or fewer columns, ids >= 64, a truncated varint)
// takes the general datum walk, which also raises the reference's errors.
B2_HD bool fast_row_probe_v1(const DevPlan& P, Row& row) {
  const RowView& r = row.rv;
  row.fast = 0;
  if (!P.fast_v1) return false;
  // straight-line on purpose (no early exits, varint lengths by select): lanes of a warp hold datums of different
  // lengths, and any branch on them would keep the lanes apart for the rest of the unrolled walk
  uint32_t pos = 0, bad = 0;
  uint64_t lo = 0, hi = 0;
#pragma unroll
  for (int h = 0; h < 8; ++h) {
    if (h < P.fast_n) {
      const uint32_t at = pos < r.n ? pos : 0u;  // keep the loads inside the row even after a mismatch
      const uint32_t w = ld32(r.v + at);         // 08, zigzag(id), datum flag, first payload byte
      const uint32_t want = 0x08u | ((uint32_t)((P.fast_ids >> (8 * h)) & 0xffu) << 9);
      const uint32_t flag = (w >> 16) & 0xffu;
      const uint64_t pay = ld64(r.v + at + 3);
      const uint64_t stop = ~pay & 0x8080808080808080ull;
      const uint32_t vlen = stop ? (ctz64(stop) >> 3) + 1 : ((r.v[at + 11] & 0x80u) ? 10u : 9u);  // varint bytes (number.rs:530-567)
      const bool is_var = flag == 8 || flag == 9, is_fix = flag == 3 || flag == 4;
      const uint32_t dl = 1 + (is_var ? vlen : 8u);
      bad |= ((w & 0xffffu) != want) | (!is_var && !is_fix) | (pos + 2 + dl > r.n);
      pos += 2 + dl;
      if (h < 4) lo |= (uint64_t)(pos & 0xffffu) << (16 * h); else hi |= (uint64_t)(pos & 0xffffu) << (16 * (h - 4));
    }
  }
  if (bad || pos != r.n || pos > 0xffffu) return false;
  row.o_lo = lo; row.o_hi = hi;
  row.fast = 2;
  return true;
}
// Does this v2 row hold exactly the plan's columns (process_v2 would find column k at position v2_hint), all
// non-null, offsets monotone and inside the value area, integer-class columns 1/2/4/8 bytes wide?  On success the
// end-offsets stay in two registers: no per-column search, no Cells traffic.
B2_HD bool fast_offsets_ok(const DevPlan& P, Row& row);
B2_HD bool fast_row_probe(const DevPlan& P, Row& row) {
  const RowView& r = row.rv;
  row.fast = 0;
  if (!(P.fast_n > 0 && !r.big && r.nn_cnt == (uint32_t)P.fast_n && r.null_cnt == 0)) return false;
  if (((ld64(r.v + r.ids_off) ^ P.fast_ids) & (P.fast_n >= 8 ? ~0ull : ((1ull << (8 * P.fast_n)) - 1))) != 0) return false;
  row.o_lo = ld64(r.v + r.offs_off);
  row.o_hi = P.fast_n > 4 ? ld64(r.v + r.offs_off + 8) : 0;
  return fast_offsets_ok(P, row);
}
// the end offsets in row.o_lo / o_hi are monotone, inside the value area, and integer-class columns are 1/2/4/8 bytes wide
B2_HD bool fast_offsets_ok(const DevPlan& P, Row& row) {
  const RowView& r = row.rv;
  if (P.fast_cls == (1u << P.fast_n) - 1u) {
    // all stored columns are integer-class: the eight widths are checked at once, four 16-bit lanes per register.
    // width = end - previous end (mod 2^16); it must be 1, 2, 4 or 8: (w & 0xfff0) == 0, w != 0, w & (w - 1) == 0.
    // (A decreasing offset wraps to a width >= 2^16 - 64 and fails the first test; a row cannot climb past 2^16 in
    // eight steps of at most 8.)  Lanes beyond fast_n hold row data, not offsets: they are forced to width 1.
    const uint64_t H = 0x8000800080008000ull, ONE = 0x0001000100010001ull;
    const uint64_t p_lo = row.o_lo << 16, p_hi = (row.o_hi << 16) | (row.o_lo >> 48);
    uint64_t d_lo = ((row.o_lo | H) - (p_lo & ~H)) ^ ((row.o_lo ^ ~p_lo) & H);
    uint64_t d_hi = ((row.o_hi | H) - (p_hi & ~H)) ^ ((row.o_hi ^ ~p_hi) & H);
    const uint64_t m_lo = P.fast_n >= 4 ? ~0ull : ((1ull << (16 * P.fast_n)) - 1);
    const uint64_t m_hi = P.fast_n >= 8 ? ~0ull : (P.fast_n <= 4 ? 0ull : ((1ull << (16 * (P.fast_n - 4))) - 1));
    d_lo = (d_lo & m_lo) | (ONE & ~m_lo);
    d_hi = (d_hi & m_hi) | (ONE & ~m_hi);
    const uint64_t big = (d_lo | d_hi) & 0xfff0fff0fff0fff0ull;
    const uint64_t zero = (((d_lo - ONE) & ~d_lo) | ((d_hi - ONE) & ~d_hi)) & H;  // exact: every lane is < 2^15 once `big` is 0
    const uint64_t npow2 = (d_lo & (d_lo - ONE)) | (d_hi & (d_hi - ONE));         // no borrows once no lane is 0
    if (big | zero) return false;
    if (npow2) return false;
    const uint32_t last = (uint32_t)(((P.fast_n <= 4 ? row.o_lo : row.o_hi) >> (((P.fast_n - 1) & 3) * 16)) & 0xffffu);
    if (last > r.vals_len) return false;
    row.fast = 1;
    return true;
  }
  uint32_t prev = 0, bad = 0;
#pragma unroll
  for (int h = 0; h < 8; ++h) {
    if (h < P.fast_n) {
      uint32_t end = fast_end(row, h);
      if ((P.fast_cls >> h) & 1u) bad |= ~shr_clamp(0x116u, end - prev);  // widths 1, 2, 4, 8 (a decreasing offset wraps to a huge width)
      else bad |= end < prev ? 1u : 0u;
      prev = end;
    }
  }
  if ((bad & 1u) || prev > r.vals_len) return false;
  row.fast = 1;
  return true;
}

// ---- clean-entry front end -------------------------------------------------------------------------------------
// The overwhelmingly common CF_WRITE entry of a table scan: an int-handle record key (35 bytes: memcomparable
// 't' tid "_r" handle, then !commit_ts) that is the first version of its user key, visible at read_ts, holding
// `P varint(start_ts) v len row` and nothing else, the row being an exact-layout v2 row.  For such an entry the
// general walk (same_user_key + resolve_run + parse_write + row_open + row_split) collapses into a few word loads
// with one shared funnel shift each.  Every function below either accepts an entry and yields exactly what the
// general functions yield for it, or rejects it (then the caller runs the general functions: errors, version walks,
// CF_DEFAULT lookups, odd keys and rows all live there).
//
// N consecutive little-endian 64-bit words from an arbitrary byte address: 2N+1 aligned 32-bit loads, one shift amount.
// May read up to 3 bytes before and 4 bytes after the 8N requested ones (inside the padded stage / heap).
template <int N>
B2_HD void ld64xN(const uint8_t* p, uint64_t (&out)[N]) {
#if defined(__CUDA_ARCH__)
  const uint32_t mis = (uint32_t)(unsigned long long)p & 3u;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p - mis);
  const uint32_t s = mis * 8u;
  uint32_t x[2 * N + 1];
#pragma unroll
  for (int i = 0; i < 2 * N + 1; ++i) x[i] = w[i];
#pragma unroll
  for (int i = 0; i < N; ++i) out[i] = ((uint64_t)__funnelshift_r(x[2 * i + 1], x[2 * i + 2], s) << 32) | __funnelshift_r(x[2 * i], x[2 * i + 1], s);
#else
  __builtin_memcpy(out, p, 8 * N);
#endif
}

// enc[12..36) of a 35-byte CF_WRITE key: a = raw handle bytes 0..4, group marker, handle bytes 5..6;
// b = handle byte 7, five pad zeros, terminal marker 0xFA, first ts byte; c = ts bytes 1..7 (+ one byte past the key)
struct KeyTail { uint64_t a, b, c; };
// true: the key has the shape of an int-handle record key from byte 12 on (bytes 0..11, 't' tid[0..7] FF tid[7] "_r",
// are validated once per unit of work: every key of a sorted range shares them when its first and last key do)
B2_HD bool fast_key_tail(const uint8_t* kp, uint32_t klen, KeyTail* t) {
  if (klen != 35) return false;
  uint64_t w[3];
  ld64xN<3>(kp + 12, w);
  t->a = w[0]; t->b = w[1]; t->c = w[2];
  return ((w[0] >> 40) & 0xffu) == 0xffu && (w[1] & 0x00ffffffffffff00ull) == 0x00fa000000000000ull;
}
B2_HD uint64_t key_tail_commit_ts(const KeyTail& t) { return ~bswap64((t.b >> 56) | (t.c << 8)); }
// commit_ts <= read_ts without assembling the timestamp: the key holds !commit_ts big-endian, so compare it with !read_ts
B2_HD bool key_tail_visible(const KeyTail& t, uint64_t not_read_ts) {
#if defined(__CUDA_ARCH__)
  const uint32_t bh = (uint32_t)(t.b >> 32), cl = (uint32_t)t.c, ch = (uint32_t)(t.c >> 32);
  const uint32_t hi = __byte_perm(bh, cl, 0x3456), lo = __byte_perm(cl, ch, 0x3456);  // bytes (b7 c0 c1 c2) and (c3 c4 c5 c6), most significant first
  return (((uint64_t)hi << 32) | lo) >= not_read_ts;
#else
  return bswap64((t.b >> 56) | (t.c << 8)) >= not_read_ts;
#endif
}
// same user key as the entry before?  (both keys validated by fast_key_tail, both inside one unit: bytes 0..11 and 21..26 agree)
B2_HD bool key_tail_same(uint64_t a, uint64_t b, uint64_t pa, uint64_t pb) { return a == pa && ((b ^ pb) & 0xffu) == 0; }
// the same for any two 35-byte keys of one unit (no marker validation needed): bytes 12..26 equal
B2_HD bool key_tail_same_exact(uint64_t a, uint64_t b, uint64_t pa, uint64_t pb) { return a == pa && ((b ^ pb) & 0x00ffffffffffffffull) == 0; }
// key words of any 35-byte key + whether it is a well-formed int-handle record key from byte 12 on
B2_HD bool key_tail_load(const uint8_t* kp, KeyTail* t) {
  uint64_t w[3];
  ld64xN<3>(kp + 12, w);
  t->a = w[0]; t->b = w[1]; t->c = w[2];
  return ((w[0] >> 40) & 0xffu) == 0xffu && (w[1] & 0x00ffffffffffff00ull) == 0x00fa000000000000ull;
}
// first 12 bytes of the keys of a unit: what check_record_key / decode_int_handle need of them (table.rs:187-226)
B2_HD bool record_key_prefix_ok(const uint8_t* k) { return k[0] == 't' && k[8] == 0xff && k[10] == '_' && k[11] == 'r'; }

// `P varint(start_ts) v len row`, nothing after the row (parse_write's common record): row = vp + *row_off
B2_HD bool fast_write_head(const uint8_t* vp, uint32_t vlen, uint32_t* row_off, uint32_t* row_len) {
  if (vlen < 4) return false;
  uint64_t w[2];
  ld64xN<2>(vp, w);
  // terminal byte of the varint: first of value bytes 1..9 with bit 7 clear (a 10-byte varint is left to the general parser)
  const uint64_t s0 = ~w[0] & 0x8080808080808000ull;
  const uint32_t s1 = ~(uint32_t)w[1] & 0x8080u;
  uint32_t term;
  if (s0) term = ctz64(s0) >> 3;
  else if (s1) term = 8u + (ctz64((uint64_t)s1) >> 3);
  else return false;
  const uint32_t pos = term + 1;
  if (pos + 2 > vlen) return false;
  const uint32_t tag = vp[pos], len = vp[pos + 1];
  *row_off = pos + 2; *row_len = len;
  return (w[0] & 0xffu) == 'P' && tag == 'v' && pos + 2 + len == vlen;
}

// The same without branches, for the lean kernels (fast_kernel.cuh): bit 0 = `P varint v len row` and nothing after
// (a visible Put with an inline value), bit 1 = `D varint` and nothing after (a plain Delete).  Anything else is left to
// the general parser.  *row_off / *row_len are only meaningful with bit 0.
B2_HD uint32_t fast_write_kind(const uint8_t* vp, uint32_t vlen, uint32_t* row_off, uint32_t* row_len) {
  uint64_t w[2];
  ld64xN<2>(vp, w);
  const uint64_t s0 = ~w[0] & 0x8080808080808000ull;
  const uint32_t s1 = ~(uint32_t)w[1] & 0x8080u;
  const uint32_t term = s0 ? (ctz64(s0) >> 3) : (8u + (ctz32(s1 | 0x800000u) >> 3));  // 10 when no terminal byte in 1..9
  const uint32_t pos = term + 1;
  const bool var_ok = (s0 != 0 || s1 != 0) && vlen >= 2;
  const uint32_t at = pos + 1 < vlen ? pos : 0;  // keep the two byte loads inside the value
  const uint32_t tag = vp[at], len = vp[at + 1];
  const uint32_t type = (uint32_t)w[0] & 0xffu;
  *row_off = pos + 2; *row_len = len;
  const bool put = var_ok && type == 'P' && pos + 2 <= vlen && tag == 'v' && pos + 2 + len == vlen;
  const bool del = var_ok && type == 'D' && pos == vlen;
  return (put ? 1u : 0u) | (del ? 2u : 0u);
}

// ---- who owns a version run: the lean kernel or the general walk ------------------------------------------------------
// The lean kernels (fast_kernel.cuh) look at 32 consecutive entries per warp, one per lane, and decide without walking:
//   same   the lane's entry has the user key of the entry before it (both 35-byte keys, words equal; never at the range start)
//   vis    commit_ts <= read_ts.  Versions of a key are sorted newest first, so `vis` is monotone inside a run
//   chosen vis && (!same || !vis(previous entry)): the first visible version — what forward.rs:310-375 walks to
//   kind   fast_write_kind of the entry's value: 1 Put with an inline value, 2 plain Delete, 0 anything else
// A run is *committed* here by its chosen lane when everything about it is plain; otherwise exactly one lane *pushes* the
// run's first entry onto the list the general kernel works through afterwards (it re-checks that the entry is a run
// start, so pushing a non-start is harmless; pushing a start twice would double-count: the rules below are exclusive):
//   (a) a run start whose key is not a well-formed 35-byte record key: pushed by itself; its lanes never commit
//   (b) the chosen lane holds something that is not a plain Put / Delete, or its row needs the general decoder:
//       pushed by the chosen lane — if the run starts in this warp (else rule (c) already fired in an earlier warp)
//   (c) a run start with no chosen lane before the warp ends: the run may go on in the next warp, whose lanes cannot see
//       this one: pushed by the start lane; lanes of later warps never commit a run that started before their warp
//   (d) RcCheckTs: a version above the snapshot is a WriteConflict (forward.rs:342-354): pushed by the start lane, and
//       only a chosen lane that is its run's start commits
enum { FA_COMMIT = 1, FA_PUSH = 2 };
B2_HD uint32_t clz32(uint32_t v) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__clz((int)v);
#else
  return v ? (uint32_t)__builtin_clz(v) : 32u;
#endif
}
// start_m / chosen_m / valid_m: ballots of (valid && !same), chosen, valid.  Returns FA_* flags; *push_back = how many
// entries before this lane's entry the pushed run start lies.
B2_HD uint32_t fast_lane_decide(uint32_t lane, uint32_t start_m, uint32_t chosen_m, uint32_t valid_m, bool valid, bool same, bool chosen, bool kok,
                                uint32_t kind, bool vis, bool rc_check, uint32_t* push_back) {
  *push_back = 0;
  if (!valid) return 0;
  if (start_m == valid_m && chosen_m == valid_m && !rc_check)  // the warp holds 32 single-version, visible keys: nothing to look up
    return !kok || kind == 0u ? (uint32_t)FA_PUSH : (kind == 1u ? (uint32_t)FA_COMMIT : 0u);
  const uint32_t upto = 0xffffffffu >> (31u - lane);  // lanes 0..lane
  const uint32_t below = start_m & upto;
  const bool orphan = below == 0;                     // the run started before this warp
  const uint32_t sl = orphan ? 0u : 31u - clz32(below);
  const bool is_start = !same;
  if (!kok) return is_start ? (uint32_t)FA_PUSH : 0u;  // (a); continuation lanes of such a run share its key: they do nothing
  uint32_t flags = 0;
  if (is_start) {
    const uint32_t above = start_m & ~upto;
    const uint32_t next = above ? ctz32(above) : 32u;
    const uint32_t run = (next >= 32u ? ~0u : ((1u << next) - 1u)) & ~(upto >> 1) & valid_m;  // lanes [lane, next)
    const bool open_end = (run >> (31u - clz32(valid_m))) & 1u;                                 // touches the warp's last valid lane
    if ((chosen_m & run) == 0 && open_end) flags |= FA_PUSH;                                     // (c)
    if (rc_check && !vis) flags |= FA_PUSH;                                                      // (d)
  }
  if (chosen && !orphan && (!rc_check || is_start)) {
    *push_back = lane - sl;
    if (kind == 1u) flags |= FA_COMMIT;      // (the caller turns this into a push when the row needs the general decoder)
    else if (kind == 0u) flags |= FA_PUSH;   // (b)
  }
  return flags;
}

// ---- CRC-64/XZ as a linear map (checksum.rs:105-114 without a table walk per value byte) ------------------------------
// One table step is c' = T[(c ^ byte) & 0xff] ^ (c >> 8): linear over GF(2) in (c, byte).  For a message of n bytes from
// state c0 the final state is A^n(c0) ^ Lin(message), where A is the zero-byte step and Lin(m) = XOR_i A^(n-1-i)(T[m_i])
// depends only on each byte's distance from the END of the message.  So for the KV message `key part ‖ value`:
//   ~crc(kv) = ~( A^vlen(state after the key part) ^ Lin(value) )
// and the XOR over all KVs of a scan is
//   (odd count ? ~0 : 0)  ^  XOR_vlen A^vlen( XOR of the key states of the KVs with that value length )
//                         ^  Lin( XOR of all values, right-aligned )
// i.e. per KV one 8-byte table step for the handle and plain XORs of the value words; the table walks over value bytes
// happen once per thread at the end of the kernel.  T = slicing-by-8 tables (8 x 256 u64, T[k * 256 + i] = T0 advanced k bytes).
B2_HD uint64_t crc_step1(const unsigned long long* T, uint64_t c, uint32_t byte) { return T[((uint32_t)c ^ byte) & 0xffu] ^ (c >> 8); }
B2_HD uint64_t crc_step8(const unsigned long long* T, uint64_t c, uint64_t w) {
  c ^= w;
  const uint32_t lo = (uint32_t)c, hi = (uint32_t)(c >> 32);
  return T[7 * 256 + (lo & 0xffu)] ^ T[6 * 256 + ((lo >> 8) & 0xffu)] ^ T[5 * 256 + ((lo >> 16) & 0xffu)] ^ T[4 * 256 + (lo >> 24)] ^
         T[3 * 256 + (hi & 0xffu)] ^ T[2 * 256 + ((hi >> 8) & 0xffu)] ^ T[1 * 256 + ((hi >> 16) & 0xffu)] ^ T[hi >> 24];
}
B2_HD uint64_t crc_advance_zeros(const unsigned long long* T, uint64_t c, uint32_t n_bytes) {
  for (; n_bytes >= 8; n_bytes -= 8) c = crc_step8(T, c, 0);
  for (; n_bytes; --n_bytes) c = crc_step1(T, c, 0);
  return c;
}
// the handle bytes raw[11..19) of an int-handle record key, in message (memory) order, from its key tail words
B2_HD uint64_t key_tail_handle_le(uint64_t a, uint64_t b) { return (a & 0xffffffffffull) | ((a >> 48) << 40) | ((b & 0xffull) << 56); }

// row_open + fast_row_probe fused for a small v2 row without checksum that holds exactly the plan's columns: header,
// ids and end offsets come out of one run of words (every field sits at a compile-time offset in a specialised kernel)
B2_HD bool fast_row_v2(const DevPlan& P, const uint8_t* r, uint32_t n, Row& row) {
  const int K = P.fast_n;
  row.fast = 0;
  if (K <= 0 || n < 6u + 3u * (uint32_t)K) return false;
  uint64_t w[4];
  if (K <= 2) { uint64_t t[2]; ld64xN<2>(r, t); w[0] = t[0]; w[1] = t[1]; w[2] = w[3] = 0; }
  else if (K <= 4) { uint64_t t[3]; ld64xN<3>(r, t); w[0] = t[0]; w[1] = t[1]; w[2] = t[2]; w[3] = 0; }
  else ld64xN<4>(r, w);
  auto field = [&](int j) -> uint64_t {  // 8 row bytes from byte j
    const int q = j >> 3, sh = (j & 7) * 8;
    if (sh == 0) return w[q];
    return (w[q] >> sh) | (q + 1 < 4 ? (w[q + 1] << (64 - sh)) : 0ull);
  };
  // 0x80, flags 0 (small, no checksum), K non-null ids, no null ids
  if ((w[0] & 0xffffffffffffull) != (0x80ull | ((uint64_t)K << 16))) return false;
  if (((field(6) ^ P.fast_ids) & (K >= 8 ? ~0ull : ((1ull << (8 * K)) - 1))) != 0) return false;
  RowView& v = row.rv;
  v.v = r; v.n = n; v.fmt = 2; v.big = 0; v.nn_cnt = (uint16_t)K; v.null_cnt = 0;
  v.ids_off = 6; v.null_ids_off = 6u + (uint32_t)K; v.offs_off = 6u + (uint32_t)K; v.vals_off = 6u + 3u * (uint32_t)K; v.vals_len = n - v.vals_off;
  row.o_lo = field(6 + K);
  row.o_hi = K > 4 ? field(14 + K) : 0;
  return fast_offsets_ok(P, row);
}

// process_kv_pair (table_scan_executor.rs:365-475): everything that can fail regardless of which rows are
// later selected.  For v1 rows it records the cell of every plan column in `cells`.
B2_HD int row_split(const DevPlan& P, Row& row, Cells& cells) {
  const RowView& r = row.rv;
  uint64_t filled = 0;
  row.fast = 0;
  int err = DE_NONE;
  if (r.fmt == 1 && fast_row_probe_v1(P, row)) {
    filled = P.fast_filled;
  } else if (r.fmt == 1) {
    uint32_t pos = 0, n = r.n;
    int decoded = 0;
    while (pos < n && decoded < P.n_cols) {
      if (r.v[pos] != 8) return DE_ROW_COLID_NOT_VARINT;
      ++pos;
      int64_t cid;
      uint32_t c = dec_var_i64(r.v + pos, n - pos, &cid);
      if (!c) return DE_ROW_EOF;
      pos += c;
      uint32_t dl = split_datum(r.v + pos, n - pos, &err);
      if (!dl) return err;
      // column_id_index lookup: last plan column with this id that is not a handle / shadowed
      for (int k = 0; k < P.n_cols; ++k) {
        if (P.cols[k].col_id == cid && P.cols[k].role != CR_HANDLE && P.cols[k].role != CR_SHADOWED) {
          if (!((filled >> k) & 1)) {
            cells.off[k] = pos; cells.len_kind[k] = (dl << 2) | CELL_V1;
            filled |= 1ull << k;
            ++decoded;
          }
          break;
        }
      }
      pos += dl;
    }
  } else if (r.fmt == 2 && fast_row_probe(P, row)) {
    // exact-layout fast path: the row holds precisely the plan's columns, all non-null, with well-formed offsets and
    // integer widths (anything else, including rows that would raise an error, takes the general branch below)
    filled = P.fast_filled;
  } else if (r.fmt == 2) {
    for (int k = 0; k < P.n_cols; ++k) {
      const DevCol& c = P.cols[k];
      if (c.role == CR_HANDLE || c.role == CR_SHADOWED) continue;
      uint32_t off = 0, len = 0;
      int kind = v2_locate(r, c.col_id, c.v2_hint, &off, &len, &err);
      if (err) return err;
      if (kind == CELL_V2) {
        if (c.v2_class == V2_INT || c.v2_class == V2_UINT) {
          if (len != 1 && len != 2 && len != 4 && len != 8) return DE_ROW_V2_BAD_INT;
        } else if (c.v2_class == V2_UNSUPPORTED) return DE_UNSUPPORTED_TYPE;
        filled |= 1ull << k;
      } else if (kind == CELL_NULL) filled |= 1ull << k;
      if (kind != CELL_MISSING) { cells.off[k] = off; cells.len_kind[k] = (len << 2) | (uint32_t)kind; }
    }
  }
  // key side (:386-442)
  int rawlen = raw_key_len(row.enc_key, row.enc_key_len);
  if (rawlen < 0) return DE_BAD_USER_KEY;
  const uint8_t* ek = row.enc_key;
  bool rec_ok = rawlen >= 11 && raw_at(ek, 0) == 't' && raw_at(ek, 9) == '_' && raw_at(ek, 10) == 'r';
  if (P.has_handle_cols) {
    if (!rec_ok || rawlen < 19) return DE_BAD_RECORD_KEY;
  } else if (!rec_ok) return DE_BAD_RECORD_KEY;
  for (int k = 0; !row.fast && k < P.n_cols; ++k) {
    const DevCol& c = P.cols[k];
    if (c.role == CR_HANDLE || c.role == CR_TABLE_ID || c.role == CR_COMMIT_TS) { filled |= 1ull << k; continue; }
    if (!((filled >> k) & 1)) {
      if (c.def_state == DS_NONE && c.not_null) return DE_MISSING_NOT_NULL;
    }
  }
  row.filled = filled;
  return DE_NONE;
}

// BatchIndexScanExecutor::process_kv_pair -> process_old_collation_kv (index_scan_executor.rs:363-380, 514-574): the index
// columns are the datums of the key after 't' tid "_i" idx (19 raw bytes), the int handle follows them in the key (non-unique
// index) or is the value (unique index, 8 bytes big-endian).  The raw key bytes [19, rawlen) are copied into `buf` (the
// memcomparable group markers removed), `cells` point at the datums there, and the row then decodes like a v1 row.
enum { IDX_RAW_MAX = 112 };
B2_HD int index_row_split(const DevPlan& P, Row& row, Cells& cells, const uint8_t* val, uint32_t val_len, uint8_t* buf) {
  const uint8_t* ek = row.enc_key;
  const int rawlen = raw_key_len(ek, row.enc_key_len);
  if (rawlen < 0) return DE_BAD_USER_KEY;
  if (rawlen < 1 || raw_at(ek, 0) != 't') return DE_IDX_BAD_KEY;
  if (rawlen < 11) return DE_ROW_EOF;
  if (raw_at(ek, 9) != '_' || raw_at(ek, 10) != 'i') return DE_IDX_BAD_KEY;
  if (rawlen < 19) return DE_ROW_EOF;
  if (val_len > 9) return DE_IDX_NEW_LAYOUT;
  const uint32_t n = (uint32_t)rawlen - 19u;
  if (n > IDX_RAW_MAX) return DE_UNSUPPORTED_TYPE;
  for (uint32_t j = 0; j < n; ++j) buf[j] = (uint8_t)raw_at(ek, 19u + j);
  row.rv.v = buf; row.rv.n = n; row.rv.fmt = 1;
  row.fast = 0;
  uint32_t pos = 0;
  uint64_t filled = 0;
  int err = DE_NONE;
  for (int i = 0; i < P.idx_cols; ++i) {  // extract_columns_from_datum_format :493-506
    if (pos >= n) return DE_IDX_MISSING_COL;
    const uint32_t dl = split_datum(buf + pos, n - pos, &err);
    if (!dl) return err;
    cells.off[i] = pos; cells.len_kind[i] = (dl << 2) | CELL_V1;
    filled |= 1ull << i;
    pos += dl;
  }
  for (int k = P.idx_cols; k < P.n_cols; ++k) {
    filled |= 1ull << k;
    if (P.cols[k].role != CR_IDX_HANDLE) continue;
    if (pos >= n) {  // unique index: decode_int_handle_from_value :406-412
      if (val_len < 8) return DE_IDX_BAD_HANDLE;
      row.idx_handle = ld_be64(val);
    } else {         // decode_int_handle_from_key :451-471
      const uint32_t flag = buf[pos];
      if ((flag != 3 && flag != 4) || n - pos < 9) return DE_IDX_BAD_HANDLE;
      uint64_t u = 0;
      for (int b = 0; b < 8; ++b) u = (u << 8) | buf[pos + 1 + b];
      row.idx_handle = flag == 3 ? (u ^ 0x8000000000000000ull) : u;
    }
  }
  row.filled = filled;
  return DE_NONE;
}

struct Value { uint64_t bits; bool null; };

// Time::from_packed_u64 (mysql/time/mod.rs:2002-2043) for DATE / DATETIME: packed = ((y * 13 + m) << 5 | d) << 17 | h << 12 | mi << 6 | s,
// then << 24 | micro; the result is the CoreTime bit field (:167-196): year 63..50, month 49..46, day 45..41, hour 40..36,
// minute 35..30, second 29..24, micro 23..4, fsp_tt 3..0 (Date = 0b1110, DateTime = fsp << 1).  Zero stays all-zero fields.
B2_HD uint64_t time_bits_from_packed(uint64_t value, bool is_date, uint32_t fsp) {
  const uint64_t fsp_tt = is_date ? 0xeull : ((uint64_t)fsp << 1);
  if (value == 0) return fsp_tt;
  const uint64_t ymdhms = value >> 24, ymd = ymdhms >> 17, ym = ymd >> 5, hms = ymdhms & 0x1ffffu;
  const uint64_t day = ymd & 31, month = ym % 13, year = ym / 13, second = hms & 63, minute = (hms >> 6) & 63, hour = hms >> 12, micro = value & 0xffffffu;
  return ((year & 0x3fff) << 50) | ((month & 15) << 46) | ((day & 31) << 41) | ((hour & 31) << 36) | ((minute & 63) << 30) | ((second & 63) << 24) |
         ((micro & 0xfffff) << 4) | fsp_tt;
}
// DecimalDecoder::read_decimal (mysql/decimal.rs:2204-2289): (precision, frac, binary decimal) -> the 40-byte struct of a chunk cell
B2_HD bool raw_decimal_parse(const unsigned char* p, unsigned int n, b2_decimal* out) {
  if (n < 3) return false;
  const unsigned int prec = p[0], frac = p[1];
  if (prec < frac) return false;
  p += 2; n -= 2;
  const unsigned char d2b[10] = {0, 1, 1, 2, 2, 3, 3, 4, 4, 4};
  const unsigned int pow10[10] = {1u, 10u, 100u, 1000u, 10000u, 100000u, 1000000u, 10000000u, 100000000u, 1000000000u};
  const unsigned int int_cnt = prec - frac, iw = int_cnt / 9, lead = int_cnt - iw * 9, fw = frac / 9, trail = frac - fw * 9;
  if (iw + (lead > 0) + fw + (trail > 0) > 9) return false;
  const unsigned int mask = (p[0] & 0x80) ? 0u : 0xffffffffu;
  b2_decimal d;
  d.int_cnt = (unsigned char)int_cnt; d.frac_cnt = (unsigned char)frac; d.result_frac_cnt = (unsigned char)frac; d.negative = mask != 0;
  for (int i = 0; i < 9; ++i) d.word_buf[i] = 0;
  bool first = true, ok = true;
  auto word = [&](unsigned int size) -> unsigned int {  // read_word :2159-2200: big-endian, sign-extended, first byte's top bit flipped
    if (n < size) { ok = false; return 0u; }
    unsigned int b0 = p[0];
    if (first) { b0 ^= 0x80u; first = false; }
    int r = (int)(signed char)b0;
    for (unsigned int i = 1; i < size; ++i) r = (int)(((unsigned int)r << 8) | p[i]);
    p += size; n -= size;
    return (unsigned int)r;
  };
  unsigned int w = 0;
  if (lead) {
    d.word_buf[w] = word(d2b[lead]) ^ mask;
    if (!ok || d.word_buf[w] >= pow10[lead + 1]) return false;
    if (d.word_buf[w] != 0) ++w; else d.int_cnt -= (unsigned char)lead;
  }
  for (unsigned int i = 0; i < iw; ++i) {
    d.word_buf[w] = word(4) ^ mask;
    if (!ok || d.word_buf[w] > 999999999u) return false;
    if (w > 0 || d.word_buf[w] != 0) ++w; else d.int_cnt -= 9;
  }
  for (unsigned int i = 0; i < fw; ++i) {
    d.word_buf[w] = word(4) ^ mask;
    if (!ok || d.word_buf[w] > 999999999u) return false;
    ++w;
  }
  if (trail) {
    const unsigned long long x = (unsigned long long)(word(d2b[trail]) ^ mask) * pow10[9 - trail];
    if (!ok || x > 999999999ull) return false;
    d.word_buf[w] = (unsigned int)x;
  }
  if (d.int_cnt == 0 && d.frac_cnt == 0) { d.int_cnt = 1; d.negative = 0; for (int i = 0; i < 9; ++i) d.word_buf[i] = 0; }  // Decimal::zero()
  d.result_frac_cnt = (unsigned char)frac;
  *out = d;
  return true;
}
B2_HD uint64_t raw_ref_make(const uint8_t* gaddr, uint32_t len) { return ((uint64_t)(unsigned long long)gaddr << 16) | len; }
B2_HD const uint8_t* raw_ref_addr(uint64_t r) { return (const uint8_t*)(unsigned long long)(r >> 16); }
B2_HD uint32_t raw_ref_len(uint64_t r) { return (uint32_t)(r & 0xffffu); }

// One cell of a column the executors never decode (Column::from_raw_datums, chunk/column.rs:72-151, per-type appenders
// :697-913; v2 cells as write_v2_as_datum would have converted them, compat_v1.rs:54-129).  DATE / DATETIME and DURATION
// become their 8-byte chunk cell here; bytes / json / decimal become a reference to the cell's payload in HBM, which the
// kernels in kernels.cu (raw_*) turn into the column's heap / 40-byte structs once the launch's rows are in place.
// (`heap` = the HBM address of p's first byte: the caller maps p, which may point into a shared-memory copy of the row, through Row::gv;
//  the row itself is not passed: an out-of-line function taking the row by reference would pin it in local memory for every caller)
B2_COLD int cell_value_raw(const DevCol& c, const uint8_t* heap, const uint8_t* p, uint32_t len, int kind, Value* out) {
  const uint64_t S = 0x8000000000000000ull;
  const uint8_t* q = p;
  uint32_t qn = len;
  uint32_t flag = 0xffu;  // v2: no datum flag
  if (kind != CELL_V2) {
    flag = p[0]; q = p + 1; qn = len - 1;
    if (flag == 0) { out->null = true; return DE_NONE; }
  }
  if (c.kind == CK_TIME) {
    uint64_t u;
    if (kind == CELL_V2) { if (len != 1 && len != 2 && len != 4 && len != 8) return DE_ROW_V2_BAD_INT; u = ld_le(p, (int)len); }
    else if (flag == 4) { if (qn < 8) return DE_DATUM_DECODE; u = ld_be64(q); }
    else if (flag == 9) { if (!dec_var_u64(q, qn, &u)) return DE_DATUM_DECODE; }
    else return DE_DATUM_DECODE;
    out->bits = time_bits_from_packed(u, c.tp == B2_TP_DATE, c.fsp);
    return DE_NONE;
  }
  if (c.kind == CK_DUR) {
    if (kind == CELL_V2) {
      if (len != 1 && len != 2 && len != 4 && len != 8) return DE_ROW_V2_BAD_INT;
      uint64_t u = ld_le(p, (int)len);
      if (len < 8) { const uint32_t sh = 64 - 8 * len; u = (uint64_t)(((int64_t)(u << sh)) >> sh); }
      out->bits = u;
    } else if (flag == 7) { if (qn < 8) return DE_DATUM_DECODE; out->bits = ld_be64(q) ^ S; }
    else if (flag == 8) { int64_t v; if (!dec_var_i64(q, qn, &v)) return DE_DATUM_DECODE; out->bits = (uint64_t)v; }
    else return DE_DATUM_DECODE;
    return DE_NONE;
  }
  if (kind != CELL_V2) {
    if (c.kind == CK_BYTES) {
      if (flag == 1) return DE_UNSUPPORTED_TYPE;  // memcomparable bytes (index keys): the cell is not a slice of the stored bytes
      if (flag != 2) return DE_DATUM_DECODE;
      int64_t vn;
      const uint32_t used = dec_var_i64(q, qn, &vn);
      if (!used || vn < 0 || (uint64_t)vn > qn - used) return DE_DATUM_DECODE;
      q += used; qn = (uint32_t)vn;
    } else if (c.kind == CK_DEC) { if (flag != 6) return DE_DATUM_DECODE; }
    else return DE_DATUM_DECODE;  // CK_JSON: a v1 JSON datum never gets here (split_datum does not size binary JSON on the device)
  }
  if (qn > 0xffffu) return DE_RAW_TOO_LONG;
  out->bits = raw_ref_make(heap + (q - p), qn);
  return DE_NONE;
}

// Decode plan column `k` of the row (LazyBatchColumn::ensure_decoded for one cell, lazy_column.rs:165-221).
B2_HD int cell_value(const DevPlan& P, const Row& row, const Cells& cells, int k, Value* out) {
  const DevCol& c = P.cols[k];
  out->null = false; out->bits = 0;
  const uint64_t S = 0x8000000000000000ull;
  if (row.fast && c.role == CR_NORMAL && c.kind == CK_INT) {  // hot case: integer column of an exact-layout v2 row
    if ((row.cv_mask >> c.v2_hint) & 1u) { out->bits = row.cv[c.v2_hint]; return DE_NONE; }
    out->bits = fast_cell_dyn(row, c.v2_hint, c.v2_class != V2_INT, P.fast_v1 != 0);
    return DE_NONE;
  }
  if (c.role == CR_HANDLE) { out->bits = raw_be64(row.enc_key, 11) ^ S; return DE_NONE; }       // table.rs:214-218
#ifndef B2_NO_IDX
  if (c.role == CR_IDX_HANDLE) { out->bits = row.idx_handle; return DE_NONE; }
#endif
  if (c.role == CR_TABLE_ID) { out->bits = raw_be64(row.enc_key, 1) ^ S; return DE_NONE; }
  if (c.role == CR_COMMIT_TS) { out->bits = row.commit_ts; return DE_NONE; }
  if (c.kind == CK_OTHER) return DE_UNSUPPORTED_TYPE;
  const RowView& r = row.rv;
  const uint8_t* p = nullptr;
  uint32_t len = 0;
  int kind = CELL_MISSING;
  if (row.fast == 1 || (!P.fast_v1 && row.fast)) {
    uint32_t h = c.v2_hint;
    uint32_t end = (uint32_t)((h < 4 ? row.o_lo : row.o_hi) >> ((h & 3) * 16)) & 0xffffu;
    uint32_t start = h == 0 ? 0u : ((uint32_t)((h - 1 < 4 ? row.o_lo : row.o_hi) >> (((h - 1) & 3) * 16)) & 0xffffu);
    p = r.v + r.vals_off + start; len = end - start; kind = CELL_V2;
  } else if ((row.filled >> k) & 1) {
    p = r.v + cells.off[k]; len = cells.len_kind[k] >> 2; kind = cells.len_kind[k] & 3;  // located once by row_split
  }
  if (kind == CELL_NULL) { out->null = true; return DE_NONE; }
  if (kind == CELL_MISSING) {
    if (c.def_state == DS_VALUE) { out->bits = (uint64_t)c.default_bits; return DE_NONE; }
    if (c.def_state == DS_ERROR) return DE_DATUM_DECODE;
    out->null = true;  // DS_NULL, or nullable without default
    return DE_NONE;
  }
  if (c.kind >= CK_TIME) return cell_value_raw(c, row.gv + (p - r.v), p, len, kind, out);
  if (kind == CELL_V2) {
    if (c.kind == CK_INT) {
      // compat_v1.rs:13-38: sign- or zero-extend by width, then INT/UINT datum -> i64 bits
      uint64_t u = ld_le(p, (int)len);
      if (c.v2_class == V2_INT && len < 8) {
        uint32_t sh = 64 - 8 * len;
        u = (uint64_t)(((int64_t)(u << sh)) >> sh);
      }
      out->bits = u;
      return DE_NONE;
    }
    // Real: payload copied as FLOAT datum; read_datum_payload_f64 needs 8 bytes
    if (len < 8) return DE_DATUM_DECODE;
    double f = cmp_u64_to_f64(ld_be64(p));
    if (c.tp == B2_TP_FLOAT) f = (double)(float)f;
    if (f != f) { out->null = true; return DE_NONE; }
    out->bits = f64_bits(f);
    return DE_NONE;
  }
  // v1 datum (datum_codec.rs:401-446)
  uint8_t flag = p[0];
  const uint8_t* q = p + 1;
  uint32_t qn = len - 1;
  if (flag == 0) { out->null = true; return DE_NONE; }
  if (c.kind == CK_INT) {
    if (flag == 3) { if (qn < 8) return DE_DATUM_DECODE; out->bits = ld_be64(q) ^ S; return DE_NONE; }
    if (flag == 4) { if (qn < 8) return DE_DATUM_DECODE; out->bits = ld_be64(q); return DE_NONE; }
    if (flag == 8) { int64_t v; if (!dec_var_i64(q, qn, &v)) return DE_DATUM_DECODE; out->bits = (uint64_t)v; return DE_NONE; }
    if (flag == 9) { uint64_t v; if (!dec_var_u64(q, qn, &v)) return DE_DATUM_DECODE; out->bits = v; return DE_NONE; }
    return DE_DATUM_DECODE;
  }
  if (flag == 5) {
    if (qn < 8) return DE_DATUM_DECODE;
    double f = cmp_u64_to_f64(ld_be64(q));
    if (c.tp == B2_TP_FLOAT) f = (double)(float)f;
    if (f != f) { out->null = true; return DE_NONE; }
    out->bits = f64_bits(f);
    return DE_NONE;
  }
  return DE_DATUM_DECODE;
}

// ---- RPN evaluation for one row -----------------------------------------------------------------------
B2_HD int cmp_i64(int64_t a, bool au, int64_t b, bool bu) {  // impl_compare.rs:63-149
  if (!au && !bu) return a < b ? -1 : (a > b ? 1 : 0);
  if (au && bu) return (uint64_t)a < (uint64_t)b ? -1 : ((uint64_t)a > (uint64_t)b ? 1 : 0);
  if (au) { if (b < 0 || a < 0) return 1; return a < b ? -1 : (a > b ? 1 : 0); }
  if (a < 0 || b < 0) return -1;
  return a < b ? -1 : (a > b ? 1 : 0);
}

B2_HD bool add_ovf_i64(int64_t a, int64_t b, int64_t* r) {
  uint64_t s = (uint64_t)a + (uint64_t)b;
  *r = (int64_t)s;
  return ((a ^ (int64_t)s) & (b ^ (int64_t)s)) < 0;
}
B2_HD bool sub_ovf_i64(int64_t a, int64_t b, int64_t* r) {
  uint64_t s = (uint64_t)a - (uint64_t)b;
  *r = (int64_t)s;
  return ((a ^ b) & (a ^ (int64_t)s)) < 0;
}
B2_HD bool add_ovf_u64(uint64_t a, uint64_t b, uint64_t* r) { *r = a + b; return *r < a; }
B2_HD bool sub_ovf_u64(uint64_t a, uint64_t b, uint64_t* r) { *r = a - b; return a < b; }
B2_HD uint64_t mulhi_u64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
B2_HD bool mul_ovf_u64(uint64_t a, uint64_t b, uint64_t* r) { *r = a * b; return mulhi_u64(a, b) != 0; }
B2_HD bool mul_ovf_i64(int64_t a, int64_t b, int64_t* r) {
  // magnitude product must fit: |a*b| <= 2^63-1, or == 2^63 when the result is negative
  uint64_t ua = a < 0 ? (uint64_t)0 - (uint64_t)a : (uint64_t)a, ub = b < 0 ? (uint64_t)0 - (uint64_t)b : (uint64_t)b, m;
  bool neg = (a < 0) != (b < 0);
  if (mul_ovf_u64(ua, ub, &m)) return true;
  if (neg) { if (m > 0x8000000000000000ull) return true; *r = (int64_t)((uint64_t)0 - m); return false; }
  if (m > 0x7fffffffffffffffull) return true;
  *r = (int64_t)m;
  return false;
}
// IEEE round-to-nearest operations that the compiler may not contract into an FMA: in a plan-specialised kernel the
// stack machine is unrolled, and `a * b + c` fused would differ from the reference's separately rounded steps
B2_HD double f64_add(double x, double y) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(x, y);
#else
  return x + y;
#endif
}
B2_HD double f64_sub(double x, double y) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(x, y);
#else
  return x - y;
#endif
}
B2_HD double f64_mul(double x, double y) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(x, y);
#else
  return x * y;
#endif
}
B2_HD double f64_div(double x, double y) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(x, y);
#else
  return x / y;
#endif
}
B2_HD bool f64_finite(double x) { return (f64_bits(x) & 0x7ff0000000000000ull) != 0x7ff0000000000000ull; }
B2_HD bool f64_isinf(double x) { return (f64_bits(x) & 0x7fffffffffffffffull) == 0x7ff0000000000000ull; }

// The less common scalar functions.  They are compiled into plan-specialised kernels only (B2_EXT_SIGS=1, set by jit.cu
// when the plan uses one; the constant plan then keeps just the operators it needs): inside the generic kernels either
// form cost every aggregation 40 % — inlined through code size, out of line through the registers saved around the call
// — so a plan with one of these always runs specialised (engine.cu), and the generic evaluator reports them unsupported.
#ifndef B2_EXT_SIGS
#if defined(__CUDACC__) || defined(B2_NVRTC)
#define B2_EXT_SIGS 0
#else
#define B2_EXT_SIGS 1  // host emulation of the device logic (tests)
#endif
#endif
// ---- Decimal comparison (`Ord for Decimal`, decimal.rs:2323-2338 over calc_sub_carry :265-342) ----
// -1 / 0 / 1 for a < b / a == b / a > b.  Operands are parsed cells (raw_decimal_parse): the signs decide when they differ;
// otherwise the magnitudes compare by the number of integer words left after the leading zero words, then word by word
// through the fraction words (trailing zero words do not count).
B2_HD int dec_cmp_dev(const b2_decimal& a, const b2_decimal& b) {
  if (a.negative != b.negative) return a.negative ? -1 : 1;
  int l_int = (a.int_cnt + 8) / 9, l_frac = (a.frac_cnt + 8) / 9, r_int = (b.int_cnt + 8) / 9, r_frac = (b.frac_cnt + 8) / 9;
  const int l_stop = l_int, r_stop = r_int;
  int l_idx = 0, r_idx = 0;
  while (l_idx < l_stop && a.word_buf[l_idx] == 0) ++l_idx;
  while (r_idx < r_stop && b.word_buf[r_idx] == 0) ++r_idx;
  l_int = l_stop - l_idx; r_int = r_stop - r_idx;
  int carry;  // -1 equal, 0 |a| > |b|, 1 |a| < |b|
  if (r_int > l_int) carry = 1;
  else if (r_int < l_int) carry = 0;
  else {
    int l_end = l_stop + l_frac - 1, r_end = r_stop + r_frac - 1;
    while (l_idx <= l_end && a.word_buf[l_end] == 0) --l_end;
    while (r_idx <= r_end && b.word_buf[r_end] == 0) --r_end;
    while (l_idx <= l_end && r_idx <= r_end && a.word_buf[l_idx] == b.word_buf[r_idx]) { ++l_idx; ++r_idx; }
    if (l_idx <= l_end) carry = (r_idx <= r_end && b.word_buf[r_idx] > a.word_buf[l_idx]) ? 1 : 0;
    else if (r_idx <= r_end) carry = 1;
    else carry = -1;
  }
  if (carry < 0) return 0;
  return ((carry > 0) == (a.negative != 0)) ? 1 : -1;
}

// ---- LIKE (impl_like.rs:7-74) ----
// One character of `s` (n bytes left): its code and, as the return value, its length; 0 at the end.  Binary charset: one byte
// (charset.rs:17-24).  utf8mb4: core::str::next_code_point as CharsetUtf8mb4::decode_one runs it (charset.rs:43-54) -- the
// lead byte gives the length, nothing is validated; a sequence cut off by the end of the string uses what is there.
B2_HD uint32_t like_next(const uint8_t* s, uint32_t n, bool utf8, uint32_t* code) {
  if (n == 0) return 0;
  const uint32_t x = s[0];
  if (!utf8 || x < 128) { *code = x; return 1; }
  const uint32_t y = n > 1 ? (s[1] & 0x3fu) : 0;
  uint32_t ch = ((x & 0x1fu) << 6) | y, len = 2;
  if (x >= 0xe0) {
    const uint32_t yz = (y << 6) | (n > 2 ? (s[2] & 0x3fu) : 0);
    ch = ((x & 0x1fu) << 12) | yz; len = 3;
    if (x >= 0xf0) { ch = ((x & 7u) << 18) | (yz << 6) | (n > 3 ? (s[3] & 0x3fu) : 0); len = 4; }
  }
  *code = ch;
  return len < n ? len : n;
}
// like::<C, CS> for the collators whose force-no-pad comparison of one character is byte equality (binary, *_bin)
B2_HD bool like_match(const uint8_t* t, uint32_t tn, const uint8_t* p, uint32_t pn, uint32_t escape, bool utf8) {
  uint32_t px = 0, tx = 0, next_px = 0, next_tx = 0;
  while (px < pn || tx < tn) {
    uint32_t code = 0, poff = like_next(p + px, pn - px, utf8, &code);
    if (poff) {
      uint32_t tc;
      if (code == '_') {
        const uint32_t toff = like_next(t + tx, tn - tx, utf8, &tc);
        if (toff) { px += poff; tx += toff; continue; }
      } else if (code == '%') {
        px += poff;
        next_px = px;
        if (next_px >= pn) return true;  // the last '%' matches whatever is left
        next_tx = tx;
        continue;
      } else {
        bool stop = false;
        if (code == escape && px + poff < pn) {
          px += poff;
          uint32_t c2;
          poff = like_next(p + px, pn - px, utf8, &c2);
          if (!poff) stop = true;
        }
        if (stop) break;
        const uint32_t toff = like_next(t + tx, tn - tx, utf8, &tc);
        if (toff && toff == poff) {
          bool same = true;
          for (uint32_t i = 0; i < toff; ++i) same = same && t[tx + i] == p[px + i];
          if (same) { tx += toff; px += poff; continue; }
        }
      }
    }
    // mismatch: back to the position after the last '%', one target character further
    if (0 < next_px && next_tx < tn) {
      uint32_t tc;
      const uint32_t toff = like_next(t + next_tx, tn - next_tx, utf8, &tc);
      next_tx += toff ? toff : 1;
      px = next_px;
      tx = next_tx;
      continue;
    }
    return false;
  }
  return true;
}

B2_HD bool is_dec_sig(int sig) { return (sig >= 100 && sig < 170 && sig % 10 == 2) || sig == B2_SIG_IN_DECIMAL || sig == B2_SIG_DECIMAL_IS_NULL; }
B2_HD bool is_ext_sig(int sig) {
  if (sig == B2_SIG_LIKE || is_dec_sig(sig)) return true;
  if ((sig >= B2_SIG_BIT_AND && sig <= B2_SIG_BIT_NEG) || sig == B2_SIG_CAST_INT_AS_INT || sig == B2_SIG_CAST_INT_AS_REAL || sig == B2_SIG_CAST_REAL_AS_REAL) return true;
  return sig == B2_SIG_INT_DIVIDE_INT || sig == B2_SIG_MOD_INT || sig == B2_SIG_MOD_REAL || sig == B2_SIG_DIVIDE_REAL || (sig >= B2_SIG_ABS_INT && sig <= B2_SIG_ABS_REAL) ||
         sig == B2_SIG_UNARY_MINUS_INT || sig == B2_SIG_UNARY_MINUS_REAL || (sig >= B2_SIG_IF_NULL_INT && sig <= B2_SIG_CASE_WHEN_REAL);
}
B2_HD int eval_ext_fn(int sig, int na, bool ret_unsigned, int64_t* sv, uint8_t* sn, int* sp_io, uint32_t* warn) {
  const int64_t I64_MIN = -9223372036854775807ll - 1, I64_MAX = 9223372036854775807ll;
  const int base = *sp_io - na;
  int64_t r = 0;
  bool rn = true;
  if (sig == B2_SIG_IF_INT || sig == B2_SIG_IF_REAL || sig == B2_SIG_CASE_WHEN_INT || sig == B2_SIG_CASE_WHEN_REAL || sig == B2_SIG_COALESCE_INT ||
      sig == B2_SIG_COALESCE_REAL) {
      bool done = false;
      // if_condition (impl_control.rs:88-100), case_when (:34-50), coalesce (impl_compare.rs:239-248): every argument
      // has been evaluated already (RPN), the function only picks one of them
      if (sig == B2_SIG_COALESCE_INT || sig == B2_SIG_COALESCE_REAL) {
        for (int i = 0; i < na; ++i)
          if (!done && !(sn[base + i] & 1)) { r = sv[base + i]; rn = false; done = true; }
      } else if (sig == B2_SIG_IF_INT || sig == B2_SIG_IF_REAL) {
        const int pick = (!(sn[base] & 1) && sv[base] != 0) ? 1 : 2;
        r = sv[base + pick]; rn = sn[base + pick] & 1;
      } else {
        for (int i = 0; i + 1 < na; i += 2)
          if (!done && !(sn[base + i] & 1) && sv[base + i] != 0) { r = sv[base + i + 1]; rn = sn[base + i + 1] & 1; done = true; }
        if (!done && (na & 1)) { r = sv[base + na - 1]; rn = sn[base + na - 1] & 1; }
      }
  } else {
    const int64_t a = sv[base], b = na == 2 ? sv[base + 1] : 0;
    const bool an = sn[base] & 1, au = sn[base] & 2, bn = na == 2 ? (sn[base + 1] & 1) : false, bu = na == 2 ? (sn[base + 1] & 2) : false;
    switch (sig) {
        case B2_SIG_BIT_AND: if (!an && !bn) { rn = false; r = a & b; } break;  // impl_op.rs:144-175
        case B2_SIG_BIT_OR: if (!an && !bn) { rn = false; r = a | b; } break;
        case B2_SIG_BIT_XOR: if (!an && !bn) { rn = false; r = a ^ b; } break;
        case B2_SIG_BIT_NEG: if (!an) { rn = false; r = ~a; } break;
        case B2_SIG_CAST_INT_AS_INT: case B2_SIG_CAST_REAL_AS_REAL: if (!an) { rn = false; r = a; } break;  // impl_cast.rs:281-305, 505-507 (in_union false)
        case B2_SIG_CAST_INT_AS_REAL:  // impl_cast.rs:466-501: `as f64` of the signed value only when both sides are signed
          if (!an) { rn = false; r = (int64_t)f64_bits((au || ret_unsigned) ? (double)(uint64_t)a : (double)a); }
          break;
        case B2_SIG_IF_NULL_INT: case B2_SIG_IF_NULL_REAL:  // impl_control.rs:7-14
          if (!an) { rn = false; r = a; } else if (!bn) { rn = false; r = b; }
          break;
        case B2_SIG_UNARY_MINUS_INT:  // impl_op.rs:70-101 (map_unary_minus_int_func picks by the argument's UNSIGNED flag)
          if (an) break;
          if (au) { if ((uint64_t)a > 0x8000000000000000ull) return DE_OVERFLOW_BIGINT; }
          else if (a == I64_MIN) return DE_OVERFLOW_BIGINT;
          rn = false; r = (int64_t)((uint64_t)0 - (uint64_t)a);
          break;
        case B2_SIG_UNARY_MINUS_REAL: if (!an) { rn = false; r = a ^ I64_MIN; } break;  // :103-107
        case B2_SIG_ABS_INT:  // impl_math.rs:224-231
          if (an) break;
          if (a == I64_MIN) return DE_OVERFLOW_BIGINT;
          rn = false; r = a < 0 ? -a : a;
          break;
        case B2_SIG_ABS_UINT: if (!an) { rn = false; r = a; } break;
        case B2_SIG_ABS_REAL: if (!an) { rn = false; r = a & I64_MAX; } break;
        case B2_SIG_INT_DIVIDE_INT: {  // impl_arithmetic.rs:396-455 over codec/overflow.rs:9-58; x DIV 0 is NULL
          if (an || bn || b == 0) break;
          const uint64_t ua = (uint64_t)a, ub = (uint64_t)b;
          if (!au && !bu) { if (a == I64_MIN && b == -1) return DE_OVERFLOW_DIV; r = a / b; }
          else if (!au && bu) { if (a < 0) { if ((uint64_t)0 - ua >= ub) return DE_OVERFLOW_DIV; r = 0; } else r = (int64_t)(ua / ub); }
          else if (au && bu) r = (int64_t)(ua / ub);
          else { if (b < 0) { if (ua != 0 && (uint64_t)0 - ub <= ua) return DE_OVERFLOW_DIV; r = 0; } else r = (int64_t)(ua / ub); }
          rn = false;
          break;
        }
        case B2_SIG_MOD_INT: {  // :215-278; x % 0 is NULL.  (i64::MIN % -1 is 0 here; the reference's `%` panics on it)
          if (an || bn || b == 0) break;
          const uint64_t ua = (uint64_t)a, ub = (uint64_t)b;
          const uint64_t abs_a = a < 0 ? (uint64_t)0 - ua : ua, abs_b = b < 0 ? (uint64_t)0 - ub : ub;
          if (!au && !bu) r = b == -1 ? 0 : a % b;
          else if (!au && bu) r = a > 0 ? (int64_t)(ua % ub) : (int64_t)((uint64_t)0 - abs_a % ub);
          else if (au && !bu) r = (int64_t)(ua % abs_b);
          else r = (int64_t)(ua % ub);
          rn = false;
          break;
        }
        case B2_SIG_DIVIDE_REAL: {  // :515-533: x / 0 is NULL with warning 1365 (handle_division_by_zero); an infinite quotient overflows
          if (an || bn) break;
          const double y = bits_f64((uint64_t)b);
          if (y == 0.0) { *warn += 1; break; }
          const double z = f64_div(bits_f64((uint64_t)a), y);
          if (f64_isinf(z)) return DE_OVERFLOW_DOUBLE;
          rn = false; r = (int64_t)f64_bits(z);
          break;
        }
        case B2_SIG_MOD_REAL: {  // :280-291
          if (an || bn) break;
          const double y = bits_f64((uint64_t)b);
          if (y == 0.0) break;
          rn = false; r = (int64_t)f64_bits(fmod(bits_f64((uint64_t)a), y));
          break;
        }
        default: return DE_UNSUPPORTED_SIG;
    }
  }
  sv[base] = rn ? 0 : r; sn[base] = (rn ? 1 : 0) | (ret_unsigned ? 2 : 0);
  *sp_io = base + 1;
  return DE_NONE;
}

B2_HD bool plan_uses_ext_sigs(const DevPlan& P) {
  for (int i = 0; i < P.n_nodes; ++i)
    if (P.nodes[i].kind == B2_RPN_FN && is_ext_sig(P.nodes[i].sig)) return true;
  return false;
}

B2_HD int eval_expr_general(const DevPlan& P, DevExpr ex, const Row& row, const Cells& cells, Value* result, bool* res_unsigned);

// leaf node (column reference or constant) -> value + flags (bit0 null, bit1 unsigned)
B2_HD int eval_leaf(const DevPlan& P, const DevNode& nd, const Row& row, const Cells& cells, int64_t* v, uint32_t* f) {
  if (nd.kind == B2_RPN_COLUMN_REF) {
    Value x;
    int e = cell_value(P, row, cells, (int)nd.imm, &x);
    if (e) return e;
    *v = (int64_t)x.bits; *f = (x.null ? 1u : 0u) | (P.cols[nd.imm].is_unsigned ? 2u : 0u);
    if (P.cols[nd.imm].kind == CK_TIME) { *v &= ~15ll; *f |= 2u; }  // `Ord for Time`: the fsp / time-type bits do not take part; the rest orders as u64
    return DE_NONE;
  }
  *v = node_imm(row, nd); *f = (nd.kind == B2_RPN_CONST_NULL ? 1u : 0u) | (nd.is_unsigned ? 2u : 0u);
  return DE_NONE;
}

// RpnExpression::eval for one row.  Leaves and `leaf <cmp> leaf` (the shape of almost every pushed-down predicate,
// group key and aggregate argument) are evaluated in registers; everything else goes through the stack machine.
B2_HD int eval_expr(const DevPlan& P, DevExpr ex, const Row& row, const Cells& cells, Value* result, bool* res_unsigned) {
  const DevNode& n0 = P.nodes[ex.start];
  if (ex.n == 1 && n0.kind != B2_RPN_FN) {
    int64_t v; uint32_t f;
    int e = eval_leaf(P, n0, row, cells, &v, &f);
    if (e) return e;
    result->bits = (uint64_t)v; result->null = f & 1;
    if (res_unsigned) *res_unsigned = f & 2;
    return DE_NONE;
  }
  if (ex.n == 3) {
    const DevNode& n1 = P.nodes[ex.start + 1];
    const DevNode& n2 = P.nodes[ex.start + 2];
    int sig = n2.sig;
    if (n0.kind != B2_RPN_FN && n1.kind != B2_RPN_FN && n2.kind == B2_RPN_FN && sig >= 100 && sig < 160 && sig % 10 <= 1) {  // (Int / Real compares: the others carry cell references)
      int64_t a, b; uint32_t af, bf;
      int e = eval_leaf(P, n0, row, cells, &a, &af);
      if (e) return e;
      e = eval_leaf(P, n1, row, cells, &b, &bf);
      if (e) return e;
      if (res_unsigned) *res_unsigned = n2.is_unsigned;
      if ((af | bf) & 1) { result->null = true; result->bits = 0; return DE_NONE; }  // NULL-propagating compare
      int c;
      if (sig % 10 == 1) { double x = bits_f64((uint64_t)a), y = bits_f64((uint64_t)b); c = x < y ? -1 : (x > y ? 1 : 0); }
      else c = cmp_i64(a, af & 2, b, bf & 2);
      bool t;
      switch (sig / 10 * 10) {
        case B2_SIG_LT_INT: t = c < 0; break;
        case B2_SIG_LE_INT: t = c <= 0; break;
        case B2_SIG_GT_INT: t = c > 0; break;
        case B2_SIG_GE_INT: t = c >= 0; break;
        case B2_SIG_NE_INT: t = c != 0; break;
        default: t = c == 0; break;
      }
      result->null = false; result->bits = t;
      return DE_NONE;
    }
  }
  return eval_expr_general(P, ex, row, cells, result, res_unsigned);
}

B2_HD int eval_expr_general(const DevPlan& P, DevExpr ex, const Row& row, const Cells& cells, Value* result, bool* res_unsigned) {
  int64_t sv[MAX_STACK];
  uint8_t sn[MAX_STACK];  // bit0 null, bit1 unsigned
  int sp = 0;
  for (uint32_t k = ex.start; k < (uint32_t)ex.start + ex.n; ++k) {
    const DevNode& nd = P.nodes[k];
    if (nd.kind == B2_RPN_COLUMN_REF) {
      Value v;
      int e = cell_value(P, row, cells, (int)nd.imm, &v);
      if (e) return e;
      sv[sp] = (int64_t)v.bits; sn[sp] = (v.null ? 1 : 0) | (P.cols[nd.imm].is_unsigned ? 2 : 0);
      if (P.cols[nd.imm].kind == CK_TIME) { sv[sp] &= ~15ll; sn[sp] |= 2; }
      ++sp;
      continue;
    }
    if (nd.kind != B2_RPN_FN) {  // constants
      sv[sp] = node_imm(row, nd); sn[sp] = (nd.kind == B2_RPN_CONST_NULL ? 1 : 0) | (nd.is_unsigned ? 2 : 0);
      ++sp;
      continue;
    }
    if (nd.sig == B2_SIG_IN_INT || nd.sig == B2_SIG_IN_REAL) {
      // compare_in_int_type_by_hash / compare_in_by_hash (impl_compare_in.rs:178-258): NULL base -> NULL; a list value
      // equal to the base -> 1 (integers of different signedness only match when the base is non-negative);
      // otherwise NULL if the list held a NULL, else 0
      const int base = sp - nd.n_args;
      const int64_t x = sv[base];
      const bool xn = sn[base] & 1, xu = sn[base] & 2;
      bool hit = false, has_null = false;
      for (int i = 1; i < nd.n_args; ++i) {
        const int64_t y = sv[base + i];
        if (sn[base + i] & 1) { has_null = true; continue; }
        if (nd.sig == B2_SIG_IN_REAL) hit |= bits_f64((uint64_t)x) == bits_f64((uint64_t)y);
        else hit |= x == y && (x >= 0 || xu == (bool)(sn[base + i] & 2));
      }
      sp = base;
      sv[sp] = hit ? 1 : 0; sn[sp] = (xn || (!hit && has_null)) ? 1 : 0;
      ++sp;
      continue;
    }
#if B2_EXT_SIGS
    if (is_dec_sig(nd.sig)) {  // operands: cell references to (precision, fraction, binary decimal) payloads, columns and constants alike
      const int na = nd.n_args, base = sp - na;
      int64_t r = 0; bool rn = true;
      if (nd.sig == B2_SIG_DECIMAL_IS_NULL) { rn = false; r = sn[base] & 1; }
      else {
        b2_decimal x;
        const bool xn = sn[base] & 1;
        if (!xn && !raw_decimal_parse(raw_ref_addr((uint64_t)sv[base]), raw_ref_len((uint64_t)sv[base]), &x)) return DE_DATUM_DECODE;
        if (nd.sig == B2_SIG_IN_DECIMAL) {
          bool hit = false, has_null = false;
          for (int i = 1; i < na; ++i) {
            if (sn[base + i] & 1) { has_null = true; continue; }
            b2_decimal y;
            if (!raw_decimal_parse(raw_ref_addr((uint64_t)sv[base + i]), raw_ref_len((uint64_t)sv[base + i]), &y)) return DE_DATUM_DECODE;
            if (!xn) hit |= dec_cmp_dev(x, y) == 0;
          }
          rn = xn || (!hit && has_null); r = hit;
        } else {
          const bool yn = sn[base + 1] & 1, nulleq = nd.sig == B2_SIG_NULLEQ_DECIMAL;
          b2_decimal y;
          if (!yn && !raw_decimal_parse(raw_ref_addr((uint64_t)sv[base + 1]), raw_ref_len((uint64_t)sv[base + 1]), &y)) return DE_DATUM_DECODE;
          if (xn || yn) { if (nulleq) { rn = false; r = xn && yn; } }
          else {
            const int c = dec_cmp_dev(x, y);
            rn = false;
            switch (nd.sig) {
              case B2_SIG_LT_DECIMAL: r = c < 0; break;
              case B2_SIG_LE_DECIMAL: r = c <= 0; break;
              case B2_SIG_GT_DECIMAL: r = c > 0; break;
              case B2_SIG_GE_DECIMAL: r = c >= 0; break;
              case B2_SIG_NE_DECIMAL: r = c != 0; break;
              default: r = c == 0; break;  // EQ, NULLEQ
            }
          }
        }
      }
      sv[base] = rn ? 0 : r; sn[base] = rn ? 1 : 0;
      sp = base + 1;
      continue;
    }
    if (nd.sig == B2_SIG_LIKE) {  // (target, pattern: cell references into HBM; escape: int) -> int; NULL if any argument is
      const int base = sp - 3;
      const bool nul = (sn[base] | sn[base + 1] | sn[base + 2]) & 1;
      const uint64_t tr = (uint64_t)sv[base], pr = (uint64_t)sv[base + 1];
      sv[base] = nul ? 0 : (int64_t)like_match(raw_ref_addr(tr), raw_ref_len(tr), raw_ref_addr(pr), raw_ref_len(pr), (uint32_t)sv[base + 2], nd.imm != 0);
      sn[base] = nul ? 1 : 0;
      sp = base + 1;
      continue;
    }
#endif
    if (is_ext_sig(nd.sig)) {
#if B2_EXT_SIGS
      int e = eval_ext_fn(nd.sig, nd.n_args, nd.is_unsigned, sv, sn, &sp, &row.warn);
      if (e) return e;
      continue;
#else
      return DE_UNSUPPORTED_SIG;  // never reached: such plans only run on their specialised kernel
#endif
    }
    int64_t b = 0; uint8_t bf = 0;
    if (nd.n_args == 2) { --sp; b = sv[sp]; bf = sn[sp]; }
    --sp;
    int64_t a = sv[sp]; uint8_t af = sn[sp];
    bool an = af & 1, bn = bf & 1, au = af & 2, bu = bf & 2;
    int64_t r = 0; bool rn = true;
    int sig = nd.sig;
    int base = sig / 10 * 10;
    bool real = (sig % 10) == 1;
    if (sig >= 100 && sig < 170) {  // comparisons
      bool nulleq = base == B2_SIG_NULLEQ_INT;
      if (an && bn) { if (nulleq) { rn = false; r = 1; } }
      else if (an || bn) { if (nulleq) { rn = false; r = 0; } }
      else {
        int c;
        if (real) { double x = bits_f64((uint64_t)a), y = bits_f64((uint64_t)b); c = x < y ? -1 : (x > y ? 1 : 0); }
        else c = cmp_i64(a, au, b, bu);
        bool t;
        switch (base) {
          case B2_SIG_LT_INT: t = c < 0; break;
          case B2_SIG_LE_INT: t = c <= 0; break;
          case B2_SIG_GT_INT: t = c > 0; break;
          case B2_SIG_GE_INT: t = c >= 0; break;
          case B2_SIG_NE_INT: t = c != 0; break;
          default: t = c == 0; break;  // EQ, NULLEQ
        }
        rn = false; r = t;
      }
    } else {
      switch (sig) {
        case B2_SIG_LOGICAL_AND:
          if ((!an && a == 0) || (!bn && b == 0)) { rn = false; r = 0; }
          else if (!an && !bn) { rn = false; r = 1; }
          break;
        case B2_SIG_LOGICAL_OR:
          if (!an && !bn && a == 0 && b == 0) { rn = false; r = 0; }
          else if ((an && bn) || (an && b == 0) || (bn && a == 0)) {}
          else { rn = false; r = 1; }
          break;
        case B2_SIG_LOGICAL_XOR: if (!an && !bn) { rn = false; r = (a == 0) != (b == 0); } break;
        case B2_SIG_UNARY_NOT_INT: if (!an) { rn = false; r = a == 0; } break;
        case B2_SIG_UNARY_NOT_REAL: if (!an) { rn = false; r = bits_f64((uint64_t)a) == 0.0; } break;
        case B2_SIG_INT_IS_NULL: case B2_SIG_REAL_IS_NULL: rn = false; r = an; break;
        case B2_SIG_INT_IS_TRUE: rn = false; r = !an && a != 0; break;
        case B2_SIG_REAL_IS_TRUE: rn = false; r = !an && bits_f64((uint64_t)a) != 0.0; break;
        case B2_SIG_INT_IS_FALSE: rn = false; r = !an && a == 0; break;
        case B2_SIG_REAL_IS_FALSE: rn = false; r = !an && bits_f64((uint64_t)a) == 0.0; break;
        case B2_SIG_PLUS_INT: case B2_SIG_MINUS_INT: case B2_SIG_MULTIPLY_INT: case B2_SIG_MULTIPLY_INT_UNSIGNED: {
          if (an || bn) break;
          bool xu = au, yu = bu, ovf;
          if (sig == B2_SIG_MULTIPLY_INT_UNSIGNED) xu = yu = true;
          uint64_t w = 0;
          if (sig == B2_SIG_PLUS_INT) {
            if (!xu && !yu) ovf = add_ovf_i64(a, b, &r);
            else if (xu && yu) { ovf = add_ovf_u64((uint64_t)a, (uint64_t)b, &w); r = (int64_t)w; }
            else {
              int64_t s = xu ? b : a; uint64_t u = (uint64_t)(xu ? a : b);
              if (s >= 0) ovf = add_ovf_u64((uint64_t)s, u, &w); else ovf = sub_ovf_u64(u, (uint64_t)0 - (uint64_t)s, &w);
              r = (int64_t)w;
            }
          } else if (sig == B2_SIG_MINUS_INT) {
            if (!xu && !yu) ovf = sub_ovf_i64(a, b, &r);
            else if (xu && yu) { ovf = sub_ovf_u64((uint64_t)a, (uint64_t)b, &w); r = (int64_t)w; }
            else if (!xu) { if (a >= 0) ovf = sub_ovf_u64((uint64_t)a, (uint64_t)b, &w); else ovf = true; r = (int64_t)w; }
            else { if (b >= 0) ovf = sub_ovf_u64((uint64_t)a, (uint64_t)b, &w); else ovf = add_ovf_u64((uint64_t)a, (uint64_t)0 - (uint64_t)b, &w); r = (int64_t)w; }
          } else {
            if (!xu && !yu) ovf = mul_ovf_i64(a, b, &r);
            else if (xu && yu) { ovf = mul_ovf_u64((uint64_t)a, (uint64_t)b, &w); r = (int64_t)w; }
            else { int64_t s = xu ? b : a; uint64_t u = (uint64_t)(xu ? a : b); if (s >= 0) ovf = mul_ovf_u64((uint64_t)s, u, &w); else ovf = true; r = (int64_t)w; }
          }
          if (ovf) return (xu || yu) ? DE_OVERFLOW_UBIGINT : DE_OVERFLOW_BIGINT;
          rn = false;
          break;
        }
        case B2_SIG_PLUS_REAL: case B2_SIG_MINUS_REAL: case B2_SIG_MULTIPLY_REAL: {
          if (an || bn) break;
          double x = bits_f64((uint64_t)a), y = bits_f64((uint64_t)b);
          double z = sig == B2_SIG_PLUS_REAL ? f64_add(x, y) : (sig == B2_SIG_MINUS_REAL ? f64_sub(x, y) : f64_mul(x, y));
          bool bad = sig == B2_SIG_MULTIPLY_REAL ? f64_isinf(z) : !f64_finite(z);
          if (bad) return DE_OVERFLOW_DOUBLE;
          rn = false; r = (int64_t)f64_bits(z);
          break;
        }
        default: return DE_UNSUPPORTED_SIG;
      }
    }
    sv[sp] = r; sn[sp] = (rn ? 1 : 0) | (nd.is_unsigned ? 2 : 0);
    ++sp;
  }
  result->bits = (uint64_t)sv[0];
  result->null = sn[0] & 1;
  if (res_unsigned) *res_unsigned = sn[0] & 2;
  return DE_NONE;
}

// AND of the selection conditions on one row (selection_executor.rs:81-195): sequential, stop at first false/NULL
B2_HD int eval_conds(const DevPlan& P, const Row& row, const Cells& cells, bool* keep) {
  *keep = true;
  if (row.fast && P.n_fconds > 0) {
    // every condition is `integer column <cmp> constant` and the row has the exact layout: no NULLs, no decode errors,
    // the column is read by stored position (impl_compare.rs:63-149 semantics through cmp_i64)
    for (int i = 0; i < P.n_fconds; ++i) {
      const FastCond f = P.fconds[i];
      const int c = cmp_i64((int64_t)(((row.cv_mask >> f.h) & 1u) ? row.cv[f.h] : fast_cell_dyn(row, f.h, f.zero_ext, P.fast_v1 != 0)), f.col_uns, f.imm_slot ? row.imms[f.imm_slot - 1] : f.imm, f.imm_uns);
      bool t;
      switch (f.op) {
        case 0: t = c < 0; break;
        case 1: t = c <= 0; break;
        case 2: t = c > 0; break;
        case 3: t = c >= 0; break;
        case 4: t = c == 0; break;
        default: t = c != 0; break;
      }
      if (!t) { *keep = false; return DE_NONE; }
    }
    return DE_NONE;
  }
  for (int i = 0; i < P.n_conds; ++i) {
    Value v;
    const DevExpr ex = P.conds[i];
    int e = eval_expr(P, ex, row, cells, &v, nullptr);
    if (e) return e;
    bool t;
    if (v.null) t = false;
    else if (P.nodes[ex.start + ex.n - 1].et == 1) t = bits_f64(v.bits) != 0.0;
    else t = v.bits != 0;
    if (!t) { *keep = false; return DE_NONE; }
  }
  return DE_NONE;
}

// ---- exact SUM over Real ------------------------------------------------------------------------------------------
// AggrFnSum<Real> (impl_sum.rs:71-150, summable.rs:25-87) adds f64 values in row order; any parallel order rounds
// differently.  The device therefore accumulates every value exactly: the sum lives in a 2112-bit fixed-point number
// (bit 0 = 2^-1074, enough for every finite double) held as F64_ACC_DIGITS 32-bit digits, one per u64 word, carry-save
// (a word takes 2^31 additions before it could overflow).  Adding a value is at most three integer atomic adds, merging
// two partial sums (CTAs, launches, GPUs) is word-wise integer addition, and f64_acc_round delivers the correctly rounded
// (round-to-nearest-even) double of the exact sum: deterministic, independent of order, within 0.5 ULP of the true sum
// (the reference's own sequential result is within (n-1) ulps-of-partial-sums of it).
enum { F64_ACC_DIGITS = 66 };
// x (finite) = sign * m * 2^(s - 1074), m < 2^53, s = max(exponent field, 1) - 1: pieces of m << (s & 31) at digit s >> 5
template <class AddFn>
B2_HD void f64_acc_add(uint64_t bits, AddFn add) {
  uint64_t m = bits & 0xfffffffffffffull;
  uint32_t e = (uint32_t)(bits >> 52) & 0x7ffu;
  if (e) m |= 1ull << 52; else e = 1;
  if (!m) return;
  const uint32_t s = e - 1, d = s >> 5, o = s & 31u;
  const uint64_t lo64 = m << o;
  const uint64_t hi = o ? (m >> (64 - o)) : 0ull;
  int64_t p0 = (int64_t)(lo64 & 0xffffffffull), p1 = (int64_t)(lo64 >> 32), p2 = (int64_t)hi;
  if (bits >> 63) { p0 = -p0; p1 = -p1; p2 = -p2; }
  if (p0) add(d, p0);
  if (p1) add(d + 1, p1);
  if (p2) add(d + 2, p2);
}
// the correctly rounded value of the accumulator (w: F64_ACC_DIGITS carry-save words)
template <class W>
B2_HD uint64_t f64_acc_round(const W* w) {
  uint32_t dig[F64_ACC_DIGITS + 1];
  int64_t carry = 0;
  for (int i = 0; i < F64_ACC_DIGITS; ++i) {
    const int64_t v = (int64_t)w[i] + carry;  // |w[i]| < 2^63 - 2^32 by construction
    dig[i] = (uint32_t)v;
    carry = v >> 32;
  }
  dig[F64_ACC_DIGITS] = (uint32_t)carry;
  const bool neg = carry < 0;
  if (neg) {  // two's complement magnitude
    uint64_t c = 1;
    for (int i = 0; i <= F64_ACC_DIGITS; ++i) { c += (uint32_t)~dig[i]; dig[i] = (uint32_t)c; c >>= 32; }
  }
  int top = F64_ACC_DIGITS;
  while (top >= 0 && dig[top] == 0) --top;
  if (top < 0) return 0;  // +0.0
  uint32_t t = dig[top], lz = 0;
  while (!(t & 0x80000000u)) { t <<= 1; ++lz; }
  const int p = 32 * top + 31 - (int)lz;  // position of the most significant bit
  const uint64_t sign = neg ? 0x8000000000000000ull : 0ull;
  auto digit = [&](int i) -> uint64_t { return i >= 0 && i <= F64_ACC_DIGITS ? dig[i] : 0u; };
  if (p <= 52) return sign | (digit(0) | (digit(1) << 32));  // subnormal, or exponent field 1: the bits are the value
  const int q = p - 52, k = q >> 5, r = q & 31;  // mantissa = 53 bits from position q
  const uint64_t lo = digit(k) | (digit(k + 1) << 32), hi = digit(k + 2);
  uint64_t m = (r ? ((lo >> r) | (hi << (64 - r))) : lo) & ((1ull << 53) - 1);
  // round to nearest even on the bits below q
  const int gq = q - 1;
  const bool guard = (digit(gq >> 5) >> (gq & 31)) & 1u;
  bool sticky = (digit(gq >> 5) & ((1ull << (gq & 31)) - 1)) != 0;
  for (int i = (gq >> 5) - 1; i >= 0 && !sticky; --i) sticky = dig[i] != 0;
  uint64_t e = (uint64_t)(q + 1);
  if (guard && (sticky || (m & 1))) {
    ++m;
    if (m >> 53) { m >>= 1; ++e; }
  }
  if (e >= 2047) return sign | 0x7ff0000000000000ull;  // beyond DBL_MAX
  return sign | (e << 52) | (m & 0xfffffffffffffull);
}

// MAX / MIN state (impl_max_min.rs:425-560): [count of non-NULL inputs, extremum key].  The key is an order-preserving
// u64 (signed: sign flip; unsigned: as is; real: IEEE total order), complemented for MIN, so that both are a running
// unsigned maximum over a zero-initialised word (atomicMax), additive-style mergeable across CTAs and GPUs.
B2_HD uint64_t extremum_key(uint64_t bits, int arg_et, bool arg_unsigned, bool is_min) {
  uint64_t k = bits;
  if (arg_et == 1) {
    if ((k << 1) == 0) k = 0;  // -0.0 == 0.0
    k = (k >> 63) ? ~k : (k | 0x8000000000000000ull);
  } else if (!arg_unsigned) k ^= 0x8000000000000000ull;
  return is_min ? ~k : k;
}
B2_HD uint64_t extremum_value(uint64_t key, int arg_et, bool arg_unsigned, bool is_min) {
  uint64_t k = is_min ? ~key : key;
  if (arg_et == 1) return (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
  return arg_unsigned ? k : (k ^ 0x8000000000000000ull);
}

// FIRST / BIT_AND / BIT_OR / BIT_XOR state.  Every state is all-zero words before its first row, like the others.
//   BIT_OR  [bits]: |= v          BIT_XOR [bits]: ^= v          BIT_AND [bits]: |= ~v, the result is ~bits
//   FIRST   [key, value] at an even word: the pair with the larger key wins (128-bit compare-and-swap); key 0 = no row
// (impl_bit_op.rs BitOp::init_state / AggrFnStateBitOp::update_concrete: NULL inputs are skipped, the state starts at
// !0 / 0 / 0; impl_first.rs AggrFnStateFirst::update: the first row's value, NULL included)
B2_HD bool agg_is_extremum(int kind) { return kind == AGG_MAX || kind == AGG_MIN; }
B2_HD bool agg_is_bit(int kind) { return kind >= AGG_BIT_AND; }
// the word a BIT_* row contributes (0 for NULL: the identity of OR and XOR)
B2_HD uint64_t bit_agg_word(int kind, bool has, uint64_t bits) { return !has ? 0ull : (kind == AGG_BIT_AND ? ~bits : bits); }
// FIRST's key of the row at block entry `entry`: 2^63 | ((2^62 - 1 - r) << 1) | is_null, where r is the row's rank in scan
// order.  It is the TopN tie rule (`desc ? ~entry : entry`): ranges arrive ascending and non-overlapping, so entries rise in
// a forward scan and fall in a backward one.  A larger key is a row scanned earlier; the lean kernel and the list-mode
// kernel commit different rows of one unit and must agree on this key.
B2_HD uint64_t first_agg_key(uint64_t entry, bool desc, bool is_null) {
  const uint64_t r62 = (1ull << 62) - 1, r = desc ? r62 - entry : entry;
  return (1ull << 63) | ((r62 - r) << 1) | (is_null ? 1ull : 0ull);
}
// one row into a FIRST / BIT_* state, sequentially (what the kernels' pre-aggregation and atomics compute)
B2_HD void first_bit_update(int kind, uint64_t* w, uint64_t entry, bool desc, bool has, uint64_t bits) {
  if (kind == AGG_FIRST) {
    const uint64_t key = first_agg_key(entry, desc, !has);
    if (key > w[0]) { w[0] = key; w[1] = has ? bits : 0ull; }
  } else if (kind == AGG_BIT_XOR) w[0] ^= bit_agg_word(kind, has, bits);
  else w[0] |= bit_agg_word(kind, has, bits);
}
// the result cell of a FIRST / BIT_* state; false = NULL (FIRST without a row, or whose first row's value is NULL)
B2_HD bool first_bit_result(int kind, const uint64_t* w, uint64_t* out) {
  if (kind == AGG_FIRST) {
    const bool has = w[0] != 0 && !(w[0] & 1);
    *out = has ? w[1] : 0ull;
    return has;
  }
  *out = kind == AGG_BIT_AND ? ~w[0] : w[0];
  return true;
}
// how a word of the accumulator state merges (b2_exec_agg_word_ops); the FIRST value word follows its key word
B2_HD int agg_word_op(const DevPlan& P, int w) {
  for (int a = 0; a < P.n_aggs; ++a) {
    const DevAgg& g = P.aggs[a];
    if (agg_is_extremum(g.kind) && w == g.acc_off + 1) return B2_MERGE_MAX;
    if ((g.kind == AGG_BIT_AND || g.kind == AGG_BIT_OR) && w == g.acc_off) return B2_MERGE_OR;
    if (g.kind == AGG_BIT_XOR && w == g.acc_off) return B2_MERGE_XOR;
    if (g.kind == AGG_FIRST && w == g.acc_off) return B2_MERGE_FIRST_KEY;
    if (g.kind == AGG_FIRST && w == g.acc_off + 1) return B2_MERGE_FIRST_VALUE;
  }
  return B2_MERGE_ADD;  // counts, integer limbs, the digits of exact Real sums and alignment padding
}
#ifdef __CUDACC__
// FIRST: store (key, value) at `w` (16-byte aligned, shared or global) unless the stored key is at least as large
__device__ __forceinline__ void first_agg_update(unsigned long long* w, unsigned long long key, unsigned long long value) {
  unsigned long long lo = *(volatile unsigned long long*)&w[0];
  while (key > lo) {
    unsigned long long hi = *(volatile unsigned long long*)&w[1];
    const unsigned long long want_lo = lo, want_hi = hi;
    asm volatile("{\n\t.reg .b128 d, c, s;\n\tmov.b128 c, {%0, %1};\n\tmov.b128 s, {%2, %3};\n\tatom.cas.b128 d, [%4], c, s;\n\tmov.b128 {%0, %1}, d;\n\t}"
                 : "+l"(lo), "+l"(hi) : "l"(key), "l"(value), "l"(w) : "memory");
    if (lo == want_lo && hi == want_hi) break;
  }
}
#endif

// one output cell of a PM_SCAN pipeline: a scan column (LazyBatchColumn::ensure_decoded) or, under a Projection
// (projection_executor.rs:199-222), the value of its `oc`-th selected expression
B2_HD int output_value(const DevPlan& P, const Row& row, const Cells& cells, int oc, Value* v) {
  if (P.n_proj) return eval_expr(P, P.proj[P.out_cols[oc]], row, cells, v, nullptr);
  return cell_value(P, row, cells, P.out_cols[oc], v);
}

// fx-like 64-bit mixer for the group hash table (any good mixer works: group order is unspecified)
B2_HD uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

// CRC-64/XZ bytewise step table entry (reflected poly 0xC96C5795D7870F42), computed — not stored — on the host
B2_HD uint64_t crc64_table_entry(uint32_t i) {
  uint64_t c = i;
  for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xC96C5795D7870F42ull : (c >> 1);
  return c;
}

// exact i128/u128 value hi * 2^32 + lo -> MySQL Decimal words (base 1e9), canonical form of Decimal::from (decimal.rs:1787-1815)
B2_HD void limbs_to_decimal(unsigned long long lo, unsigned long long hi, bool is_unsigned, b2_decimal* d) {
  // value = hi * 2^32 + lo as 128-bit two's complement (hi sign-extended when signed)
  unsigned long long w0 = lo + (hi << 32);                 // low 64 bits
  unsigned long long carry = w0 < lo ? 1ull : 0ull;
  unsigned long long hi_ext = is_unsigned ? (hi >> 32) : (unsigned long long)((long long)hi >> 32);
  unsigned long long w1 = hi_ext + carry;                  // high 64 bits
  bool neg = !is_unsigned && ((long long)w1 < 0);
  if (neg) {  // magnitude
    w0 = ~w0 + 1;
    w1 = ~w1 + (w0 == 0 ? 1ull : 0ull);
  }
  // repeated division of the 128-bit magnitude by 1e9 using 32-bit limbs
  unsigned int limb[4] = {(unsigned int)(w1 >> 32), (unsigned int)w1, (unsigned int)(w0 >> 32), (unsigned int)w0};
  unsigned int words[9];
  int nw = 0;
  for (;;) {
    unsigned long long rem = 0;
    bool nonzero = false;
    for (int i = 0; i < 4; ++i) {
      unsigned long long cur = (rem << 32) | limb[i];
      limb[i] = (unsigned int)(cur / 1000000000ull);
      rem = cur % 1000000000ull;
      nonzero |= limb[i] != 0;
    }
    words[nw++] = (unsigned int)rem;
    if (!nonzero || nw == 9) break;
  }
  d->int_cnt = (uint8_t)(nw * 9); d->frac_cnt = 0; d->result_frac_cnt = 0; d->negative = neg;
  for (int i = 0; i < 9; ++i) d->word_buf[i] = i < nw ? words[nw - 1 - i] : 0;
}


// One TopN candidate: order-by values as order-preserving words + global entry id as the final tie-break
// (earlier rows win ties, like TopNHeap::add_row's strict `<`, top_n_heap.rs:46-50).
struct TopItem {
  unsigned long long w[MAX_ORDER];
  unsigned long long id;  // global CF_WRITE entry index of the row's first version
  unsigned int nulls;     // bit k: order-by value k is NULL; bit 31: empty slot (sorts last)
  unsigned int slot;      // (source list << 16) | index, filled by the merge kernel
};

// HeapItemUnsafe::cmp_sort_key (top_n_heap.rs:188-222) + ScalarValueRef::cmp_sort_key (scalar.rs:374-411):
// column by column, NULL < any value, unsigned compare for unsigned field types, reversed for DESC; the entry id
// makes the order total so that the earliest rows win ties.
B2_HD bool item_less(const TopItem& a, const TopItem& b, const DevPlan& P) {
  bool ea = a.nulls >> 31, eb = b.nulls >> 31;
  if (ea || eb) return !ea && eb;
  for (int k = 0; k < P.n_order; ++k) {
    unsigned int na = (a.nulls >> k) & 1, nb = (b.nulls >> k) & 1;
    int c;
    if (na || nb) c = (int)nb - (int)na;  // NULL (n=1) sorts first: a NULL, b not -> -1
    else c = a.w[k] < b.w[k] ? -1 : (a.w[k] > b.w[k] ? 1 : 0);
    if (c == 0) continue;
    if (P.order[k].desc) c = -c;
    return c < 0;
  }
  return a.id < b.id;
}

// order-preserving word of one non-NULL order-by value (sign flip / IEEE total order, -0.0 == 0.0)
B2_HD unsigned long long order_key_word(const DevOrder& o, unsigned long long w) {
  if (o.et == 1) {
    if (bits_f64(w) == 0.0) w = 0;
    return (w >> 63) ? ~w : (w | 0x8000000000000000ull);
  }
  return o.is_unsigned ? w : (w ^ 0x8000000000000000ull);
}
// Can a row whose FIRST sort key is `v0` still beat `thr`?  (false = it certainly cannot: skip the rest of its keys)
B2_HD bool first_key_may_beat(const DevPlan& P, const Value& v0, const TopItem& thr) {
  const unsigned int tn = thr.nulls & 1u, rn = v0.null ? 1u : 0u;
  int c;
  if (rn || tn) c = (int)tn - (int)rn;  // NULL sorts first
  else { const unsigned long long w = order_key_word(P.order[0], v0.bits); c = w < thr.w[0] ? -1 : (w > thr.w[0] ? 1 : 0); }
  if (P.order[0].desc) c = -c;
  return c <= 0;
}

// `first`: the row's first sort key when the caller has evaluated it already (evaluated twice, it would warn twice)
B2_HD int make_item(const DevPlan& P, const Row& row, const Cells& cells, uint64_t id, TopItem* it, const Value* first = nullptr) {
  it->nulls = 0; it->id = id; it->slot = 0;
  for (int k = 0; k < MAX_ORDER; ++k) it->w[k] = 0;
  for (int k = 0; k < P.n_order; ++k) {
    Value v;
    if (k == 0 && first) v = *first;
    else if (int e = eval_expr(P, P.order[k].e, row, cells, &v, nullptr)) return e;
    if (v.null) { it->nulls |= 1u << k; continue; }
    it->w[k] = order_key_word(P.order[k], v.bits);
  }
  return DE_NONE;
}


}  // namespace b2
