/*
 * b2_copr.h — C ABI of the GPU-native (H100, sm_90a) coprocessor batch-execution engine.
 *
 * This is the drop-in boundary for TiKV's DAG-pushdown hot path.  Every entry
 * point names the reference interface it replaces (paths relative to the
 * tikv/tikv tree):
 *
 *   b2_exec_*           <- trait BatchExecutor
 *                          components/tidb_query_executors/src/interface.rs:36-97
 *   b2_batch            <- struct BatchExecuteResult             interface.rs:205-236
 *   b2_dag_handle       <- RequestHandler::handle_request for BatchDagHandler
 *                          src/coprocessor/mod.rs:67-94, src/coprocessor/dag/mod.rs:189-192
 *   b2_check_supported  <- BatchExecutorsRunner::check_supported
 *                          components/tidb_query_executors/src/runner.rs:111-206
 *   b2_checksum_handle  <- ChecksumContext::handle_request       src/coprocessor/checksum.rs:59-98
 *   b2_region_source    <- trait Storage (bulk instead of row-at-a-time pull)
 *                          components/tidb_query_common/src/storage/mod.rs:32-71
 *   b2_dag_plan         <- tipb::DagRequest as consumed by build_executors, runner.rs:252-603
 *   b2_sst_decode       <- the RocksDB data-block iterator under RegionSnapshot / Cursor
 *                          (components/engine_rocks, external librocksdb: BlockBasedTable data blocks;
 *                          block size / format version set in src/config/mod.rs:966, :704)
 *
 * Plain C types only: pointers, sizes, PODs.  No C++/torch types cross this line.
 * Handles are single-threaded (externally synchronised), like `BatchExecutor: Send`.
 * Output memory is callee-owned and valid until the next call on the same handle.
 */
#ifndef B2_COPR_H_
#define B2_COPR_H_

#ifdef B2_NVRTC /* run-time compilation of the plan-specialised kernel: no host headers */
typedef signed char int8_t; typedef unsigned char uint8_t; typedef short int16_t; typedef unsigned short uint16_t;
typedef int int32_t; typedef unsigned int uint32_t; typedef long long int64_t; typedef unsigned long long uint64_t;
#else
#include <stddef.h>
#include <stdint.h>
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define B2_ABI_VERSION 4

/* ---- status codes (tidb_query_common::error::Error classes, dag/mod.rs:231-244) ---- */
enum {
  B2_OK = 0,
  B2_ERR_STORAGE = 1,        /* Error::Storage: bad write record, default CF miss, ... */
  B2_ERR_KEY_IS_LOCKED = 2,  /* txn_types::ErrorInner::KeyIsLocked (lock.rs:457-476) */
  B2_ERR_WRITE_CONFLICT = 3, /* RcCheckTs newer version (forward.rs:342-354) */
  B2_ERR_EVALUATE = 4,       /* Error::Evaluate{code,msg}; code in b2_error_info.mysql_code */
  B2_ERR_CORRUPTED = 5,      /* row / datum decode failure (other_err! in table_scan_executor.rs) */
  B2_ERR_DEADLINE = 6,
  B2_ERR_UNSUPPORTED = 7,    /* plan not supported on the device path: host falls back */
  B2_ERR_CUDA = 8,
  B2_ERR_INVALID_ARG = 9,
  B2_PENDING = 100           /* b2_exec_poll: the batch started by b2_exec_next_batch_async is not ready yet */
};

/* MySQL error codes preserved across the boundary */
#define B2_MYSQL_ERR_DATA_OUT_OF_RANGE 1690
#define B2_MYSQL_ERR_TRUNCATED 1292
#define B2_MYSQL_ERR_DIVISION_BY_ZERO 1365

/* ---- field types (tidb_query_datatype/src/def/field_type.rs; MySQL protocol codes) ---- */
enum {
  B2_TP_TINY = 1, B2_TP_SHORT = 2, B2_TP_LONG = 3, B2_TP_FLOAT = 4, B2_TP_DOUBLE = 5,
  B2_TP_NULL = 6, B2_TP_TIMESTAMP = 7, B2_TP_LONGLONG = 8, B2_TP_INT24 = 9, B2_TP_DATE = 10,
  B2_TP_DURATION = 11, B2_TP_DATETIME = 12, B2_TP_YEAR = 13, B2_TP_VARCHAR = 15, B2_TP_BIT = 16,
  B2_TP_JSON = 0xf5, B2_TP_NEWDECIMAL = 0xf6, B2_TP_ENUM = 0xf7, B2_TP_SET = 0xf8,
  B2_TP_BLOB = 0xfc, B2_TP_VARSTRING = 0xfd, B2_TP_STRING = 0xfe
};
#define B2_FLAG_NOT_NULL 1u
#define B2_FLAG_UNSIGNED 32u

/* extra column ids (codec/table.rs:49-57) */
#define B2_EXTRA_PHYSICAL_TABLE_ID_COL_ID (-3)
#define B2_EXTRA_COMMIT_TS_COL_ID (-5)

/* ---- data source: sorted column-family blocks ---------------------------------------
 * One block = n KV entries in ascending key order (RocksDB iteration order, data prefix
 * 'z' already stripped as RegionSnapshot does).  Entry i: key  = keys[key_offs[i]..key_offs[i+1])
 *                                                        value= vals[val_offs[i]..val_offs[i+1])
 * Heaps must be 16-byte aligned and readable for at least 16 bytes past offs[n] (the loader
 * moves whole 16-byte lines and the parsers read 8-byte words that may start on the last
 * bytes of the last entry; host-resident blocks are padded by the engine when it stages them,
 * B2_LOC_DEVICE callers pad their own buffers).  All versions of one user key live in the
 * same block.  `location` says where the pointers live.                                    */
enum { B2_LOC_HOST = 0, B2_LOC_DEVICE = 1 };

typedef struct b2_cf_block {
  const uint8_t* keys;
  const uint32_t* key_offs; /* n+1 entries */
  const uint8_t* vals;
  const uint32_t* val_offs; /* n+1 entries */
  uint32_t n;
  uint32_t _pad;
} b2_cf_block;

/* kvrpcpb::IsolationLevel */
enum { B2_ISO_SI = 0, B2_ISO_RC = 1, B2_ISO_RC_CHECK_TS = 2 };

/* B2_LOC_DEVICE blocks must be complete when the request opens (b2_exec_open, b2_dag_handle, b2_checksum_handle): the
 * engine reads them on its own stream (b2_exec_config.cuda_stream or a non-blocking stream it creates) and does not
 * order itself behind other streams, the legacy default stream included.  A producer that writes the blocks
 * asynchronously synchronises (or makes cuda_stream wait on its work) before the call.  b2_gen_create, b2_sst_decode and
 * b2_region_pin return with their blocks complete. */
typedef struct b2_region_source {
  int32_t location;              /* of write/default blocks; lock block is always host memory */
  int32_t device;                /* CUDA ordinal for B2_LOC_DEVICE pointers / where to run */
  const b2_cf_block* write;      /* CF_WRITE blocks, globally ordered */
  uint32_t n_write;
  const b2_cf_block* dflt;       /* CF_DEFAULT blocks (long values), may be NULL */
  uint32_t n_dflt;
  const b2_cf_block* lock;       /* CF_LOCK, host memory, may be NULL (or RC isolation) */
  uint64_t read_ts;              /* ScannerConfig::ts */
  int32_t isolation_level;
  int32_t check_has_newer_ts_data;
  const uint64_t* bypass_locks;  /* TsSet */
  uint32_t n_bypass_locks;
  const uint64_t* access_locks;  /* non-empty => B2_ERR_UNSUPPORTED when one is hit */
  uint32_t n_access_locks;
} b2_region_source;

/* raw (not memcomparable-encoded) key range, like coppb::KeyRange */
typedef struct b2_key_range {
  const uint8_t* start; uint32_t start_len;
  const uint8_t* end;   uint32_t end_len;
} b2_key_range;

/* ---- plan descriptor ------------------------------------------------------------------ */
/* tipb::ColumnInfo as used by BatchTableScanExecutor::new (table_scan_executor.rs:56-150) */
typedef struct b2_column_info {
  int64_t col_id;
  int32_t tp;                /* B2_TP_* */
  uint32_t flag;             /* B2_FLAG_* */
  int32_t pk_handle;         /* int handle stored in the key */
  uint32_t default_len;
  const uint8_t* default_val;/* datum-encoded default, NULL/0 = none */
  int32_t decimal;           /* tipb ColumnInfo.decimal: the fsp of DATE / DATETIME / TIMESTAMP columns */
  int32_t _pad;
} b2_column_info;

/* RPN node kinds (tidb_query_expr/src/types/expr.rs:11-30) */
enum { B2_RPN_CONST_NULL = 0, B2_RPN_CONST_INT = 1, B2_RPN_CONST_UINT = 2, B2_RPN_CONST_REAL = 3,
       B2_RPN_COLUMN_REF = 4, B2_RPN_FN = 5,
       B2_RPN_CONST_TIME = 6,      /* i64 = Time::to_packed_u64 (the payload of tipb ExprType::MysqlTime); field_tp DATE / DATETIME */
       B2_RPN_CONST_DURATION = 7,  /* i64 = nanoseconds (tipb ExprType::MysqlDuration) */
       B2_RPN_CONST_DECIMAL = 9,   /* tipb ExprType::MysqlDecimal: i64 = address of its payload (precision byte, fraction byte,
                                      binary decimal: what a stored DECIMAL cell holds), n_args = the payload's length */
       B2_RPN_CONST_BYTES = 8      /* tipb ExprType::Bytes / String: i64 = address of the bytes (host memory, borrowed for the
                                      handle's lifetime like the plan itself), n_args = their length (< 65536) */ };

/* Scalar function signatures.  Names follow tipb::ScalarFuncSig; numeric values follow
 * tipb expression.proto as pinned by Cargo.lock (pingcap/tipb @ 1374320b, not vendored in
 * the reference tree) and are re-exported by name in INTEGRATION.md's binding.            */
enum {
  B2_SIG_LT_INT = 100, B2_SIG_LT_REAL = 101,
  B2_SIG_LE_INT = 110, B2_SIG_LE_REAL = 111,
  B2_SIG_GT_INT = 120, B2_SIG_GT_REAL = 121,
  B2_SIG_GE_INT = 130, B2_SIG_GE_REAL = 131,
  B2_SIG_EQ_INT = 140, B2_SIG_EQ_REAL = 141,
  B2_SIG_NE_INT = 150, B2_SIG_NE_REAL = 151,
  B2_SIG_NULLEQ_INT = 160, B2_SIG_NULLEQ_REAL = 161,
  B2_SIG_PLUS_REAL = 200, B2_SIG_PLUS_INT = 203,
  B2_SIG_MINUS_REAL = 204, B2_SIG_MINUS_INT = 207,
  B2_SIG_MULTIPLY_REAL = 208, B2_SIG_MULTIPLY_INT = 210,
  B2_SIG_MULTIPLY_INT_UNSIGNED = 218,
  B2_SIG_LOGICAL_AND = 3101, B2_SIG_LOGICAL_OR = 3102, B2_SIG_LOGICAL_XOR = 3103,
  B2_SIG_UNARY_NOT_INT = 3104, B2_SIG_UNARY_NOT_REAL = 3106,
  B2_SIG_REAL_IS_NULL = 3113, B2_SIG_INT_IS_NULL = 3116,
  B2_SIG_INT_IS_TRUE = 3122, B2_SIG_REAL_IS_TRUE = 3123,
  B2_SIG_INT_IS_FALSE = 3125, B2_SIG_REAL_IS_FALSE = 3126,
  B2_SIG_IN_INT = 4001, B2_SIG_IN_REAL = 4002, /* variadic: n_args = 1 + list length (impl_compare_in.rs) */
  /* impl_arithmetic.rs:215-290, 396-455 (signedness variants are picked from the arguments' UNSIGNED flags, like map_int_sig) */
  B2_SIG_INT_DIVIDE_INT = 213, B2_SIG_MOD_REAL = 215, B2_SIG_MOD_INT = 217,
  B2_SIG_DIVIDE_REAL = 211, /* impl_arithmetic.rs:515-533: x / 0 is NULL + warning 1365 "Division by 0" (expr/ctx.rs:267-286) */
  B2_SIG_ABS_INT = 2101, B2_SIG_ABS_UINT = 2102, B2_SIG_ABS_REAL = 2103,           /* impl_math.rs:224-243 */
  B2_SIG_UNARY_MINUS_INT = 3108, B2_SIG_UNARY_MINUS_REAL = 3109,                    /* impl_op.rs:70-107 */
  B2_SIG_IF_NULL_INT = 4101, B2_SIG_IF_NULL_REAL = 4102, B2_SIG_IF_INT = 4107, B2_SIG_IF_REAL = 4108, /* impl_control.rs */
  B2_SIG_COALESCE_INT = 4201, B2_SIG_COALESCE_REAL = 4202,                          /* impl_compare.rs:239-248, variadic */
  B2_SIG_CASE_WHEN_INT = 4208, B2_SIG_CASE_WHEN_REAL = 4209,                        /* impl_control.rs:34-50, variadic: [cond, value]* [else] */
  /* comparisons over DATE / DATETIME and DURATION values (impl_compare.rs:63-240 with `Ord for Time`,
   * mysql/time/mod.rs:2814-2840: the fsp / time-type bits do not take part; `Ord for Duration`: nanoseconds) */
  B2_SIG_LT_TIME = 104, B2_SIG_LT_DURATION = 105, B2_SIG_LE_TIME = 114, B2_SIG_LE_DURATION = 115,
  B2_SIG_GT_TIME = 124, B2_SIG_GT_DURATION = 125, B2_SIG_GE_TIME = 134, B2_SIG_GE_DURATION = 135,
  B2_SIG_EQ_TIME = 144, B2_SIG_EQ_DURATION = 145, B2_SIG_NE_TIME = 154, B2_SIG_NE_DURATION = 155,
  B2_SIG_NULLEQ_TIME = 164, B2_SIG_NULLEQ_DURATION = 165,
  B2_SIG_TIME_IS_NULL = 3115, B2_SIG_DURATION_IS_NULL = 3112,
  B2_SIG_IN_TIME = 4005, B2_SIG_IN_DURATION = 4006,
  /* comparisons over DECIMAL values (`Ord for Decimal`, decimal.rs:2323-2338: by value, the signs first) */
  B2_SIG_LT_DECIMAL = 102, B2_SIG_LE_DECIMAL = 112, B2_SIG_GT_DECIMAL = 122, B2_SIG_GE_DECIMAL = 132, B2_SIG_EQ_DECIMAL = 142,
  B2_SIG_NE_DECIMAL = 152, B2_SIG_NULLEQ_DECIMAL = 162, B2_SIG_DECIMAL_IS_NULL = 3111, B2_SIG_IN_DECIMAL = 4003,
  /* impl_op.rs:144-175 */
  B2_SIG_BIT_AND = 3118, B2_SIG_BIT_OR = 3119, B2_SIG_BIT_XOR = 3120, B2_SIG_BIT_NEG = 3121,
  /* impl_cast.rs:281-305 (Int -> Int keeps the bits), :466-501 (Int -> Real by the signedness of either side),
   * :505-507 (Real -> Real); UNION's in_union metadata is not carried by this ABI (treated as false) */
  B2_SIG_CAST_INT_AS_INT = 0, B2_SIG_CAST_INT_AS_REAL = 1, B2_SIG_CAST_REAL_AS_REAL = 11,
  /* impl_like.rs:7-74: LIKE(target bytes, pattern bytes, escape int) over a bytes column / constant.  The collator is the
   * node's own collation, the charset the target's when target and pattern agree, else the node's (lib.rs:99-135
   * map_like_sig).  On the device path: the binary collation and the *_bin collations of utf8 / utf8mb4 (their
   * force-no-pad comparison of one character is byte equality); `_` then steps one byte or one UTF-8 character. */
  B2_SIG_LIKE = 4310
};

typedef struct b2_rpn_node {
  int32_t kind;       /* B2_RPN_* */
  int32_t sig;        /* B2_SIG_* when kind == FN */
  int32_t n_args;     /* FN arity */
  int32_t field_tp;   /* return field type B2_TP_* */
  uint32_t field_flag;/* return field flags (UNSIGNED matters for compare dispatch, lib.rs:223-259) */
  int32_t collation;  /* tipb FieldType.collate of the node's type as TiDB sends it (Collation::from_i32, field_type.rs:130-146:
                         63 / -63 binary, -46 / -83 / -65 utf8mb4_bin, >= 0 otherwise: utf8mb4_bin without padding ...); only LIKE reads it */
  int64_t i64;        /* CONST_INT/UINT payload, or COLUMN_REF offset into the child schema */
  double f64;         /* CONST_REAL payload */
} b2_rpn_node;

typedef struct b2_rpn_expr {
  const b2_rpn_node* nodes; /* post-order */
  uint32_t n_nodes;
  uint32_t _pad;
} b2_rpn_expr;

/* tipb::ExprType aggregate kinds (tidb_query_aggr/src/parser.rs:67-88) */
enum { B2_AGG_COUNT = 3001, B2_AGG_SUM = 3002, B2_AGG_AVG = 3003, B2_AGG_MIN = 3004,
       B2_AGG_MAX = 3005, B2_AGG_FIRST = 3006,
       /* Agg_BitAnd / Agg_BitOr / Agg_BitXor over an Int argument (a Real argument is B2_ERR_UNSUPPORTED: no Real->Int
        * cast here).  The output column is B2_COL_I64, B2_TP_LONGLONG, UNSIGNED | NOT_NULL, the type TiDB infers for them
        * (b2_aggr_desc carries no output field type).  FIRST outputs one column of its argument's type, NOT_NULL cleared. */
       B2_AGG_BIT_AND = 3008, B2_AGG_BIT_OR = 3009, B2_AGG_BIT_XOR = 3010 };

typedef struct b2_aggr_desc {
  int32_t kind;      /* B2_AGG_* */
  int32_t _pad;
  b2_rpn_expr arg;   /* argument expression (COUNT(1) = one CONST_INT node) */
} b2_aggr_desc;

typedef struct b2_order_by {
  b2_rpn_expr expr;
  int32_t desc;
  int32_t _pad;
} b2_order_by;

/* tipb::ExecType */
enum { B2_EXEC_TABLE_SCAN = 0, B2_EXEC_INDEX_SCAN = 1, B2_EXEC_SELECTION = 2,
       B2_EXEC_AGGREGATION = 3 /* hash */, B2_EXEC_TOPN = 4, B2_EXEC_LIMIT = 5,
       B2_EXEC_STREAM_AGG = 6,
       B2_EXEC_PROJECTION = 7 /* projection_executor.rs: its expressions travel in `conditions` / `n_conditions` */ };

typedef struct b2_executor_desc {
  int32_t tp; /* B2_EXEC_* */
  int32_t desc;                       /* TableScan.desc */
  int64_t table_id;                   /* TableScan */
  const b2_column_info* columns;      /* TableScan */
  uint32_t n_columns;
  uint32_t n_conditions;
  const b2_rpn_expr* conditions;      /* Selection: AND of conditions */
  const b2_rpn_expr* group_by;        /* Aggregation */
  uint32_t n_group_by;
  uint32_t n_aggrs;
  const b2_aggr_desc* aggrs;          /* Aggregation */
  const b2_order_by* order_by;        /* TopN */
  uint32_t n_order_by;
  uint32_t _pad;
  uint64_t limit;                     /* TopN (at most 4096 on the device path) / Limit */
} b2_executor_desc;

typedef struct b2_dag_plan {
  const b2_executor_desc* executors;  /* executors[0] is the scan, like DagRequest.executors */
  uint32_t n_executors;
  uint32_t n_output_offsets;
  const uint32_t* output_offsets;     /* NULL = all columns */
  uint64_t flags;                     /* DagRequest.flags (expr/ctx.rs:24-52) */
} b2_dag_plan;

typedef struct b2_exec_config {
  int32_t output_location;  /* B2_LOC_HOST: results copied to host memory; B2_LOC_DEVICE: device ptrs */
  int32_t staging_tiles;    /* 0 = default */
  uint64_t cuda_stream;     /* 0 = handle creates its own stream; else a cudaStream_t to run on (device-resident blocks
                             * must be complete when the request opens: see b2_region_source) */
  int32_t jit;              /* plan-specialised kernel (compiled at run time, cached per plan): B2_JIT_AUTO = background
                             * compile for large requests and switch when ready, B2_JIT_SYNC = wait for it at open,
                             * B2_JIT_OFF = always the generic kernel.  Environment B2_JIT=auto|sync|off overrides.
                             * Plans that use DIV / MOD / unary minus / ABS / IFNULL / IF / CASE WHEN / COALESCE always
                             * behave as B2_JIT_SYNC: those functions are only compiled into specialised kernels. */
  int32_t _pad;
  uint64_t deadline_ns;     /* CLOCK_MONOTONIC nanoseconds; once passed, calls answer B2_ERR_DEADLINE before (and between) launches:
                             * Deadline::check at the top of every batch, runner.rs:974; tikv_util deadline.rs.  0 = none */
  uint64_t paging_size;     /* b2_dag_handle only: a paging request (runner.rs:790-806) stops after the batch in which this many rows
                             * have been produced and answers B2_DRAIN_PAGING; b2_exec_take_scanned_range then gives the range to
                             * resume from.  0 = not a paging request */
  uint64_t reserved[1];
} b2_exec_config;
enum { B2_JIT_AUTO = 0, B2_JIT_SYNC = 1, B2_JIT_OFF = 2 };

/* ---- results ------------------------------------------------------------------------------ */
enum { B2_COL_I64 = 0, B2_COL_F64 = 1, B2_COL_DECIMAL = 2,
       B2_COL_BYTES = 3,    /* VARCHAR / BLOB ...: `offsets` + byte heap (ChunkedVecBytes, chunked_vec_bytes.rs:9-15)      */
       B2_COL_TIME = 4,     /* DATE / DATETIME / TIMESTAMP: u64 CoreTime bit field (mysql/time/mod.rs:167-196)           */
       B2_COL_DURATION = 5, /* i64 nanoseconds (mysql/duration.rs)                                                      */
       B2_COL_JSON = 6 };   /* binary JSON [type code][value] per cell, `offsets` + byte heap (chunked_vec_json.rs)      */

/* #[repr(C)] Decimal, codec/mysql/decimal.rs:927-942 (raw 40 bytes as write_decimal_to_chunk dumps) */
typedef struct b2_decimal {
  uint8_t int_cnt, frac_cnt, result_frac_cnt, negative;
  uint32_t word_buf[9];
} b2_decimal;

/* one decoded column: ChunkedVecSized<T>{data, bitmap} (chunked_vec_sized.rs:17-22) */
typedef struct b2_column {
  int32_t kind;               /* B2_COL_* */
  int32_t field_tp;
  uint32_t field_flag;
  uint32_t _pad;
  uint64_t len;
  const void* data;           /* len elements of i64 / f64 / u64 / b2_decimal (NULL cells hold 0); BYTES / JSON: the byte heap */
  const uint64_t* null_bitmap;/* bit i (word i>>6, bit i&63) = 1 => non-null (bit_vec.rs:25-38) */
  const int64_t* offsets;     /* BYTES / JSON only: len + 1 offsets into `data`, cell i = data[offsets[i] .. offsets[i+1])
                                 (the layout of a var-length chunk column, chunk/column.rs:1052-1072); NULL otherwise */
} b2_column;

enum { B2_DRAIN_REMAIN = 0, B2_DRAIN_DRAINED = 1, B2_DRAIN_PAGING = 2 };

/* BatchExecuteResult: logical_rows is the identity here (columns come back compacted) */
typedef struct b2_batch {
  const b2_column* columns;
  uint32_t n_columns;
  int32_t is_drained;         /* B2_DRAIN_* */
  uint64_t n_rows;
  uint32_t n_warnings;
  uint32_t _pad;
} b2_batch;

/* ExecSummary (execute_stats.rs:8-16) + the scan counters callers read back (stats.rs:95-114) */
typedef struct b2_exec_stats {
  uint64_t num_iterations;
  uint64_t num_produced_rows;
  uint64_t time_processed_ns;   /* device time from CUDA events */
  uint64_t write_entries_scanned; /* CF_WRITE entries visited (all versions) */
  uint64_t write_processed_keys;  /* rows returned by the MVCC scan */
  uint64_t processed_size;        /* sum(len(user_key)+len(value)) over returned rows, forward.rs:517-519 */
  uint64_t default_lookups;       /* CF_DEFAULT fetches */
  uint64_t lock_processed_keys;
  int32_t met_newer_ts_data;      /* -1 unknown, 0 not met, 1 met (NewerTsCheckState) */
  int32_t _pad;
  uint64_t kernel_time_ns;        /* CUDA-event time spent inside the dominant (scan) kernel launches */
  uint64_t kernel_launches;       /* launches of this library's kernels */
  uint64_t h2d_bytes;             /* bytes staged host->device by the engine (host-resident sources) */
  uint64_t d2h_bytes;             /* result bytes copied device->host */
  uint64_t jit_launches;          /* of kernel_launches: launches of the plan-specialised (run-time compiled) scan kernel */
} b2_exec_stats;

typedef struct b2_error_info {
  int32_t status;
  int32_t mysql_code;
  uint64_t entry_index;  /* global CF_WRITE entry index of the failing row, or ~0 */
  char message[232];
} b2_error_info;

typedef struct b2_exec b2_exec; /* opaque */

/* version / build info, following the coprocessor_plugin_api precedent
 * (components/coprocessor_plugin_api/src/util.rs:7-33) */
uint32_t b2_abi_version(void);
const char* b2_build_info(void);

/* thread-local message of the last failing call on this thread */
const char* b2_last_error_message(void);

/* runner.rs:111-206 — B2_OK or B2_ERR_UNSUPPORTED (message says why) */
int32_t b2_check_supported(const b2_dag_plan* plan);
/* Prepared plan: compile the plan-specialised scan kernel for `device` now (blocking; cached for the process).  Later
 * requests carrying the same plan start on it.  B2_ERR_UNSUPPORTED: run-time compilation (NVRTC) is not available, the
 * generic kernels serve the plan. */
int32_t b2_plan_prepare(const b2_dag_plan* plan, int32_t device);
/* The same ahead of time and without a GPU: NVRTC compiles the kernel(s) of the plan *shape* into the on-disk cache
 * (B2_JIT_CACHE_DIR, default <library dir>/jit_cache; keyed by plan shape + kernel sources).  Constants, IN lists, LIMIT,
 * read_ts and the isolation level are launch parameters, not part of the shape: `col < 5` and `col < 7` share one kernel.
 * *n_compiled (may be NULL): kernels compiled by this call (0 = all cached already). */
int32_t b2_plan_precompile(const b2_dag_plan* plan, int32_t* n_compiled);
/* process-wide counters: NVRTC compilations run so far, kernels loaded from the on-disk cache */
void b2_jit_counters(uint64_t* nvrtc_compiles, uint64_t* disk_cache_hits);

/* interface.rs:36-97 */
int32_t b2_exec_open(const b2_dag_plan* plan, const b2_key_range* ranges, uint32_t n_ranges,
                     const b2_region_source* src, const b2_exec_config* cfg, b2_exec** out);
/* schema(): field types of the outermost executor's output columns */
int32_t b2_exec_schema(b2_exec* h, int32_t* field_tps, uint32_t* field_flags, uint32_t* n_inout);
/* next_batch(scan_rows).  On error the batch still describes the rows produced before it
 * (interface.rs:229-235) and b2_exec_last_error gives details. */
int32_t b2_exec_next_batch(b2_exec* h, uint64_t scan_rows, b2_batch* out);
int32_t b2_exec_collect_stats(b2_exec* h, b2_exec_stats* out);
/* next_batch without blocking the caller (the reference's `async fn next_batch` on a yatp thread, interface.rs:53): _async
 * starts the batch on the handle's worker and returns at once; b2_exec_poll answers B2_PENDING until it has finished, then
 * the batch's own status with *out filled (exactly what b2_exec_next_batch would have returned).  One batch in flight per
 * handle; no other call on the handle in between except poll. */
int32_t b2_exec_next_batch_async(b2_exec* h, uint64_t scan_rows);
int32_t b2_exec_poll(b2_exec* h, b2_batch* out);
/* EvalWarnings of the request so far (BatchExecuteResult::warnings, interface.rs:205-236; expr/ctx.rs:180-215): *count_out =
 * warning_cnt (every warning raised), of which at most min(cap, 64) are written (max_warning_cnt). */
typedef struct b2_warning {
  int32_t mysql_code;
  int32_t _pad;
  char message[120];
} b2_warning;
int32_t b2_exec_warnings(b2_exec* h, b2_warning* out, uint32_t cap, uint64_t* count_out);
int32_t b2_exec_last_error(b2_exec* h, b2_error_info* out);
/* Response encoding of the batch most recently returned by b2_exec_next_batch / b2_dag_handle on this handle:
 * encode_result_to_chunk (components/tidb_query_executors/src/runner.rs:1051-1088), i.e. tipb::Chunk.rows_data in
 * EncodeType::TypeDefault (datum rows, lazy_column_vec.rs:172-187 + vector.rs:362-470) or EncodeType::TypeChunk
 * (one column block per output column, chunk/column.rs:1052-1072).  Runs on the device from the HBM-resident columns;
 * only the encoded bytes cross PCIe when `location` is B2_LOC_HOST.  The buffer is valid until the next call on the
 * handle.  TypeDefault writes every cell in the canonical fixed-width datum form the reference uses for decoded
 * columns and for all v2 rows (v1 rows' never-evaluated columns keep their stored VAR_INT form in the reference). */
enum { B2_ENCODE_TYPE_DEFAULT = 0, B2_ENCODE_TYPE_CHUNK = 1 };
typedef struct b2_encoded_chunk {
  const uint8_t* rows_data;
  uint64_t len;
  uint64_t n_rows;
  int32_t encode_type;
  int32_t location;
} b2_encoded_chunk;
int32_t b2_exec_encode_batch(b2_exec* h, int32_t encode_type, int32_t location, b2_encoded_chunk* out);
/* BatchExecutor::take_scanned_range (interface.rs:70-75) -> RangesScanner::take_scanned_range
 * (tidb_query_common/src/storage/scanner.rs:204-229), forward scans: the raw-key interval [lower, upper) covered since
 * the previous call.  upper = key of the last row the MVCC scan returned + 0x00, or the end of the last range once the
 * executor is drained.  The pointers stay valid until the next call on the handle. */
int32_t b2_exec_take_scanned_range(b2_exec* h, const uint8_t** lower, uint32_t* lower_len, const uint8_t** upper, uint32_t* upper_len);
/* RangesScanner::collect_scanned_rows_per_range (scanner.rs:196-201): rows returned by the MVCC scan inside each input
 * range since the previous call.  *n_inout: capacity of `rows` in, number of ranges out. */
int32_t b2_exec_collect_scanned_rows_per_range(b2_exec* h, uint64_t* rows, uint32_t* n_inout);
/* storage_impl.rs:108-123: no newer-ts data and no lock seen */
int32_t b2_exec_can_be_cached(b2_exec* h);
void b2_exec_close(b2_exec* h);

/* Partial aggregation state of an Aggregation pipeline, for the multi-GPU / multi-region final merge (what TiDB's
 * final HashAgg does with the per-region partial results; fast_hash_aggr_executor.rs emits partial results only).
 * Valid after the drained batch was produced.  Per group `acc_words` additive u64 words, per aggregate in plan order:
 *   COUNT: [count]   SUM/AVG over Int: [count, sum of low 32 bits, sum of high 32 bits]
 *   SUM/AVG over Real: [count, 66 words]: the exact sum as a 2112-bit fixed-point number (bit 0 = 2^-1074), one signed
 *   32-bit digit per word, carry-save; partial sums merge by word-wise integer addition and round once at the end
 *   MAX/MIN: [count, extremum key]: the key merges by unsigned 64-bit maximum (bit w of max_word_mask marks such words)
 *   BIT_OR: [bits], merges by OR   BIT_XOR: [bits], merges by XOR   BIT_AND: [OR of the complemented inputs], merges by
 *   OR; the result is ~bits
 *   FIRST: [key, value] at an even word (padding words before it are additive zeros): the pair with the larger key wins;
 *   key 0 = no row, bit 0 of the key = the value is NULL.  Keys order the rows of one request only: a merge across
 *   requests takes the first request, in scan order, whose key is nonzero
 * b2_exec_agg_word_ops tells how each word merges. */
typedef struct b2_agg_partials {
  uint32_t n_groups;
  uint32_t acc_words;
  int32_t location;           /* always B2_LOC_DEVICE */
  int32_t has_group;
  const uint64_t* keys;       /* n_groups * key_words group keys (bits, 0 where NULL); unused without GROUP BY */
  const uint8_t* key_null;    /* n_groups NULL masks: bit q set = the q-th group-by value is NULL */
  const uint64_t* acc;        /* n_groups * acc_words */
  uint64_t max_word_mask;     /* words of a group's state that merge by unsigned maximum instead of addition */
  uint32_t key_words;         /* group-by expressions (1 for the fast hash executor, 2..4 for BatchSlowHashAggregation) */
  uint32_t _pad;
} b2_agg_partials;
int32_t b2_exec_agg_partials(b2_exec* h, b2_agg_partials* out);
/* How each word of b2_agg_partials.acc merges: ops[w] = B2_MERGE_*, w < acc_words.  Valid whenever b2_exec_agg_partials
 * is.  *n_inout: capacity of `ops` in, acc_words out (B2_ERR_INVALID_ARG when the capacity is smaller). */
enum { B2_MERGE_ADD = 0, B2_MERGE_MAX = 1, B2_MERGE_OR = 2, B2_MERGE_XOR = 3, B2_MERGE_FIRST_KEY = 4, B2_MERGE_FIRST_VALUE = 5 };
int32_t b2_exec_agg_word_ops(b2_exec* h, uint8_t* ops, uint32_t* n_inout);
/* Final merge of partial tables gathered from several requests / GPUs, on the device.  n_rows rows (< 2^31), on
 * `device`: row r has key_words (1..4) key words keys[r * keys_stride + k], the NULL mask key_null[r] (bit q = q-th key
 * is NULL, below 2^key_words) and acc_words state words acc[r * acc_stride + w] (strides in words).  The rows of part p
 * are [part_offs[p], part_offs[p + 1]) (host array, n_parts + 1 offsets from 0 to n_rows).  A group is a distinct
 * (NULL mask, key words); with one key word a NULL row's key bits do not count.  Groups come out sorted ascending by the
 * NULL mask, then by the key words as signed int64; each state word merges by ops[w] (B2_MERGE_*: ADD wraps modulo
 * 2^64, MAX is unsigned; a FIRST pair comes from the earliest part holding a nonzero key, the latest when `desc`, and
 * inside that part from the largest unsigned key, the last such row on ties).  out_keys (n_rows * key_words; 0 for a
 * NULL single key), out_null (n_rows) and out_acc (n_rows * acc_words) are device buffers with room for n_rows groups;
 * *n_groups receives the number written.  Runs on `cuda_stream` (0 = legacy default stream) and returns when the result
 * is there. */
int32_t b2_agg_merge(int32_t device, uint64_t cuda_stream, uint64_t n_rows, uint32_t key_words, uint32_t acc_words,
                     const int64_t* keys, uint64_t keys_stride, const uint8_t* key_null, const int64_t* acc, uint64_t acc_stride,
                     const uint64_t* part_offs, uint32_t n_parts, const uint8_t* ops, int32_t desc,
                     int64_t* out_keys, uint8_t* out_null, int64_t* out_acc, uint64_t* n_groups);

/* RequestHandler::handle_request for a DAG: run to drain.  Result columns are owned by *out_handle
 * (close it with b2_exec_close). */
int32_t b2_dag_handle(const b2_dag_plan* plan, const b2_key_range* ranges, uint32_t n_ranges,
                      const b2_region_source* src, const b2_exec_config* cfg,
                      b2_batch* out, b2_exec** out_handle);

/* tipb::ChecksumResponse */
typedef struct b2_checksum_response {
  uint64_t checksum;
  uint64_t total_kvs;
  uint64_t total_bytes;
} b2_checksum_response;

/* checksum.rs:59-98 with ChecksumRewriteRule{old_prefix,new_prefix} */
int32_t b2_checksum_handle(const b2_key_range* ranges, uint32_t n_ranges,
                           const uint8_t* old_prefix, uint32_t old_prefix_len,
                           const uint8_t* new_prefix, uint32_t new_prefix_len,
                           const b2_region_source* src, const b2_exec_config* cfg,
                           b2_checksum_response* out, b2_exec_stats* stats);

/* ---- HBM-resident block cache ---------------------------------------------------------------------------------------
 * TiKV serves repeated reads of a region from its block cache; here the cached copy lives in device memory, so a warm
 * request runs at HBM speed instead of PCIe speed.  b2_region_pin copies the CF blocks of `host_src` (B2_LOC_HOST) to the
 * device once, keyed by (device, region_id, data_version), and fills *dev_src with a B2_LOC_DEVICE source over the cached
 * copy (same read_ts / isolation fields; valid until the matching b2_region_unpin).  Pinning the same key again returns
 * the existing copy.  B2_ERR_UNSUPPORTED when the cache budget (B2_BLOCK_CACHE_BYTES, default 3/4 of the device memory) is full. */
int32_t b2_region_pin(int32_t device, uint64_t region_id, uint64_t data_version, const b2_region_source* host_src, b2_region_source* dev_src);
int32_t b2_region_unpin(int32_t device, uint64_t region_id, uint64_t data_version);
void b2_region_cache_stats(int32_t device, uint64_t* bytes_cached, uint64_t* hits, uint64_t* misses);

/* ---- RocksDB data blocks as the data source (SURVEY.md §8(f)4: the on-disk block reader) -----------------------------
 * BlockBasedTable data blocks keep their keys prefix-compressed between restart points (RocksDB is an external
 * dependency of the reference; block size and format version come from src/config/mod.rs:966 and :704).  TiKV's block
 * cache holds them uncompressed; in the file, levels 2-4 of the write and default CFs store them LZ4-compressed
 * (src/config/mod.rs:981-988).  b2_sst_decode takes a run of such blocks, in key order, inflates the LZ4 ones and
 * expands all of them on the device into the flat b2_cf_block layout the scan kernels read: the bytes that cross PCIe are
 * the compressed ones.
 *
 *   data block  := entry* restart[u32 LE x num_restarts] num_restarts[u32 LE]   (+ 5-byte trailer: type, checksum)
 *   entry       := varint32 shared | varint32 non_shared | varint32 value_len | key[shared..] | value
 *   key         := key_prefix_len bytes (TiKV: 'z', components/keys/src/lib.rs:28) | CF key | key_suffix_len bytes
 *                  (RocksDB internal-key footer: fixed64 LE of seq << 8 | type)
 *
 * Supported: binary-search data blocks (no hash index: top bit of num_restarts clear), value type kTypeValue (1) in every
 * footer -- i.e. files that hold one RocksDB version of each key (bottommost level, ingested SSTs).  Anything else
 * answers B2_ERR_UNSUPPORTED and the host keeps its merging iterator.  Checksums of the trailer are not verified.
 *
 * Compression (trailer_len == 5 only: the trailer's first byte is RocksDB's compression type; with trailer_len == 0 the
 * contents are plain):
 *   0 kNoCompression        the contents are the data block
 *   4 kLZ4Compression,      the contents are  varint32 uncompressed_size | LZ4 block  (format_version >= 2 framing; the
 *   5 kLZ4HCCompression     raw LZ4 block format, no frame header): inflated on the device.  A declared size below 4,
 *                           above 255 x the LZ4 bytes or above 1 GiB, or a stream that does not produce exactly that many
 *                           bytes from exactly its bytes, is a corrupted block (B2_ERR_STORAGE)
 *   7 kZSTD,                the contents are  varint32 uncompressed_size | one ZSTD frame (RFC 8878): inflated on the
 *   0x40 kZSTDNotFinal...   device.  B2_ERR_UNSUPPORTED (the host's reader decides) when the payload does not start with
 *                           the frame magic 28 B5 2F FD (a skippable or legacy frame) or the frame names a Dictionary_ID.
 *                           B2_ERR_STORAGE: a declared size below 4 or above 1 GiB, a Frame_Content_Size other than it,
 *                           a size the frame's block headers cannot produce, anything after the frame, or a frame that
 *                           does not produce exactly that size (checksum, when present, included)
 *   1, 2, 3, 6,             Snappy, zlib, BZip2, Xpress and RocksDB's custom-compressor range: B2_ERR_UNSUPPORTED,
 *   0x80 .. 0xfe            a valid block the host's reader may inflate
 *   any other value         (8..0x3f, 0x41..0x7f, 0xff) no RocksDB writer stores it: a corrupted block (B2_ERR_STORAGE)
 * Plain, LZ4 and ZSTD blocks may mix in one run.  Blocks compressed with a dictionary (CompressionOptions::max_dict_bytes
 * > 0) carry no mark of it in an LZ4 block, nor in a ZSTD frame when the dictionary is raw content (no training: the
 * frame's Dictionary_ID is 0): the caller must not pass them (TiKV's default sets no dictionary). */
typedef struct b2_sst_blocks {
  const uint8_t* data;        /* the blocks, back to back or with gaps; host or device memory (see `location`) */
  const uint64_t* block_offs; /* host memory, n_blocks + 1 ascending offsets into data: block b = [block_offs[b], block_offs[b+1])
                                 (the BlockHandle list an index block yields) */
  uint32_t n_blocks;
  uint32_t trailer_len;       /* bytes at the end of every slice that are not block contents: 5 with the block trailer, else 0 */
  uint32_t key_prefix_len;    /* dropped from the front of every key (1 for TiKV data keys) */
  uint32_t key_suffix_len;    /* dropped from the end of every key: 8 = internal-key footer (checked), 0 = user keys only */
} b2_sst_blocks;

typedef struct b2_sst_stats {
  uint64_t n_entries, key_bytes, val_bytes; /* of the decoded block */
  uint64_t n_restart_intervals;
  uint64_t h2d_bytes;                       /* block bytes as passed (LZ4 blocks compressed) + offsets copied host -> device */
  float decode_ms;                          /* device time of the inflate and expansion kernels (CUDA events) */
  uint32_t n_lz4_blocks;                    /* LZ4 / LZ4HC blocks inflated by this call */
} b2_sst_stats;

typedef struct b2_sst b2_sst; /* owner of the decoded device block */
/* Decode `in` on `device`.  *h == NULL creates a handle, otherwise the handle's buffers are reused (they only grow).
 * On success *out holds B2_LOC_DEVICE pointers owned by the handle (valid until the next decode on it or b2_sst_free),
 * padded as b2_cf_block requires.  Blocking.  The decoded heaps must stay below 4 GiB each (u32 offsets). */
int32_t b2_sst_decode(int32_t device, int32_t location, const b2_sst_blocks* in, b2_sst** h, b2_cf_block* out, b2_sst_stats* stats);
void b2_sst_free(b2_sst* h);

/* ---- Sorted runs of one LSM snapshot merged on the device ---------------------------------------------------------
 * A region that still takes writes keeps its keys in L0 files and several levels, with point tombstones (TiKV's GC
 * deletes write and default records: MvccTxn::delete_write / delete_value in src/storage/mvcc/txn.rs), rewritten keys (a
 * commit record over a rollback at the same key) and ingested files (Raft snapshots applied by the raftstore's snapshot
 * io; imports, components/sst_importer/src/util.rs:213).  b2_sst_merge decodes each run as b2_sst_decode does, keeping the
 * internal-key footer, and outputs the flat block a RocksDB reader at sequence number `snapshot_seq` sees (DBIter over a
 * MergingIterator): one entry per user key whose newest visible entry is a value, keys ascending, key_prefix_len and
 * the footer dropped, padded as b2_cf_block requires and owned by the handle exactly like b2_sst_decode's output.
 *
 *   Order       user key bytewise ascending; within one user key the footer seq << 8 | type descending
 *               (InternalKeyComparator).  Each run ascends strictly in that order (checked: B2_ERR_STORAGE otherwise);
 *               a run may hold several versions of one key (a compaction under a held snapshot writes them).
 *   Runs        listed newest first (L0 files newest first, then L1 .. Ln).  That order is used only to break ties: an
 *               equal (user key, footer) pair in two runs goes to the run listed first.
 *   Visibility  an entry with seq > snapshot_seq is invisible.  The newest visible entry of a user key decides:
 *               kTypeValue (1) outputs the key; kTypeDeletion (0) and kTypeSingleDeletion (7) output nothing (DBIter
 *               treats them alike on reads).  Any other type anywhere in the input (Merge, BlobIndex, ...):
 *               B2_ERR_UNSUPPORTED, and the host keeps its iterator.
 *   Global seq  global_seqs[r] != 0 replaces the sequence number of every entry of run r (an ingested file); its stored
 *               sequence numbers must then be 0 (B2_ERR_STORAGE otherwise).  global_seqs == NULL: every run uses its footers.
 *   Arguments   (B2_ERR_INVALID_ARG) every run has key_suffix_len == 8 and the first run's key_prefix_len; trailer_len may
 *               differ per run (block-cache blocks have none, file blocks have one); snapshot_seq and global seqnos
 *               <= 2^56 - 1; n_runs <= 1024 (0 gives an empty block); each run bounded as in b2_sst_decode, and all
 *               runs together below 2^31 entries and 4 GiB per decoded heap (footers included).
 *   Stats       every input entry is counted once: n_in == n_invisible + n_out + n_deletions + n_hidden.
 *   Not handled range tombstones (the caller checks each file's num_range_deletions or keeps the host path), memtable
 *               contents and user-defined timestamps.
 * Blocking.  Device memory of the handle: the decoded runs back to back (decoded bytes + 8 per entry for the footer + 8 per
 * entry of offsets), two id arrays and three per-entry counters (16 bytes per entry), the largest run's decode buffers
 * and the output block. */
typedef struct b2_sst_merge_stats {
  uint64_t n_in;                 /* entries in all runs */
  uint64_t n_out;                /* entries written: user keys whose newest visible entry is kTypeValue */
  uint64_t n_invisible;          /* entries newer than the snapshot */
  uint64_t n_hidden;             /* visible entries under a newer visible entry of the same user key */
  uint64_t n_deletions;          /* user keys whose newest visible entry is a deletion */
  uint64_t key_bytes, val_bytes; /* of the output */
  uint64_t h2d_bytes;            /* as b2_sst_stats, summed over the runs */
  float decode_ms, merge_ms;     /* device time (CUDA events): inflate, expansion and staging of every run / ordering, visibility and gather */
  uint32_t n_lz4_blocks, n_runs;
} b2_sst_merge_stats;
int32_t b2_sst_merge(int32_t device, int32_t location, const b2_sst_blocks* runs, uint32_t n_runs,
                     const uint64_t* global_seqs /* NULL, or n_runs values: 0 = use the footers */, uint64_t snapshot_seq, b2_sst** h,
                     b2_cf_block* out, b2_sst_merge_stats* stats);

/* tooling (tests / bench): the inverse.  Encodes a device-resident flat block as data blocks of `entries_per_block`
 * entries with a restart point every `restart_interval` entries, key_prefix / internal-key footer (seq 0, kTypeValue)
 * added as asked, 5-byte trailer (type 0, checksum field zero) when trailer_len == 5.  The encoded bytes and the
 * n_blocks + 1 offsets stay on the device, owned by the handle; copy them out with b2_copy_to_host. */
typedef struct b2_sst_encoded {
  const uint8_t* data;        /* device */
  const uint64_t* block_offs; /* device, n_blocks + 1 */
  uint64_t data_len;
  uint32_t n_blocks;
  uint32_t _pad;
} b2_sst_encoded;
int32_t b2_sst_encode(int32_t device, const b2_cf_block* flat_device_block, uint32_t entries_per_block, uint32_t restart_interval,
                      uint32_t key_prefix_len, uint8_t key_prefix_byte, uint32_t key_suffix_len, uint32_t trailer_len,
                      b2_sst** h, b2_sst_encoded* out);

/* tooling: the compiled device plan of `plan` as a C++ aggregate initialiser (what the run-time compiler is fed);
 * returns its length, writes at most cap - 1 bytes + NUL into buf, negative status on error */
int64_t b2_plan_literal(const b2_dag_plan* plan, char* buf, uint64_t cap);

/* ---- synthetic region generator (tooling for tests/bench; SURVEY.md §8(d)) -----------------
 * Builds HBM-resident CF_WRITE blocks for a table with an int handle PK and `n_cols` i64
 * columns (ids 1..n_cols), row format v2 (or v1), one Put version per key plus optional
 * older/newer/Lock/Delete versions.  Values follow xorshift64* of (seed, handle, col).     */
typedef struct b2_gen_spec {
  int64_t table_id;
  uint64_t first_handle;
  uint64_t n_rows;
  uint32_t n_cols;
  int32_t row_format;        /* 1 or 2 */
  uint64_t seed;
  /* column c (0-based) value = mix(seed,handle,c) mapped into [col_lo[c], col_lo[c]+col_range[c])
   * (col_range 0 = full-range i64); null_per_million[c] rows are NULL */
  const int64_t* col_lo;
  const uint64_t* col_range;
  const uint32_t* null_per_million;
  uint32_t extra_versions_per_million; /* keys that get a newer-than-read_ts version + an older Put */
  uint32_t delete_per_million;         /* keys whose visible version is a Delete */
  uint32_t lock_rec_per_million;       /* keys with a Lock/Rollback record above the visible Put */
  uint64_t commit_ts;                  /* visible version commit ts (start_ts = commit_ts-1) */
  uint64_t newer_ts;                   /* commit ts for the newer-than-read versions */
} b2_gen_spec;

typedef struct b2_gen_block {
  b2_cf_block block;     /* device pointers owned by the generator handle */
  uint64_t key_bytes;
  uint64_t val_bytes;
  uint64_t n_user_keys;
} b2_gen_block;

typedef struct b2_gen b2_gen; /* opaque owner of generated device memory */
int32_t b2_gen_create(int32_t device, const b2_gen_spec* spec, b2_gen** out, b2_gen_block* out_block);
void b2_gen_destroy(b2_gen* g);

/* tooling: plain device<->host copies and pinned host memory so harnesses need no second CUDA binding */
int32_t b2_copy_to_host(int32_t device, void* dst, const void* src_device, uint64_t bytes);
int32_t b2_copy_to_device(int32_t device, void* dst_device, const void* src, uint64_t bytes);
int32_t b2_device_count(void);
void* b2_host_alloc_pinned(uint64_t bytes);
/* pinned host memory placed on the NUMA node `device` is attached to (falls back to b2_host_alloc_pinned) */
void* b2_host_alloc_pinned_near(int32_t device, uint64_t bytes);
int32_t b2_device_numa_node(int32_t device); /* -1 = unknown */
void b2_host_free_pinned(void* p);

#ifdef __cplusplus
}
#endif
#endif /* B2_COPR_H_ */
