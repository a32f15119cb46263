"""ctypes mirror of include/b2_copr.h and loader of the CUDA library.

The library is the product: if it is missing this module raises, it never falls back to a CPU path.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "libb2copr.so")

# ---- enums -------------------------------------------------------------------------------------
B2_OK, B2_ERR_STORAGE, B2_ERR_KEY_IS_LOCKED, B2_ERR_WRITE_CONFLICT, B2_ERR_EVALUATE = 0, 1, 2, 3, 4
B2_ERR_CORRUPTED, B2_ERR_DEADLINE, B2_ERR_UNSUPPORTED, B2_ERR_CUDA, B2_ERR_INVALID_ARG = 5, 6, 7, 8, 9
B2_PENDING = 100

TP_TINY, TP_SHORT, TP_LONG, TP_FLOAT, TP_DOUBLE, TP_NULL, TP_TIMESTAMP, TP_LONGLONG, TP_INT24 = 1, 2, 3, 4, 5, 6, 7, 8, 9
TP_DATE, TP_DURATION, TP_DATETIME, TP_YEAR, TP_VARCHAR, TP_BIT = 10, 11, 12, 13, 15, 16
TP_JSON, TP_NEWDECIMAL, TP_ENUM, TP_SET, TP_BLOB, TP_VARSTRING, TP_STRING = 0xF5, 0xF6, 0xF7, 0xF8, 0xFC, 0xFD, 0xFE
FLAG_NOT_NULL, FLAG_UNSIGNED = 1, 32
EXTRA_PHYSICAL_TABLE_ID_COL_ID, EXTRA_COMMIT_TS_COL_ID = -3, -5

LOC_HOST, LOC_DEVICE = 0, 1
ISO_SI, ISO_RC, ISO_RC_CHECK_TS = 0, 1, 2

RPN_CONST_NULL, RPN_CONST_INT, RPN_CONST_UINT, RPN_CONST_REAL, RPN_COLUMN_REF, RPN_FN, RPN_CONST_TIME, RPN_CONST_DURATION, RPN_CONST_BYTES, RPN_CONST_DECIMAL = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9

def _header_enum(prefix):
    """Enumerators of include/b2_copr.h with this prefix: the header is the single source of the numbers."""
    import re
    with open(os.path.join(os.path.dirname(_HERE), "include", "b2_copr.h")) as f:
        text = f.read()
    return {m.group(1): int(m.group(2), 0) for m in re.finditer(r"\b" + prefix + r"(\w+)\s*=\s*(0x[0-9a-fA-F]+|\d+)", text)}


SIG = _header_enum("B2_SIG_")  # tipb::ScalarFuncSig numbers, never typed twice

AGG_COUNT, AGG_SUM, AGG_AVG, AGG_MIN, AGG_MAX, AGG_FIRST = 3001, 3002, 3003, 3004, 3005, 3006
AGG_BIT_AND, AGG_BIT_OR, AGG_BIT_XOR = 3008, 3009, 3010
MERGE_ADD, MERGE_MAX, MERGE_OR, MERGE_XOR, MERGE_FIRST_KEY, MERGE_FIRST_VALUE = 0, 1, 2, 3, 4, 5  # b2_exec_agg_word_ops
EXEC_TABLE_SCAN, EXEC_INDEX_SCAN, EXEC_SELECTION, EXEC_AGGREGATION, EXEC_TOPN, EXEC_LIMIT, EXEC_STREAM_AGG, EXEC_PROJECTION = range(8)
COL_I64, COL_F64, COL_DECIMAL, COL_BYTES, COL_TIME, COL_DURATION, COL_JSON = 0, 1, 2, 3, 4, 5, 6
DRAIN_REMAIN, DRAIN_DRAINED, DRAIN_PAGING = 0, 1, 2


# ---- structs -----------------------------------------------------------------------------------
class CfBlock(C.Structure):
    _fields_ = [("keys", C.c_void_p), ("key_offs", C.c_void_p), ("vals", C.c_void_p), ("val_offs", C.c_void_p),
                ("n", C.c_uint32), ("_pad", C.c_uint32)]


class RegionSource(C.Structure):
    _fields_ = [("location", C.c_int32), ("device", C.c_int32), ("write", C.POINTER(CfBlock)), ("n_write", C.c_uint32),
                ("dflt", C.POINTER(CfBlock)), ("n_dflt", C.c_uint32), ("lock", C.POINTER(CfBlock)),
                ("read_ts", C.c_uint64), ("isolation_level", C.c_int32), ("check_has_newer_ts_data", C.c_int32),
                ("bypass_locks", C.POINTER(C.c_uint64)), ("n_bypass_locks", C.c_uint32),
                ("access_locks", C.POINTER(C.c_uint64)), ("n_access_locks", C.c_uint32)]


class KeyRange(C.Structure):
    _fields_ = [("start", C.c_char_p), ("start_len", C.c_uint32), ("end", C.c_char_p), ("end_len", C.c_uint32)]


class ColumnInfo(C.Structure):
    _fields_ = [("col_id", C.c_int64), ("tp", C.c_int32), ("flag", C.c_uint32), ("pk_handle", C.c_int32),
                ("default_len", C.c_uint32), ("default_val", C.c_char_p), ("decimal", C.c_int32), ("_pad", C.c_int32)]


class RpnNode(C.Structure):
    _fields_ = [("kind", C.c_int32), ("sig", C.c_int32), ("n_args", C.c_int32), ("field_tp", C.c_int32),
                ("field_flag", C.c_uint32), ("collation", C.c_int32), ("i64", C.c_int64), ("f64", C.c_double)]


class RpnExpr(C.Structure):
    _fields_ = [("nodes", C.POINTER(RpnNode)), ("n_nodes", C.c_uint32), ("_pad", C.c_uint32)]


class AggrDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("_pad", C.c_int32), ("arg", RpnExpr)]


class OrderBy(C.Structure):
    _fields_ = [("expr", RpnExpr), ("desc", C.c_int32), ("_pad", C.c_int32)]


class ExecutorDesc(C.Structure):
    _fields_ = [("tp", C.c_int32), ("desc", C.c_int32), ("table_id", C.c_int64), ("columns", C.POINTER(ColumnInfo)),
                ("n_columns", C.c_uint32), ("n_conditions", C.c_uint32), ("conditions", C.POINTER(RpnExpr)),
                ("group_by", C.POINTER(RpnExpr)), ("n_group_by", C.c_uint32), ("n_aggrs", C.c_uint32),
                ("aggrs", C.POINTER(AggrDesc)), ("order_by", C.POINTER(OrderBy)), ("n_order_by", C.c_uint32),
                ("_pad", C.c_uint32), ("limit", C.c_uint64)]


class DagPlan(C.Structure):
    _fields_ = [("executors", C.POINTER(ExecutorDesc)), ("n_executors", C.c_uint32), ("n_output_offsets", C.c_uint32),
                ("output_offsets", C.POINTER(C.c_uint32)), ("flags", C.c_uint64)]


class ExecConfig(C.Structure):
    _fields_ = [("output_location", C.c_int32), ("staging_tiles", C.c_int32), ("cuda_stream", C.c_uint64),
                ("jit", C.c_int32), ("_pad", C.c_int32), ("deadline_ns", C.c_uint64), ("paging_size", C.c_uint64), ("reserved", C.c_uint64 * 1)]


class Decimal(C.Structure):
    _fields_ = [("int_cnt", C.c_uint8), ("frac_cnt", C.c_uint8), ("result_frac_cnt", C.c_uint8), ("negative", C.c_uint8),
                ("word_buf", C.c_uint32 * 9)]


class Column(C.Structure):
    _fields_ = [("kind", C.c_int32), ("field_tp", C.c_int32), ("field_flag", C.c_uint32), ("_pad", C.c_uint32),
                ("len", C.c_uint64), ("data", C.c_void_p), ("null_bitmap", C.c_void_p), ("offsets", C.c_void_p)]


class Batch(C.Structure):
    _fields_ = [("columns", C.POINTER(Column)), ("n_columns", C.c_uint32), ("is_drained", C.c_int32),
                ("n_rows", C.c_uint64), ("n_warnings", C.c_uint32), ("_pad", C.c_uint32)]


class ExecStats(C.Structure):
    _fields_ = [("num_iterations", C.c_uint64), ("num_produced_rows", C.c_uint64), ("time_processed_ns", C.c_uint64),
                ("write_entries_scanned", C.c_uint64), ("write_processed_keys", C.c_uint64), ("processed_size", C.c_uint64),
                ("default_lookups", C.c_uint64), ("lock_processed_keys", C.c_uint64), ("met_newer_ts_data", C.c_int32),
                ("_pad", C.c_int32), ("kernel_time_ns", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("jit_launches", C.c_uint64)]


class ErrorInfo(C.Structure):
    _fields_ = [("status", C.c_int32), ("mysql_code", C.c_int32), ("entry_index", C.c_uint64), ("message", C.c_char * 232)]


class ChecksumResponse(C.Structure):
    _fields_ = [("checksum", C.c_uint64), ("total_kvs", C.c_uint64), ("total_bytes", C.c_uint64)]


class AggPartials(C.Structure):
    _fields_ = [("n_groups", C.c_uint32), ("acc_words", C.c_uint32), ("location", C.c_int32), ("has_group", C.c_int32),
                ("keys", C.c_void_p), ("key_null", C.c_void_p), ("acc", C.c_void_p), ("max_word_mask", C.c_uint64),
                ("key_words", C.c_uint32), ("_pad", C.c_uint32)]


class Warning(C.Structure):
    _fields_ = [("mysql_code", C.c_int32), ("_pad", C.c_int32), ("message", C.c_char * 120)]


class GenSpec(C.Structure):
    _fields_ = [("table_id", C.c_int64), ("first_handle", C.c_uint64), ("n_rows", C.c_uint64), ("n_cols", C.c_uint32),
                ("row_format", C.c_int32), ("seed", C.c_uint64), ("col_lo", C.POINTER(C.c_int64)),
                ("col_range", C.POINTER(C.c_uint64)), ("null_per_million", C.POINTER(C.c_uint32)),
                ("extra_versions_per_million", C.c_uint32), ("delete_per_million", C.c_uint32),
                ("lock_rec_per_million", C.c_uint32), ("commit_ts", C.c_uint64), ("newer_ts", C.c_uint64)]


class GenBlock(C.Structure):
    _fields_ = [("block", CfBlock), ("key_bytes", C.c_uint64), ("val_bytes", C.c_uint64), ("n_user_keys", C.c_uint64)]


class SstBlocks(C.Structure):
    _fields_ = [("data", C.c_void_p), ("block_offs", C.c_void_p), ("n_blocks", C.c_uint32), ("trailer_len", C.c_uint32),
                ("key_prefix_len", C.c_uint32), ("key_suffix_len", C.c_uint32)]


class SstStats(C.Structure):
    _fields_ = [("n_entries", C.c_uint64), ("key_bytes", C.c_uint64), ("val_bytes", C.c_uint64), ("n_restart_intervals", C.c_uint64),
                ("h2d_bytes", C.c_uint64), ("decode_ms", C.c_float), ("n_lz4_blocks", C.c_uint32)]


class SstMergeStats(C.Structure):
    _fields_ = [("n_in", C.c_uint64), ("n_out", C.c_uint64), ("n_invisible", C.c_uint64), ("n_hidden", C.c_uint64), ("n_deletions", C.c_uint64),
                ("key_bytes", C.c_uint64), ("val_bytes", C.c_uint64), ("h2d_bytes", C.c_uint64), ("decode_ms", C.c_float), ("merge_ms", C.c_float),
                ("n_lz4_blocks", C.c_uint32), ("n_runs", C.c_uint32)]


class SstEncoded(C.Structure):
    _fields_ = [("data", C.c_void_p), ("block_offs", C.c_void_p), ("data_len", C.c_uint64), ("n_blocks", C.c_uint32), ("_pad", C.c_uint32)]


class EncodedChunk(C.Structure):
    _fields_ = [("rows_data", C.c_void_p), ("len", C.c_uint64), ("n_rows", C.c_uint64), ("encode_type", C.c_int32), ("location", C.c_int32)]


ENCODE_TYPE_DEFAULT, ENCODE_TYPE_CHUNK = 0, 1
JIT_AUTO, JIT_SYNC, JIT_OFF = 0, 1, 2

EXPORTED_SYMBOLS = [
    "b2_abi_version", "b2_build_info", "b2_last_error_message", "b2_check_supported", "b2_plan_prepare", "b2_plan_precompile", "b2_jit_counters", "b2_plan_literal", "b2_exec_open", "b2_exec_schema",
    "b2_exec_next_batch", "b2_exec_next_batch_async", "b2_exec_poll", "b2_exec_warnings", "b2_region_pin", "b2_region_unpin", "b2_region_cache_stats", "b2_exec_collect_stats", "b2_exec_last_error", "b2_exec_can_be_cached", "b2_exec_encode_batch", "b2_exec_take_scanned_range", "b2_exec_collect_scanned_rows_per_range", "b2_exec_close",
    "b2_exec_agg_partials", "b2_exec_agg_word_ops", "b2_agg_merge", "b2_dag_handle", "b2_checksum_handle", "b2_gen_create", "b2_gen_destroy", "b2_copy_to_host", "b2_copy_to_device",
    "b2_sst_decode", "b2_sst_merge", "b2_sst_free", "b2_sst_encode",
    "b2_device_count", "b2_host_alloc_pinned", "b2_host_alloc_pinned_near", "b2_device_numa_node", "b2_host_free_pinned",
]

_lib = None


def lib():
    """Load libb2copr.so (built in-tree by __graft_entry__.build()).  Fails loudly when absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: the CUDA extension is the product path and there is no CPU fallback. "
            "Run `python -c 'import __graft_entry__ as g; g.build()'` first.")
    L = C.CDLL(LIB_PATH)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32
    L.b2_abi_version.restype = u32
    L.b2_build_info.restype = C.c_char_p
    L.b2_last_error_message.restype = C.c_char_p
    L.b2_check_supported.argtypes = [C.POINTER(DagPlan)]
    L.b2_check_supported.restype = i32
    L.b2_plan_prepare.argtypes = [C.POINTER(DagPlan), i32]
    L.b2_plan_prepare.restype = i32
    L.b2_plan_precompile.argtypes = [C.POINTER(DagPlan), C.POINTER(i32)]
    L.b2_plan_precompile.restype = i32
    L.b2_jit_counters.argtypes = [C.POINTER(u64), C.POINTER(u64)]
    L.b2_jit_counters.restype = None
    L.b2_exec_open.argtypes = [C.POINTER(DagPlan), C.POINTER(KeyRange), u32, C.POINTER(RegionSource), C.POINTER(ExecConfig), C.POINTER(vp)]
    L.b2_exec_open.restype = i32
    L.b2_exec_schema.argtypes = [vp, C.POINTER(i32), C.POINTER(u32), C.POINTER(u32)]
    L.b2_exec_schema.restype = i32
    L.b2_exec_next_batch.argtypes = [vp, u64, C.POINTER(Batch)]
    L.b2_exec_next_batch.restype = i32
    L.b2_exec_next_batch_async.argtypes = [vp, u64]
    L.b2_exec_next_batch_async.restype = i32
    L.b2_exec_poll.argtypes = [vp, C.POINTER(Batch)]
    L.b2_exec_poll.restype = i32
    L.b2_exec_warnings.argtypes = [vp, C.POINTER(Warning), u32, C.POINTER(u64)]
    L.b2_exec_warnings.restype = i32
    L.b2_region_pin.argtypes = [i32, u64, u64, C.POINTER(RegionSource), C.POINTER(RegionSource)]
    L.b2_region_pin.restype = i32
    L.b2_region_unpin.argtypes = [i32, u64, u64]
    L.b2_region_unpin.restype = i32
    L.b2_region_cache_stats.argtypes = [i32, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.b2_region_cache_stats.restype = None
    L.b2_exec_collect_stats.argtypes = [vp, C.POINTER(ExecStats)]
    L.b2_exec_collect_stats.restype = i32
    L.b2_exec_last_error.argtypes = [vp, C.POINTER(ErrorInfo)]
    L.b2_exec_last_error.restype = i32
    L.b2_exec_encode_batch.argtypes = [vp, i32, i32, C.POINTER(EncodedChunk)]
    L.b2_exec_encode_batch.restype = i32
    L.b2_exec_take_scanned_range.argtypes = [vp, C.POINTER(C.c_void_p), C.POINTER(C.c_uint32), C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]
    L.b2_exec_take_scanned_range.restype = i32
    L.b2_exec_collect_scanned_rows_per_range.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    L.b2_exec_collect_scanned_rows_per_range.restype = i32
    L.b2_exec_can_be_cached.argtypes = [vp]
    L.b2_exec_can_be_cached.restype = i32
    L.b2_exec_agg_partials.argtypes = [vp, C.POINTER(AggPartials)]
    L.b2_exec_agg_partials.restype = i32
    L.b2_exec_agg_word_ops.argtypes = [vp, C.POINTER(C.c_uint8), C.POINTER(u32)]
    L.b2_exec_agg_word_ops.restype = i32
    L.b2_agg_merge.argtypes = [i32, u64, u64, u32, u32, vp, u64, vp, vp, u64, C.POINTER(u64), u32, C.POINTER(C.c_uint8), i32, vp, vp, vp, C.POINTER(u64)]
    L.b2_agg_merge.restype = i32
    L.b2_exec_close.argtypes = [vp]
    L.b2_exec_close.restype = None
    L.b2_dag_handle.argtypes = [C.POINTER(DagPlan), C.POINTER(KeyRange), u32, C.POINTER(RegionSource), C.POINTER(ExecConfig), C.POINTER(Batch), C.POINTER(vp)]
    L.b2_dag_handle.restype = i32
    L.b2_checksum_handle.argtypes = [C.POINTER(KeyRange), u32, C.c_char_p, u32, C.c_char_p, u32, C.POINTER(RegionSource), C.POINTER(ExecConfig), C.POINTER(ChecksumResponse), C.POINTER(ExecStats)]
    L.b2_checksum_handle.restype = i32
    L.b2_gen_create.argtypes = [i32, C.POINTER(GenSpec), C.POINTER(vp), C.POINTER(GenBlock)]
    L.b2_gen_create.restype = i32
    L.b2_gen_destroy.argtypes = [vp]
    L.b2_gen_destroy.restype = None
    L.b2_sst_decode.argtypes = [i32, i32, C.POINTER(SstBlocks), C.POINTER(vp), C.POINTER(CfBlock), C.POINTER(SstStats)]
    L.b2_sst_decode.restype = i32
    L.b2_sst_merge.argtypes = [i32, i32, C.POINTER(SstBlocks), u32, C.POINTER(u64), u64, C.POINTER(vp), C.POINTER(CfBlock), C.POINTER(SstMergeStats)]
    L.b2_sst_merge.restype = i32
    L.b2_sst_free.argtypes = [vp]
    L.b2_sst_free.restype = None
    L.b2_sst_encode.argtypes = [i32, C.POINTER(CfBlock), u32, u32, u32, C.c_uint8, u32, u32, C.POINTER(vp), C.POINTER(SstEncoded)]
    L.b2_sst_encode.restype = i32
    L.b2_copy_to_host.argtypes = [i32, vp, vp, u64]
    L.b2_copy_to_host.restype = i32
    L.b2_copy_to_device.argtypes = [i32, vp, vp, u64]
    L.b2_copy_to_device.restype = i32
    L.b2_device_count.restype = i32
    L.b2_host_alloc_pinned.argtypes = [u64]
    L.b2_host_alloc_pinned.restype = vp
    L.b2_host_alloc_pinned_near.argtypes = [i32, u64]
    L.b2_host_alloc_pinned_near.restype = vp
    L.b2_device_numa_node.argtypes = [i32]
    L.b2_device_numa_node.restype = i32
    L.b2_host_free_pinned.argtypes = [vp]
    L.b2_host_free_pinned.restype = None
    if L.b2_abi_version() != 4:
        raise RuntimeError("libb2copr ABI version mismatch")
    _lib = L
    return L
