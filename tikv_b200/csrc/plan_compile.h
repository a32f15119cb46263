// Host-side lowering of the ABI plan (b2_dag_plan) into the device plan (DevPlan).
// Mirrors what BatchExecutorsRunner::check_supported / build_executors do on the CPU
// (components/tidb_query_executors/src/runner.rs:111-206, 252-603) plus the aggregate SUM/AVG cast rewrite
// (components/tidb_query_aggr/src/util.rs:31-66).  Pure C++ (no CUDA) so the host emulation test can use it.
#pragma once
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "b2_device.h"

namespace b2 {

struct OutCol { int kind; int field_tp; uint32_t field_flag; };

struct CompiledPlan {
  DevPlan dev;
  std::vector<OutCol> schema;            // output schema of the outermost executor
  std::vector<uint32_t> output_offsets;  // indices into `schema` delivered to the caller
  uint64_t scan_limit = ~0ull;           // BatchLimitExecutor on top of a scan / selection pipeline (limit_executor.rs), ~0 = none
  int64_t imms[MAX_IMMS] = {};           // hoisted constants, referenced by DevNode::sig / FastCond::imm_slot (ScanArgs::imms at launch)
  int n_imms = 0;
  bool desc = false;                     // TableScan.desc
  // bytes constants (LIKE patterns): the bytes live in `pool`, uploaded with the request; their constants are launch
  // parameters holding a cell reference (address << 16 | length) that patch_pool_imms fills once the pool has an address
  std::vector<uint8_t> pool;
  struct PoolImm { int slot; uint32_t off, len; };
  std::vector<PoolImm> pool_imms;
};
// bytes constants seen by lower_expr while a plan is being compiled: (node index in DevPlan::nodes, offset, length)
struct PoolRef { int node; uint32_t off, len; };
inline std::vector<uint8_t>& lowering_pool() { static thread_local std::vector<uint8_t> p; return p; }
inline std::vector<PoolRef>& lowering_pool_refs() { static thread_local std::vector<PoolRef> r; return r; }

inline int col_kind_of_tp(int tp) {  // def/eval_type.rs:53-95
  switch (tp) {
    case B2_TP_TINY: case B2_TP_SHORT: case B2_TP_INT24: case B2_TP_LONG: case B2_TP_LONGLONG: case B2_TP_YEAR: case B2_TP_BIT: return CK_INT;
    case B2_TP_FLOAT: case B2_TP_DOUBLE: return CK_REAL;
    default: return CK_OTHER;
  }
}
// kinds of a scan column: the two above are evaluated by expressions; the rest can only be carried to the output
inline int scan_col_kind(int tp, int decimal) {
  switch (tp) {
    case B2_TP_DATE: case B2_TP_DATETIME: return decimal >= -1 && decimal <= 6 ? CK_TIME : CK_OTHER;  // (TIMESTAMP converts through the session time zone: CPU)
    case B2_TP_DURATION: return CK_DUR;
    case B2_TP_VARCHAR: case B2_TP_VARSTRING: case B2_TP_STRING: case B2_TP_BLOB: case 0xf9: case 0xfa: case 0xfb: case 0xff: return CK_BYTES;
    case B2_TP_JSON: return CK_JSON;
    case B2_TP_NEWDECIMAL: return CK_DEC;
    default: return col_kind_of_tp(tp);
  }
}
inline int out_kind_of(int ck) {
  switch (ck) {
    case CK_REAL: return B2_COL_F64;
    case CK_TIME: return B2_COL_TIME;
    case CK_DUR: return B2_COL_DURATION;
    case CK_BYTES: return B2_COL_BYTES;
    case CK_JSON: return B2_COL_JSON;
    case CK_DEC: return B2_COL_DECIMAL;
    default: return B2_COL_I64;
  }
}
inline int v2_class_of(int tp, bool is_unsigned) {  // compat_v1.rs:55-129 write_v2_as_datum
  switch (tp) {
    case B2_TP_TINY: case B2_TP_SHORT: case B2_TP_INT24: case B2_TP_LONG: case B2_TP_LONGLONG: return is_unsigned ? V2_UINT : V2_INT;
    case B2_TP_YEAR: case B2_TP_DURATION: return V2_INT;
    case B2_TP_DATE: case B2_TP_DATETIME: case B2_TP_TIMESTAMP: case B2_TP_ENUM: case B2_TP_BIT: case B2_TP_SET: return V2_UINT;
    case B2_TP_FLOAT: case B2_TP_DOUBLE: case B2_TP_NEWDECIMAL: case B2_TP_JSON: return V2_COPY;
    case B2_TP_VARCHAR: case B2_TP_VARSTRING: case B2_TP_STRING: case B2_TP_BLOB: case 0xf9: case 0xfa: case 0xfb: case 0xff: return V2_BYTES;
    case B2_TP_NULL: return V2_NIL;
    default: return V2_UNSUPPORTED;
  }
}

// lower one RPN expression; returns false + msg when unsupported
inline bool lower_expr(const b2_rpn_expr& x, DevPlan& P, DevExpr* out, uint8_t* ret_et, uint8_t* ret_unsigned, int* ret_tp, uint32_t* ret_flag, std::string* msg) {
  if (x.n_nodes == 0 || !x.nodes) { *msg = "empty expression"; return false; }
  if (P.n_nodes + (int)x.n_nodes > MAX_NODES) { *msg = "too many expression nodes"; return false; }
  out->start = (uint16_t)P.n_nodes; out->n = (uint16_t)x.n_nodes;
  uint8_t st_et[MAX_STACK];
  int sp = 0;
  for (uint32_t i = 0; i < x.n_nodes; ++i) {
    const b2_rpn_node& s = x.nodes[i];
    DevNode d;
    d.sig = s.sig; d.kind = (uint8_t)s.kind; d.n_args = (uint8_t)s.n_args; d.et = 0; d.is_unsigned = (s.field_flag & B2_FLAG_UNSIGNED) ? 1 : 0; d.imm = s.i64;
    switch (s.kind) {
      case B2_RPN_CONST_INT: d.et = 0; break;
      case B2_RPN_CONST_UINT: d.et = 0; d.is_unsigned = 1; break;
      case B2_RPN_CONST_REAL: d.et = 1; d.imm = (int64_t)f64_bits(s.f64); break;
      case B2_RPN_CONST_NULL: {
        int k = col_kind_of_tp(s.field_tp);
        if (s.field_tp == B2_TP_DATE || s.field_tp == B2_TP_DATETIME) { d.et = 2; d.is_unsigned = 1; d.imm = 0; break; }
        if (s.field_tp == B2_TP_DURATION) { d.et = 3; d.imm = 0; break; }
        if (scan_col_kind(s.field_tp, 0) == CK_BYTES) { d.et = 4; d.imm = 0; break; }
        if (s.field_tp == B2_TP_NEWDECIMAL) { d.et = 5; d.imm = 0; break; }
        if (k == CK_OTHER) { *msg = "NULL constant of a non Int/Real type"; return false; }
        d.et = (uint8_t)k; d.imm = 0;
        break;
      }
      // DATE / DATETIME and DURATION values take part in comparisons only (eval types 2 and 3 below): a time is its CoreTime
      // bit field without the fsp / type nibble, ordered as u64 (`Ord for Time`), a duration its signed nanoseconds, so
      // their comparison functions lower to the integer ones
      case B2_RPN_CONST_TIME: {
        if (s.field_tp != B2_TP_DATE && s.field_tp != B2_TP_DATETIME) { *msg = "time constant of a type other than DATE / DATETIME (TIMESTAMP needs the session time zone)"; return false; }
        d.kind = B2_RPN_CONST_UINT; d.et = 2; d.is_unsigned = 1;
        d.imm = (int64_t)(time_bits_from_packed((uint64_t)s.i64, s.field_tp == B2_TP_DATE, 0) & ~15ull);
        break;
      }
      case B2_RPN_CONST_DURATION: d.kind = B2_RPN_CONST_INT; d.et = 3; d.is_unsigned = 0; break;
      case B2_RPN_CONST_DECIMAL:  // eval type 5: a cell reference to (precision, fraction, binary decimal); comparisons take them
      case B2_RPN_CONST_BYTES: {  // eval type 4: a cell reference; only LIKE takes them
        if (s.n_args < 0 || s.n_args > 0xffff || (s.n_args && !s.i64)) { *msg = "bytes constant longer than 65535 bytes (or null pointer)"; return false; }
        std::vector<uint8_t>& pool = lowering_pool();
        lowering_pool_refs().push_back(PoolRef{P.n_nodes, (uint32_t)pool.size(), (uint32_t)s.n_args});
        const uint8_t* src = (const uint8_t*)(uintptr_t)s.i64;
        pool.insert(pool.end(), src, src + s.n_args);
        pool.resize((pool.size() + 15) & ~(size_t)15, 0);
        if (s.kind == B2_RPN_CONST_DECIMAL) {
          b2_decimal chk;
          if (!raw_decimal_parse(src, (unsigned int)s.n_args, &chk)) { *msg = "decimal constant is not a valid (precision, fraction, binary decimal) payload"; return false; }
        }
        d.kind = B2_RPN_CONST_UINT; d.et = s.kind == B2_RPN_CONST_DECIMAL ? 5 : 4; d.is_unsigned = 1; d.n_args = 0; d.imm = 0;
        break;
      }
      case B2_RPN_COLUMN_REF: {
        if (s.i64 < 0 || s.i64 >= P.n_cols) { *msg = "column offset out of range"; return false; }
        const DevCol& c = P.cols[s.i64];
        if (c.kind == CK_TIME) { d.et = 2; d.is_unsigned = 1; break; }
        if (c.kind == CK_DUR) { d.et = 3; d.is_unsigned = 0; break; }
        if (c.kind == CK_BYTES) { d.et = 4; d.is_unsigned = 1; break; }
        if (c.kind == CK_DEC) { d.et = 5; d.is_unsigned = 1; break; }
        if (c.kind > CK_REAL) { *msg = "expression over a column that is not Int / Real / DATE / DATETIME / DURATION / bytes / DECIMAL"; return false; }
        d.et = c.kind; d.is_unsigned = c.is_unsigned;
        break;
      }
      case B2_RPN_FN: {
        int sig = s.sig, na = s.n_args;
        bool cmp = sig >= 100 && sig < 170 && (sig % 10 == 0 || sig % 10 == 1);
        bool real_args = false, real_ret = false;
        int want = 2;
        bool mixed = false;  // argument types already checked
        {  // time / duration: comparisons, IN, IS NULL -> their integer twins over the lowered operands
          const bool tcmp = sig >= 100 && sig < 170 && (sig % 10 == 4 || sig % 10 == 5);
          const bool tin = sig == B2_SIG_IN_TIME || sig == B2_SIG_IN_DURATION, tnull = sig == B2_SIG_TIME_IS_NULL || sig == B2_SIG_DURATION_IS_NULL;
          if (tcmp || tin || tnull) {
            const uint8_t need = (tcmp ? sig % 10 == 4 : (sig == B2_SIG_IN_TIME || sig == B2_SIG_TIME_IS_NULL)) ? 2 : 3;
            const int w = tcmp ? 2 : (tnull ? 1 : na);
            if (na != w || na < 1 || sp < na) { *msg = "bad arity for sig " + std::to_string(sig); return false; }
            for (int k = 0; k < na; ++k)
              if (st_et[sp - 1 - k] != need) { *msg = "argument eval type does not match sig " + std::to_string(sig); return false; }
            d.sig = tcmp ? sig / 10 * 10 : (tin ? B2_SIG_IN_INT : B2_SIG_INT_IS_NULL);
            sp -= na;
            d.et = 0;
            break;
          }
        }
        if (is_dec_sig(sig)) {  // comparisons, IN, IS NULL over DECIMAL cells and constants -> int
          const bool dcmp = sig >= 100 && sig < 170;
          const int w = dcmp ? 2 : (sig == B2_SIG_DECIMAL_IS_NULL ? 1 : na);
          if (na != w || na < 1 || sp < na) { *msg = "bad arity for sig " + std::to_string(sig); return false; }
          for (int k = 0; k < na; ++k)
            if (st_et[sp - 1 - k] != 5) { *msg = "argument eval type does not match sig " + std::to_string(sig); return false; }
          sp -= na;
          d.et = 0;
          break;
        }
        if (sig == B2_SIG_LIKE) {  // (bytes, bytes, int) -> int; charset and collator as map_like_sig picks them (lib.rs:99-135)
          if (na != 3 || sp < 3) { *msg = "bad arity for sig " + std::to_string(sig); return false; }
          if (st_et[sp - 3] != 4 || st_et[sp - 2] != 4 || st_et[sp - 1] != 0) { *msg = "argument eval type does not match sig " + std::to_string(sig); return false; }
          // collation -> (byte-equality collator?, charset): field_type.rs:130-146
          auto coll = [](int n, bool* bin_eq, int* cs) {  // cs: 0 binary, 1 utf8mb4
            switch (n) {
              case -63: case 63: case 47: *bin_eq = true; *cs = 0; return true;                 // Binary
              case -46: case -83: case -65: case -309: *bin_eq = true; *cs = 1; return true;   // Utf8Mb4Bin, Utf8Mb40900Bin
              default: if (n >= 0) { *bin_eq = true; *cs = 1; return true; }                    // Utf8Mb4BinNoPadding
                       return false;                                                          // _ci collations, latin1, gbk: CPU
            }
          };
          // the children's collations: the nodes that produced the two byte operands (their last nodes in post-order)
          int tgt = -1, pat = -1;
          {  // walk back over the operand subtrees: escape (1 value), pattern, target
            int need = 1, k = (int)i - 1;
            auto skip = [&](int& k2) { int want = 1; while (want > 0 && k2 >= 0) { const b2_rpn_node& q = x.nodes[k2]; want += (q.kind == B2_RPN_FN ? q.n_args : 0) - 1; --k2; } };
            (void)need;
            skip(k); pat = k; skip(k); tgt = k;
          }
          bool be_r, be_t, be_p; int cs_r, cs_t, cs_p;
          if (tgt < 0 || pat < 0 || !coll(s.collation, &be_r, &cs_r) || !coll(x.nodes[tgt].collation, &be_t, &cs_t) || !coll(x.nodes[pat].collation, &be_p, &cs_p)) {
            *msg = "LIKE under a collation that is not binary / *_bin is not on the device path"; return false;
          }
          d.imm = cs_t == cs_p ? cs_t : cs_r;
          sp -= 3;
          d.et = 0;
          break;
        }
        if (cmp) real_args = (sig % 10) == 1;
        else switch (sig) {
          case B2_SIG_BIT_AND: case B2_SIG_BIT_OR: case B2_SIG_BIT_XOR: break;
          case B2_SIG_BIT_NEG: case B2_SIG_CAST_INT_AS_INT: want = 1; break;
          case B2_SIG_CAST_INT_AS_REAL: want = 1; real_ret = true; break;
          case B2_SIG_CAST_REAL_AS_REAL: want = 1; real_args = real_ret = true; break;
          case B2_SIG_PLUS_REAL: case B2_SIG_MINUS_REAL: case B2_SIG_MULTIPLY_REAL: real_args = real_ret = true; break;
          case B2_SIG_PLUS_INT: case B2_SIG_MINUS_INT: case B2_SIG_MULTIPLY_INT: case B2_SIG_MULTIPLY_INT_UNSIGNED:
          case B2_SIG_LOGICAL_AND: case B2_SIG_LOGICAL_OR: case B2_SIG_LOGICAL_XOR: break;
          case B2_SIG_UNARY_NOT_INT: case B2_SIG_INT_IS_NULL: case B2_SIG_INT_IS_TRUE: case B2_SIG_INT_IS_FALSE: want = 1; break;
          case B2_SIG_UNARY_NOT_REAL: case B2_SIG_REAL_IS_NULL: case B2_SIG_REAL_IS_TRUE: case B2_SIG_REAL_IS_FALSE: want = 1; real_args = true; break;
          case B2_SIG_IN_INT: want = na; if (na < 1) want = -1; break;
          case B2_SIG_IN_REAL: want = na; real_args = true; if (na < 1) want = -1; break;
          case B2_SIG_INT_DIVIDE_INT: case B2_SIG_MOD_INT: case B2_SIG_IF_NULL_INT: break;
          case B2_SIG_MOD_REAL: case B2_SIG_IF_NULL_REAL: case B2_SIG_DIVIDE_REAL: real_args = real_ret = true; break;
          case B2_SIG_UNARY_MINUS_INT: case B2_SIG_ABS_INT: case B2_SIG_ABS_UINT: want = 1; break;
          case B2_SIG_UNARY_MINUS_REAL: case B2_SIG_ABS_REAL: want = 1; real_args = real_ret = true; break;
          case B2_SIG_COALESCE_INT: want = na; if (na < 1) want = -1; break;
          case B2_SIG_COALESCE_REAL: want = na; real_args = real_ret = true; if (na < 1) want = -1; break;
          case B2_SIG_IF_INT: case B2_SIG_IF_REAL: case B2_SIG_CASE_WHEN_INT: case B2_SIG_CASE_WHEN_REAL: {
            // [cond Int, value T]* [else T]  (IF: cond, then, else); case_when_validator impl_control.rs:130-140
            const bool rr = sig == B2_SIG_IF_REAL || sig == B2_SIG_CASE_WHEN_REAL, is_if = sig == B2_SIG_IF_INT || sig == B2_SIG_IF_REAL;
            if (na < 1 || (is_if && na != 3) || sp < na) { *msg = "bad arity for sig " + std::to_string(sig); return false; }
            for (int k = 0; k < na; ++k) {
              const bool is_cond = is_if ? k == 0 : ((k & 1) == 0 && k + 1 < na);
              if (st_et[sp - na + k] != ((is_cond || !rr) ? 0 : 1)) { *msg = "argument eval type does not match sig " + std::to_string(sig); return false; }
            }
            want = na; real_ret = rr; mixed = true;
            break;
          }
          default: *msg = "ScalarFunction sig " + std::to_string(sig) + " is not supported on the device path"; return false;
        }
        if (na != want || sp < na) { *msg = "bad arity for sig " + std::to_string(sig); return false; }
        for (int k = 0; k < na && !mixed; ++k)
          if (st_et[sp - 1 - k] != (real_args ? 1 : 0)) { *msg = "argument eval type does not match sig " + std::to_string(sig); return false; }
        sp -= na;
        d.et = real_ret ? 1 : 0;
        break;
      }
      default: *msg = "bad rpn node kind"; return false;
    }
    if (sp >= MAX_STACK) { *msg = "expression too deep"; return false; }
    st_et[sp++] = d.et;
    P.nodes[P.n_nodes++] = d;
  }
  if (sp != 1) { *msg = "expression does not reduce to one value"; return false; }
  if (st_et[0] >= 2) { *msg = "DATE / DATETIME / DURATION valued expression: only comparisons over them are on the device path"; return false; }
  const b2_rpn_node& last = x.nodes[x.n_nodes - 1];
  const DevNode& dl = P.nodes[P.n_nodes - 1];
  if (ret_et) *ret_et = dl.et;
  if (ret_unsigned) *ret_unsigned = dl.is_unsigned;
  if (last.kind == B2_RPN_COLUMN_REF) {
    if (ret_tp) *ret_tp = P.cols[last.i64].tp;
    if (ret_flag) *ret_flag = (P.cols[last.i64].is_unsigned ? B2_FLAG_UNSIGNED : 0) | (P.cols[last.i64].not_null ? B2_FLAG_NOT_NULL : 0);
  } else {
    if (ret_tp) *ret_tp = last.field_tp ? last.field_tp : (dl.et ? B2_TP_DOUBLE : B2_TP_LONGLONG);
    if (ret_flag) *ret_flag = last.field_flag;
  }
  return true;
}

// decode a datum-encoded column default (datum_codec.rs:401-446) at plan time
inline void lower_default(const b2_column_info& ci, DevCol& c) {
  c.def_state = DS_NONE; c.default_bits = 0;
  if (!ci.default_val || ci.default_len == 0) return;
  const uint8_t* p = ci.default_val;
  uint32_t n = ci.default_len;
  const uint64_t S = 0x8000000000000000ull;
  uint8_t flag = p[0];
  if (flag == 0) { c.def_state = DS_NULL; return; }
  c.def_state = DS_ERROR;
  if (c.kind == CK_INT) {
    if ((flag == 3 || flag == 4) && n >= 9) { c.default_bits = (int64_t)(ld_be64(p + 1) ^ (flag == 3 ? S : 0)); c.def_state = DS_VALUE; }
    else if (flag == 8) { int64_t v; if (dec_var_i64(p + 1, n - 1, &v)) { c.default_bits = v; c.def_state = DS_VALUE; } }
    else if (flag == 9) { uint64_t v; if (dec_var_u64(p + 1, n - 1, &v)) { c.default_bits = (int64_t)v; c.def_state = DS_VALUE; } }
  } else if (c.kind == CK_REAL) {
    if (flag == 5 && n >= 9) {
      double f = cmp_u64_to_f64(ld_be64(p + 1));
      if (c.tp == B2_TP_FLOAT) f = (double)(float)f;
      if (f != f) c.def_state = DS_NULL; else { c.default_bits = (int64_t)f64_bits(f); c.def_state = DS_VALUE; }
    }
  } else {
    c.def_state = DS_VALUE;  // never materialised on the device; only "has a default" matters
  }
}

// returns B2_OK or B2_ERR_UNSUPPORTED / B2_ERR_INVALID_ARG with *msg set
inline int compile_plan(const b2_dag_plan* plan, CompiledPlan* out, std::string* msg) {
  DevPlan& P = out->dev;
  memset(&P, 0, sizeof(P));
  lowering_pool().clear(); lowering_pool_refs().clear();
  out->pool.clear(); out->pool_imms.clear();
  if (!plan || plan->n_executors == 0 || !plan->executors) { *msg = "empty plan"; return B2_ERR_INVALID_ARG; }
  const b2_executor_desc& scan = plan->executors[0];
  if (scan.tp != B2_EXEC_TABLE_SCAN && scan.tp != B2_EXEC_INDEX_SCAN) { *msg = "first executor must be TableScan or IndexScan"; return B2_ERR_UNSUPPORTED; }
  const bool is_index = scan.tp == B2_EXEC_INDEX_SCAN;
  out->desc = scan.desc != 0;  // scan_executor.rs:89-101: ranges in reverse order, each scanned backward (engine.cu: reversed chunks)
  if (scan.n_columns == 0 || scan.n_columns > MAX_COLS) { *msg = "TableScan with 0 or more than 64 columns"; return B2_ERR_UNSUPPORTED; }
  P.n_cols = (int)scan.n_columns;
  for (int i = 0; i < P.n_cols; ++i) {
    const b2_column_info& ci = scan.columns[i];
    DevCol& c = P.cols[i];
    c.col_id = ci.col_id; c.tp = (uint8_t)ci.tp;
    c.is_unsigned = (ci.flag & B2_FLAG_UNSIGNED) ? 1 : 0;
    c.not_null = (ci.flag & B2_FLAG_NOT_NULL) ? 1 : 0;
    c.kind = (uint8_t)scan_col_kind(ci.tp, ci.decimal);
    c.fsp = (uint8_t)(ci.decimal > 0 && ci.decimal <= 6 ? ci.decimal : 0);
    c.v2_class = (uint8_t)v2_class_of(ci.tp, c.is_unsigned);
    c.role = CR_NORMAL;
    if (ci.pk_handle && is_index) { c.role = CR_IDX_HANDLE; c.kind = CK_INT; }
    else if (ci.pk_handle) { c.role = CR_HANDLE; c.kind = CK_INT; P.has_handle_cols = 1; }
    else if (ci.col_id == B2_EXTRA_PHYSICAL_TABLE_ID_COL_ID) { c.role = CR_TABLE_ID; c.kind = CK_INT; }
    else if (ci.col_id == B2_EXTRA_COMMIT_TS_COL_ID) { c.role = CR_COMMIT_TS; c.kind = CK_INT; }
    lower_default(ci, c);
  }
  if (is_index) {
    // index_scan_executor.rs:47-170: [index columns in index order][int handle (pk_handle)]?[physical table id (col id -3)]?
    int n = P.n_cols;
    const bool has_tid = n > 0 && P.cols[n - 1].role == CR_TABLE_ID;
    const int tail = has_tid ? 1 : 0;
    const bool has_handle = n > tail && P.cols[n - 1 - tail].role == CR_IDX_HANDLE;
    P.idx_cols = n - tail - (has_handle ? 1 : 0);
    if (P.idx_cols <= 0) { *msg = "IndexScan without index columns"; return B2_ERR_UNSUPPORTED; }
    for (int i = 0; i < P.idx_cols; ++i) {
      if (P.cols[i].role != CR_NORMAL) { *msg = "IndexScan: the handle / physical table id columns must come last"; return B2_ERR_UNSUPPORTED; }
      if (P.cols[i].kind > CK_REAL) { *msg = "IndexScan over a column that is not Int/Real is not on the device path yet"; return B2_ERR_UNSUPPORTED; }
    }
  }
  // duplicate column ids: only the last one is ever filled (table_scan_executor.rs:90-94)
  if (!is_index)
  for (int i = 0; i < P.n_cols; ++i) {
    if (P.cols[i].role == CR_HANDLE) continue;
    for (int j = i + 1; j < P.n_cols; ++j)
      if (P.cols[j].role != CR_HANDLE && P.cols[j].col_id == P.cols[i].col_id) { P.cols[i].role = CR_SHADOWED; break; }
  }
  // v2 position hint: rank of the column id among the ids a row is expected to hold (the plan's own columns)
  for (int i = 0; i < P.n_cols; ++i) {
    int rank = 0;
    for (int j = 0; j < P.n_cols; ++j)
      if (j != i && P.cols[j].role == CR_NORMAL && P.cols[j].col_id > 0 && P.cols[j].col_id < P.cols[i].col_id) ++rank;
    P.cols[i].v2_hint = (uint8_t)rank;
  }
  // exact-layout fast path: the sorted ids of the plan's row-stored columns, when there are at most 8 of them (< 256)
  {
    std::vector<int64_t> ids;
    bool ok = true;
    for (int i = 0; i < P.n_cols; ++i) {
      if (P.cols[i].role == CR_SHADOWED) ok = false;
      if (P.cols[i].role != CR_NORMAL) continue;
      if (P.cols[i].col_id <= 0 || P.cols[i].col_id > 255) ok = false;
      if (P.cols[i].v2_class == V2_UNSUPPORTED) ok = false;  // such a row raises an error: general path
      ids.push_back(P.cols[i].col_id);
    }
    std::sort(ids.begin(), ids.end());
    if (is_index) ok = false;  // index rows carry no row value
    P.fast_n = 0; P.fast_ids = 0; P.fast_cls = 0; P.fast_uns = 0; P.fast_filled = 0; P.n_out_slow = 0; P.fast_v1 = 0;
    for (int h = 0; h < 8; ++h) P.fast_out[h] = -1;
    if (ok && !ids.empty() && ids.size() <= 8) {
      P.fast_n = (int32_t)ids.size();
      for (size_t i = 0; i < ids.size(); ++i) P.fast_ids |= (uint64_t)ids[i] << (8 * i);
      for (int i = 0; i < P.n_cols; ++i) {
        const DevCol& col = P.cols[i];
        if (col.role == CR_HANDLE || col.role == CR_TABLE_ID || col.role == CR_COMMIT_TS) P.fast_filled |= 1ull << i;
        if (col.role != CR_NORMAL) continue;
        P.fast_filled |= 1ull << i;
        size_t rank = std::lower_bound(ids.begin(), ids.end(), col.col_id) - ids.begin();
        if (col.v2_class == V2_INT || col.v2_class == V2_UINT) P.fast_cls |= 1u << rank;
        if (col.v2_class != V2_INT) P.fast_uns |= 1u << rank;
      }
      // the v1 twin needs single-byte column ids (zigzag varint of ids <= 63) and integer datums only; a column whose
      // tp makes decode_int_datum irrelevant (Real ...) keeps v1 rows on the general walk
      bool v1 = P.fast_cls == (1u << P.fast_n) - 1u && ids.back() <= 63;
      for (int i = 0; i < P.n_cols; ++i) if (P.cols[i].role == CR_NORMAL && P.cols[i].kind != CK_INT) v1 = false;
      P.fast_v1 = v1 ? 1 : 0;
    }
  }
  P.mode = PM_SCAN;
  std::vector<OutCol> schema;
  for (int i = 0; i < P.n_cols; ++i) {
    OutCol oc;
    oc.kind = out_kind_of(P.cols[i].kind);
    oc.field_tp = P.cols[i].tp; oc.field_flag = scan.columns[i].flag;
    schema.push_back(oc);
  }
  bool terminal = false, projected = false;
  for (uint32_t ei = 1; ei < plan->n_executors; ++ei) {
    const b2_executor_desc& e = plan->executors[ei];
    if (terminal) { *msg = "executors after Aggregation/TopN are not supported on the device path"; return B2_ERR_UNSUPPORTED; }
    if (projected && e.tp != B2_EXEC_LIMIT) { *msg = "only Limit may follow a Projection on the device path"; return B2_ERR_UNSUPPORTED; }
    if (e.tp == B2_EXEC_SELECTION) {
      for (uint32_t k = 0; k < e.n_conditions; ++k) {
        if (P.n_conds >= MAX_CONDS) { *msg = "too many selection conditions"; return B2_ERR_UNSUPPORTED; }
        if (!lower_expr(e.conditions[k], P, &P.conds[P.n_conds], nullptr, nullptr, nullptr, nullptr, msg)) return B2_ERR_UNSUPPORTED;
        P.n_conds++;
      }
    } else if (e.tp == B2_EXEC_AGGREGATION || e.tp == B2_EXEC_STREAM_AGG) {
      if (e.n_group_by > MAX_GROUP) { *msg = "GROUP BY with more than 4 expressions is not on the device path yet"; return B2_ERR_UNSUPPORTED; }
      if (e.n_aggrs == 0 || e.n_aggrs > MAX_AGGS) { *msg = "0 or too many aggregate functions"; return B2_ERR_UNSUPPORTED; }
      P.mode = PM_AGG; terminal = true;
      schema.clear();
      int acc = 0;
      bool has_first = false;
      for (uint32_t k = 0; k < e.n_aggrs; ++k) {
        DevAgg& g = P.aggs[k];
        int tp; uint32_t flag; uint8_t et, uns;
        const int ak = e.aggrs[k].kind;
        const bool bit_op = ak == B2_AGG_BIT_AND || ak == B2_AGG_BIT_OR || ak == B2_AGG_BIT_XOR;
        if ((ak == B2_AGG_FIRST || bit_op) && e.aggrs[k].arg.n_nodes) {  // (the argument's type: its root node, the last in post-order)
          const int ck = scan_col_kind(e.aggrs[k].arg.nodes[e.aggrs[k].arg.n_nodes - 1].field_tp, 0);
          if (ck >= CK_TIME && ck <= CK_DEC) {
            *msg = ak == B2_AGG_FIRST ? "FIRST over a bytes / JSON / decimal / date-time / duration value is not on the device path yet"
                                      : "BIT_AND / BIT_OR / BIT_XOR over a bytes / JSON / decimal / date-time / duration value (cast to Int) is not supported";
            return B2_ERR_UNSUPPORTED;
          }
        }
        if (!lower_expr(e.aggrs[k].arg, P, &g.arg, &et, &uns, &tp, &flag, msg)) return B2_ERR_UNSUPPORTED;
        g.arg_et = et; g.arg_unsigned = uns;
        if (ak == B2_AGG_FIRST) acc += acc & 1;  // FIRST's [key, value] pair is one 16-byte compare-and-swap
        g.acc_off = (uint8_t)acc;
        switch (e.aggrs[k].kind) {
          case B2_AGG_COUNT: g.kind = AGG_COUNT; acc += 1; break;
          case B2_AGG_SUM: g.kind = AGG_SUM; acc += et ? 1 + F64_ACC_DIGITS : 3; break;  // Real: exact fixed-point accumulator (b2_device.h f64_acc_add)
          case B2_AGG_AVG: g.kind = AGG_AVG; acc += et ? 1 + F64_ACC_DIGITS : 3; break;
          case B2_AGG_MAX: g.kind = AGG_MAX; acc += 2; break;
          case B2_AGG_MIN: g.kind = AGG_MIN; acc += 2; break;
          case B2_AGG_FIRST: g.kind = AGG_FIRST; acc += 2; has_first = true; break;
          case B2_AGG_BIT_AND: g.kind = AGG_BIT_AND; acc += 1; break;
          case B2_AGG_BIT_OR: g.kind = AGG_BIT_OR; acc += 1; break;
          case B2_AGG_BIT_XOR: g.kind = AGG_BIT_XOR; acc += 1; break;
          default: *msg = "aggregate function " + std::to_string(e.aggrs[k].kind) + " is not on the device path yet"; return B2_ERR_UNSUPPORTED;
        }
        if ((g.kind == AGG_SUM || g.kind == AGG_AVG) && !et && tp == B2_TP_BIT) { *msg = "SUM/AVG over BIT (cast to DOUBLE) is not supported"; return B2_ERR_UNSUPPORTED; }
        if (agg_is_bit(g.kind) && et == 1) { *msg = "BIT_AND / BIT_OR / BIT_XOR over a Real value (cast to Int) is not supported"; return B2_ERR_UNSUPPORTED; }
        if (acc > MAX_ACC_WORDS) { *msg = "aggregate state too large"; return B2_ERR_UNSUPPORTED; }
        OutCol cnt = {B2_COL_I64, B2_TP_LONGLONG, B2_FLAG_UNSIGNED | B2_FLAG_NOT_NULL};  // impl_count.rs:35-40
        OutCol sum = et ? OutCol{B2_COL_F64, B2_TP_DOUBLE, 0} : OutCol{B2_COL_DECIMAL, B2_TP_NEWDECIMAL, 0};
        if (g.kind == AGG_COUNT || g.kind == AGG_AVG) schema.push_back(cnt);
        if (g.kind == AGG_SUM || g.kind == AGG_AVG) schema.push_back(sum);
        if (agg_is_extremum(g.kind) || g.kind == AGG_FIRST)  // one column of the argument's own type (impl_max_min.rs:78-84, impl_first.rs AggrFnStateFirst::push_result)
          schema.push_back(OutCol{et ? B2_COL_F64 : B2_COL_I64, tp, flag & ~(uint32_t)B2_FLAG_NOT_NULL});
        if (agg_is_bit(g.kind)) schema.push_back(cnt);  // u64, never NULL (include/b2_copr.h B2_AGG_BIT_AND)
      }
      acc += has_first ? acc & 1 : 0;  // CTA and HBM tables then hold every group's state 16-byte aligned
      if (acc > MAX_ACC_WORDS) { *msg = "aggregate state too large"; return B2_ERR_UNSUPPORTED; }
      P.n_aggs = (int)e.n_aggrs; P.acc_words = acc;
      if (e.n_group_by == 1) {
        int tp; uint32_t flag; uint8_t et, uns;
        if (!lower_expr(e.group_by[0], P, &P.group, &et, &uns, &tp, &flag, msg)) return B2_ERR_UNSUPPORTED;
        P.has_group = 1; P.group_et = et; P.group_unsigned = uns;
        schema.push_back(OutCol{et ? B2_COL_F64 : B2_COL_I64, tp, flag});
      } else if (e.n_group_by > 1) {  // BatchSlowHashAggregation: [aggregates..., group-by columns in order] (slow_hash_aggr_executor.rs:388-420)
        for (uint32_t q = 0; q < e.n_group_by; ++q) {
          int tp; uint32_t flag; uint8_t et, uns;
          if (!lower_expr(e.group_by[q], P, &P.groups[q], &et, &uns, &tp, &flag, msg)) return B2_ERR_UNSUPPORTED;
          P.groups_et[q] = et;
          schema.push_back(OutCol{et ? B2_COL_F64 : B2_COL_I64, tp, flag});
        }
        P.has_group = 1; P.n_group = (int)e.n_group_by;
      }
    } else if (e.tp == B2_EXEC_TOPN) {
      if (e.n_order_by == 0 || e.n_order_by > MAX_ORDER) { *msg = "TopN with 0 or more than 4 order-by expressions"; return B2_ERR_UNSUPPORTED; }
      P.mode = PM_TOPN; terminal = true;
      for (uint32_t k = 0; k < e.n_order_by; ++k) {
        DevOrder& o = P.order[k];
        uint8_t et, uns;
        if (!lower_expr(e.order_by[k].expr, P, &o.e, &et, &uns, nullptr, nullptr, msg)) return B2_ERR_UNSUPPORTED;
        o.desc = e.order_by[k].desc ? 1 : 0; o.et = et; o.is_unsigned = uns;
      }
      if (e.limit > 2048) { *msg = "TopN limit above 2048 is not on the device path yet"; return B2_ERR_UNSUPPORTED; }
      P.n_order = (int)e.n_order_by; P.limit = e.limit;
    } else if (e.tp == B2_EXEC_PROJECTION) {
      if (P.mode != PM_SCAN || P.n_proj) { *msg = "Projection is on the device path only on top of a scan / selection pipeline"; return B2_ERR_UNSUPPORTED; }
      if (e.n_conditions == 0 || e.n_conditions > MAX_PROJ) { *msg = "Projection with 0 or more than 16 expressions"; return B2_ERR_UNSUPPORTED; }
      schema.clear();
      for (uint32_t k = 0; k < e.n_conditions; ++k) {
        int tp; uint32_t flag; uint8_t et, uns;
        if (!lower_expr(e.conditions[k], P, &P.proj[k], &et, &uns, &tp, &flag, msg)) return B2_ERR_UNSUPPORTED;
        schema.push_back(OutCol{et ? B2_COL_F64 : B2_COL_I64, tp, flag});
      }
      P.n_proj = (int)e.n_conditions;
      projected = true;
    } else if (e.tp == B2_EXEC_LIMIT) {
      if (P.mode != PM_SCAN || ei + 1 != plan->n_executors) { *msg = "Limit is on the device path only as the last executor of a scan / selection pipeline"; return B2_ERR_UNSUPPORTED; }
      out->scan_limit = e.limit;
    } else {
      *msg = "executor type " + std::to_string(e.tp) + " is not supported on the device path";
      return B2_ERR_UNSUPPORTED;
    }
  }
  out->schema = schema;
  out->output_offsets.clear();
  if (plan->output_offsets && plan->n_output_offsets) {
    for (uint32_t i = 0; i < plan->n_output_offsets; ++i) {
      if (plan->output_offsets[i] >= schema.size()) { *msg = "output offset out of range"; return B2_ERR_INVALID_ARG; }
      out->output_offsets.push_back(plan->output_offsets[i]);
    }
  } else {
    for (uint32_t i = 0; i < schema.size(); ++i) out->output_offsets.push_back(i);
  }
  if (P.mode == PM_SCAN || P.mode == PM_TOPN) {
    // materialised scan columns must be Int/Real on the device path
    std::vector<uint32_t> mat;
    if (P.mode == PM_TOPN) for (int i = 0; i < P.n_cols; ++i) mat.push_back(i); else mat = out->output_offsets;
    if (mat.size() > MAX_COLS) { *msg = "too many output columns"; return B2_ERR_UNSUPPORTED; }
    for (size_t i = 0; i < mat.size(); ++i) {
      const DevCol& mc = P.cols[mat[i]];
      if (!P.n_proj && mc.kind == CK_OTHER) { *msg = "output column " + std::to_string(mat[i]) + " has a type the device path cannot materialise (TIMESTAMP, ENUM, SET, BIT > 64 ...)"; return B2_ERR_UNSUPPORTED; }
      if (!P.n_proj && mc.kind >= CK_TIME) {
        const b2_column_info& ci = scan.columns[mat[i]];
        if (ci.default_val && ci.default_len && ci.default_val[0] != 0) { *msg = "default value of a non Int/Real output column is not materialised on the device path"; return B2_ERR_UNSUPPORTED; }
        if (ck_is_ref(mc.kind)) {
          if (P.mode == PM_TOPN) { *msg = "TopN over a table with bytes / json / decimal columns is not on the device path yet"; return B2_ERR_UNSUPPORTED; }
          if (out->desc) { *msg = "backward scan with bytes / json / decimal output columns is not on the device path yet"; return B2_ERR_UNSUPPORTED; }
          P.n_raw++;
        }
      }
      P.out_cols[i] = (uint8_t)mat[i];
    }
    P.n_out = (int)mat.size();
    if (P.n_proj) {  // expression outputs: none comes straight from a stored position
      for (int i = 0; i < P.n_out; ++i) P.out_slow[P.n_out_slow++] = (uint8_t)i;
    } else
    // fast rows feed integer outputs straight from their stored position; everything else goes through cell_value
    for (int i = 0; i < P.n_out; ++i) {
      const DevCol& col = P.cols[P.out_cols[i]];
      if (P.fast_n > 0 && col.role == CR_NORMAL && col.kind == CK_INT && P.fast_out[col.v2_hint] < 0) P.fast_out[col.v2_hint] = (int8_t)i;
      else P.out_slow[P.n_out_slow++] = (uint8_t)i;
    }
  }
  // selection conditions of the shape `integer column <cmp> constant` are evaluated by stored position on fast rows
  P.n_fconds = 0;
  if (P.fast_n > 0 && P.n_conds > 0) {
    bool all = true;
    for (int i = 0; i < P.n_conds && all; ++i) {
      const DevExpr ex = P.conds[i];
      all = false;
      if (ex.n != 3) break;
      const DevNode &a = P.nodes[ex.start], &b = P.nodes[ex.start + 1], &f = P.nodes[ex.start + 2];
      if (f.kind != B2_RPN_FN || f.sig < 100 || f.sig >= 160 || f.sig % 10 != 0) break;
      auto is_col = [&](const DevNode& n) { return n.kind == B2_RPN_COLUMN_REF && P.cols[n.imm].role == CR_NORMAL && P.cols[n.imm].kind == CK_INT; };
      auto is_const = [&](const DevNode& n) { return n.kind == B2_RPN_CONST_INT || n.kind == B2_RPN_CONST_UINT; };
      bool col_first;
      if (is_col(a) && is_const(b)) col_first = true;
      else if (is_const(a) && is_col(b)) col_first = false;
      else break;
      const DevNode& cn = col_first ? a : b;
      const DevNode& kn = col_first ? b : a;
      const DevCol& col = P.cols[cn.imm];
      FastCond fc;
      memset(&fc, 0, sizeof(fc));
      fc.imm = kn.imm; fc._p[0] = (uint8_t)(col_first ? 1 : 0) /* which node holds the constant: resolved into imm_slot below */; fc.h = col.v2_hint; fc.col_uns = col.is_unsigned; fc.imm_uns = kn.is_unsigned; fc.zero_ext = col.v2_class != V2_INT;
      int op;  // column on the left
      switch (f.sig) {
        case B2_SIG_LT_INT: op = col_first ? 0 : 2; break;
        case B2_SIG_LE_INT: op = col_first ? 1 : 3; break;
        case B2_SIG_GT_INT: op = col_first ? 2 : 0; break;
        case B2_SIG_GE_INT: op = col_first ? 3 : 1; break;
        case B2_SIG_EQ_INT: op = 4; break;
        default: op = 5; break;
      }
      fc.op = (uint8_t)op;
      P.fconds[i] = fc;
      all = true;
    }
    if (all) P.n_fconds = P.n_conds;
  }
  // stored columns read by expressions: decoded once per row by the lean kernels (Row::cv)
  P.fast_need = 0;
  if (P.fast_n > 0)
    for (int i = 0; i < P.n_nodes; ++i)
      if (P.nodes[i].kind == B2_RPN_COLUMN_REF) {
        const DevCol& c = P.cols[P.nodes[i].imm];
        if (c.role == CR_NORMAL && c.kind == CK_INT) P.fast_need |= 1u << c.v2_hint;
      }
  for (int i = 0; i < P.n_nodes; ++i)
    if (P.nodes[i].kind == B2_RPN_COLUMN_REF && P.cols[P.nodes[i].imm].kind >= CK_BYTES) P.expr_refs = 1;
  // Constants become launch parameters: the device plan keeps only a slot number, so that requests which differ in their
  // literals (`col < 5`, `col < 7`, another IN list, another LIMIT) share one plan shape and one specialised kernel.
  out->n_imms = 0;
  out->pool.swap(lowering_pool());
  lowering_pool().clear();
  for (const PoolRef& r : lowering_pool_refs()) {  // bytes constants first: they must get a slot (their value is an address)
    if (out->n_imms >= MAX_IMMS) { lowering_pool_refs().clear(); *msg = "too many constants for the bytes constants to become launch parameters"; return B2_ERR_UNSUPPORTED; }
    out->pool_imms.push_back(CompiledPlan::PoolImm{out->n_imms, r.off, r.len});
    out->imms[out->n_imms] = 0;
    P.nodes[r.node].sig = ++out->n_imms;
    P.nodes[r.node].imm = 0;
    P.nodes[r.node].n_args = 1;  // (marks the node as placed)
  }
  lowering_pool_refs().clear();
  for (int i = 0; i < P.n_nodes; ++i) {
    DevNode& nd = P.nodes[i];
    if (nd.kind == B2_RPN_CONST_UINT && (nd.et == 4 || nd.et == 5) && nd.n_args == 1) { nd.n_args = 0; continue; }
    if ((nd.kind == B2_RPN_CONST_INT || nd.kind == B2_RPN_CONST_UINT || nd.kind == B2_RPN_CONST_REAL) && out->n_imms < MAX_IMMS) {
      out->imms[out->n_imms] = nd.imm;
      nd.sig = ++out->n_imms;
      nd.imm = 0;
    } else if (nd.kind != B2_RPN_FN) nd.sig = 0;
  }
  for (int i = 0; i < P.n_fconds; ++i) {
    FastCond& fc = P.fconds[i];
    const DevNode& kn = P.nodes[P.conds[i].start + (fc._p[0] ? 1 : 0)];
    fc._p[0] = 0;
    if (kn.sig > 0) { fc.imm_slot = (uint8_t)kn.sig; fc.imm = 0; }
  }
  return B2_OK;
}

// the bytes constants' launch parameters, once the pool sits at `base` (device memory for the kernels, host memory for the
// host build of the device logic)
inline void patch_pool_imms(CompiledPlan& cp, const uint8_t* base) {
  for (const CompiledPlan::PoolImm& r : cp.pool_imms) cp.imms[r.slot] = (int64_t)raw_ref_make(base + r.off, r.len);
}

// memcomparable encoding of a raw key (tikv_util/src/codec/bytes.rs:25-55), for range bounds
inline std::vector<uint8_t> encode_memcomparable(const uint8_t* p, size_t n) {
  std::vector<uint8_t> out;
  size_t idx = 0;
  while (idx <= n) {
    size_t remain = n - idx, pad = 0;
    if (remain >= 8) out.insert(out.end(), p + idx, p + idx + 8);
    else { pad = 8 - remain; out.insert(out.end(), p + idx, p + n); out.insert(out.end(), pad, 0); }
    out.push_back((uint8_t)(0xff - pad));
    idx += 8;
  }
  return out;
}

}  // namespace b2
