// Host only: a DevPlan as a C++ aggregate initialiser, for kernels specialised on one plan (constexpr DevPlan).
// Field order must follow the declarations in b2_device.h exactly; `plan_literal_check` (engine) compares sizes.
#pragma once
#include <sstream>
#include <string>

#include "b2_device.h"

namespace b2 {

inline std::string plan_literal(const DevPlan& P) {
  std::ostringstream o;
  auto u64 = [&](uint64_t v) { o << v << "ull"; };
  auto i64 = [&](int64_t v) { if (v == INT64_MIN) o << "(-9223372036854775807ll - 1)"; else o << v << "ll"; };
  auto expr = [&](const DevExpr& e) { o << "{" << e.start << "," << e.n << "}"; };
  o << "{";
  o << P.mode << "," << P.n_cols << "," << P.n_nodes << "," << P.n_conds << "," << P.n_aggs << "," << P.has_group << "," << P.acc_words << ","
    << P.n_order << "," << P.n_out << "," << P.isolation << "," << P.need_value << "," << P.has_handle_cols << "," << P.fast_n << "," << P.idx_cols << ",";
  u64(P.fast_filled); o << "," << P.fast_cls << "u," << P.fast_uns << "u,{";
  for (int i = 0; i < 8; ++i) o << (int)P.fast_out[i] << (i < 7 ? "," : "");
  o << "}," << P.n_out_slow << "," << P.fast_need << "u," << P.fast_v1 << ",";
  u64(P.fast_ids); o << ","; u64(0 /* read_ts stays a launch parameter */); o << ","; u64(0 /* so does the TopN limit (ScanArgs::limit) */); o << ",{";
  for (int i = 0; i < MAX_CONDS; ++i) { expr(P.conds[i]); o << (i < MAX_CONDS - 1 ? "," : ""); }
  o << "},"; expr(P.group);
  o << "," << (int)P.group_et << "," << (int)P.group_unsigned << "," << (int)P.topn_all_keys << "," << (int)P._p1 << ",{";
  for (int i = 0; i < MAX_AGGS; ++i) {
    const DevAgg& a = P.aggs[i];
    o << "{"; expr(a.arg); o << "," << (int)a.kind << "," << (int)a.arg_et << "," << (int)a.arg_unsigned << "," << (int)a.acc_off << "}" << (i < MAX_AGGS - 1 ? "," : "");
  }
  o << "},{";
  for (int i = 0; i < MAX_ORDER; ++i) {
    const DevOrder& d = P.order[i];
    o << "{"; expr(d.e); o << "," << (int)d.desc << "," << (int)d.et << "," << (int)d.is_unsigned << "," << (int)d._pad << "}" << (i < MAX_ORDER - 1 ? "," : "");
  }
  o << "},{";
  for (int i = 0; i < MAX_COLS; ++i) o << (int)P.out_cols[i] << (i < MAX_COLS - 1 ? "," : "");
  o << "},{";
  for (int i = 0; i < MAX_COLS; ++i) o << (int)P.out_slow[i] << (i < MAX_COLS - 1 ? "," : "");
  o << "}," << P.n_fconds << "," << P.n_raw << ",{";
  for (int i = 0; i < MAX_CONDS; ++i) {
    const FastCond& f = P.fconds[i];
    o << "{"; i64(f.imm); o << "," << (int)f.h << "," << (int)f.op << "," << (int)f.col_uns << "," << (int)f.imm_uns << "," << (int)f.zero_ext << "," << (int)f.imm_slot << ",{0,0}}" << (i < MAX_CONDS - 1 ? "," : "");
  }
  o << "}," << P.n_proj << "," << P.expr_refs << ",{";
  for (int i = 0; i < MAX_PROJ; ++i) { expr(P.proj[i]); o << (i < MAX_PROJ - 1 ? "," : ""); }
  o << "}," << P.n_group << "," << P._gpad << ",{";
  for (int i = 0; i < MAX_GROUP; ++i) { expr(P.groups[i]); o << (i < MAX_GROUP - 1 ? "," : ""); }
  o << "},{";
  for (int i = 0; i < MAX_GROUP; ++i) o << (int)P.groups_et[i] << (i < MAX_GROUP - 1 ? "," : "");
  o << "},{";
  for (int i = 0; i < MAX_COLS; ++i) {
    const DevCol& c = P.cols[i];
    o << "{"; i64(c.col_id); o << ","; i64(c.default_bits);
    o << "," << (int)c.kind << "," << (int)c.role << "," << (int)c.is_unsigned << "," << (int)c.not_null << "," << (int)c.tp << "," << (int)c.v2_class << "," << (int)c.def_state << ","
      << (int)c.v2_hint << "," << (int)c.fsp << ",{0,0,0,0,0,0,0}}" << (i < MAX_COLS - 1 ? "," : "");
  }
  o << "},{";
  for (int i = 0; i < MAX_NODES; ++i) {
    const DevNode& n = P.nodes[i];
    o << "{" << n.sig << "," << (int)n.kind << "," << (int)n.n_args << "," << (int)n.et << "," << (int)n.is_unsigned << ","; i64(n.imm); o << "}" << (i < MAX_NODES - 1 ? "," : "");
  }
  o << "}}";
  return o.str();
}

}  // namespace b2
