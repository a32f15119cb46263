// TEST HARNESS (not product, not oracle): the FIRST / BIT_AND / BIT_OR / BIT_XOR state code of tikv_b200/csrc/b2_device.h
// driven on the CPU.  A plan is lowered by plan_compile.h (so the state layout is the device's: acc_off, padding,
// acc_words), rows are folded into per-part states by first_bit_update, the parts are merged word by word as
// agg_word_op says (the kernels' CTA flushes and b2_exec_agg_word_ops), and the results are read by first_bit_result
// (agg_result_kernel).  The rows come from the oracle's scan, in scan order; tests/test_first_bit_emul_cpu.py compares
// the answers with the reference semantics.
#include <cstring>
#include <string>
#include <vector>

#include "../tikv_b200/csrc/plan_compile.h"

using namespace b2;

extern "C" {

// Rows i = 0 .. n_rows-1 in scan order: group[i], and per aggregate a: bits[i * n_aggs + a], has[i * n_aggs + a] (0 =
// NULL).  A row's block entry is i forward and n_rows-1-i backward (entries fall in a backward scan).  Row i is folded
// into part (i / part_rows) % n_parts, the way tiles are spread over CTAs; the parts are merged last to first.  Output
// per group g and FIRST / BIT_* aggregate a: out[g * n_aggs + a], nonnull[...].  Returns 0, or -1 with the plan's refusal
// message, or -2 when the plan's state layout breaks FIRST's 16-byte alignment.
int fbe_run(const b2_dag_plan* plan, int desc, uint32_t n_rows, uint32_t part_rows, uint32_t n_parts, const uint32_t* group,
            const uint64_t* bits, const uint8_t* has, uint32_t n_groups, uint64_t* out, uint8_t* nonnull, char* msg, size_t msg_len) {
  CompiledPlan cp;
  std::string m;
  if (compile_plan(plan, &cp, &m) != B2_OK) { snprintf(msg, msg_len, "%s", m.c_str()); return -1; }
  const DevPlan& P = cp.dev;
  const size_t W = (size_t)P.acc_words;
  for (int a = 0; a < P.n_aggs; ++a)
    if (P.aggs[a].kind == AGG_FIRST && ((P.aggs[a].acc_off & 1) || (W & 1))) return -2;
  std::vector<uint64_t> parts((size_t)n_parts * n_groups * W, 0);
  for (uint32_t i = 0; i < n_rows; ++i) {
    const uint32_t p = (i / part_rows) % n_parts;
    uint64_t* s = &parts[((size_t)p * n_groups + group[i]) * W];
    const uint64_t entry = desc ? n_rows - 1 - i : i;
    for (int a = 0; a < P.n_aggs; ++a) {
      const DevAgg& g = P.aggs[a];
      if (g.kind == AGG_FIRST || agg_is_bit(g.kind)) first_bit_update(g.kind, s + g.acc_off, entry, desc != 0, has[(size_t)i * P.n_aggs + a] != 0, bits[(size_t)i * P.n_aggs + a]);
    }
  }
  std::vector<uint64_t> total((size_t)n_groups * W, 0);
  for (int p = (int)n_parts - 1; p >= 0; --p)
    for (uint32_t gi = 0; gi < n_groups; ++gi) {
      const uint64_t* src = &parts[((size_t)p * n_groups + gi) * W];
      uint64_t* dst = &total[(size_t)gi * W];
      for (size_t w = 0; w < W; ++w) {
        switch (agg_word_op(P, (int)w)) {
          case B2_MERGE_OR: dst[w] |= src[w]; break;
          case B2_MERGE_XOR: dst[w] ^= src[w]; break;
          case B2_MERGE_MAX: dst[w] = src[w] > dst[w] ? src[w] : dst[w]; break;
          case B2_MERGE_FIRST_KEY: if (src[w] > dst[w]) { dst[w] = src[w]; dst[w + 1] = src[w + 1]; } break;
          case B2_MERGE_FIRST_VALUE: break;  // (moves with its key)
          default: dst[w] += src[w];
        }
      }
    }
  for (uint32_t gi = 0; gi < n_groups; ++gi)
    for (int a = 0; a < P.n_aggs; ++a) {
      const DevAgg& g = P.aggs[a];
      if (g.kind == AGG_FIRST || agg_is_bit(g.kind))
        nonnull[(size_t)gi * P.n_aggs + a] = first_bit_result(g.kind, &total[(size_t)gi * W + g.acc_off], &out[(size_t)gi * P.n_aggs + a]) ? 1 : 0;
    }
  return 0;
}

}  // extern "C"
