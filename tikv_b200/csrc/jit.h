// Run-time compiled, plan-specialised scan kernels (jit.cu).
#pragma once
#include <cuda_runtime.h>

#include <future>
#include <string>

#include "kernels.cuh"

namespace b2 {

struct JitKernel {
  bool ok = false;
  void* fn = nullptr;  // CUfunction: scan_body specialised for the plan
  mutable size_t max_dyn_smem = 48 * 1024;  // dynamic shared memory the function has been opted in to
  void* fn_fast = nullptr;  // CUfunction: fast_body (fast_kernel.cuh) for the order-free pipelines it covers, else null
  mutable size_t max_dyn_smem_fast = 48 * 1024;
  void* fn_topn_hbm = nullptr;  // CUfunction: TopN plans, scan_body with the candidate buffers in HBM (LIMIT above 2048)
  mutable size_t max_dyn_smem_topn_hbm = 48 * 1024;
  std::string error;
};
enum JitEntry { JIT_SCAN, JIT_FAST, JIT_TOPN_HBM };  // fn, fn_fast, fn_topn_hbm

// NVRTC, the driver API and the kernel sources are all reachable from this process?
bool jit_available(std::string* why = nullptr);
// Starts (or joins) the compilation of the kernel specialised for `plan` on `device`; never blocks.
std::shared_future<JitKernel*> jit_get(int device, const DevPlan& plan);
// NVRTC only, no GPU: compile `plan`'s kernel into the on-disk cache (0 compiled, 1 already cached, < 0 failed)
int jit_precompile(const DevPlan& plan, std::string* error);
// process-wide: NVRTC compilations run, kernels served from the on-disk cache
void jit_counters(unsigned long long* nvrtc_compiles, unsigned long long* disk_hits);
int jit_max_blocks_per_sm(const JitKernel* k, size_t smem, JitEntry entry = JIT_SCAN);
cudaError_t jit_launch(const JitKernel* k, const ScanArgs& a, int grid, size_t smem, cudaStream_t s, JitEntry entry = JIT_SCAN);
// does fast_body cover this plan?  (aggregation by at most one expression without Real sums, TopN)
bool plan_has_fast_kernel(const DevPlan& plan);

}  // namespace b2
