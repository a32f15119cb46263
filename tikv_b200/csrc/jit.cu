// Plan-specialised scan kernels, compiled at run time.
//
// The generic scan_kernel<MODE> interprets the device plan (DevPlan in a __grid_constant__ parameter): column tables,
// RPN nodes, fast-path tables are all run-time data.  A pushed-down DAG repeats for thousands of regions, so the plan
// is worth compiling once: this file builds a translation unit  "constant DevPlan literal + scan_body<MODE>"  with
// NVRTC (sm_90a cubin), loads it through the driver API and caches the function per (device, plan).  With the plan a
// compile-time constant the column loops unroll, dead paths (v1 datums, unused roles, the RPN stack machine, unused
// modes) disappear and the hot loop shrinks by about a third (DESIGN.md §5).
//
// libnvrtc / libcuda are dlopen'ed: the library keeps loading (and the generic kernels keep working) where they are
// absent.  The kernel sources are read from ../csrc relative to this shared object.
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nvrtc.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <future>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "jit.h"
#include "plan_literal.h"

namespace b2 {

enum { FK_THREADS_HOST = TILE + 32 };  // fast_kernel.cuh FK_THREADS (device header, not included here)

namespace {

struct Api {
  bool ok = false;
  std::string why;
  // nvrtc
  nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
  nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
  nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
  nvrtcResult (*GetProgramLog)(nvrtcProgram, char*) = nullptr;
  nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
  nvrtcResult (*GetCUBIN)(nvrtcProgram, char*) = nullptr;
  nvrtcResult (*DestroyProgram)(nvrtcProgram*) = nullptr;
  // driver
  CUresult (*ModuleLoadData)(CUmodule*, const void*) = nullptr;
  CUresult (*ModuleGetFunction)(CUfunction*, CUmodule, const char*) = nullptr;
  CUresult (*FuncSetAttribute)(CUfunction, CUfunction_attribute, int) = nullptr;
  CUresult (*OccupancyMaxActiveBlocksPerMultiprocessor)(int*, CUfunction, int, size_t) = nullptr;
  CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void**, void**) = nullptr;
  std::string csrc_dir, cuda_inc;
  bool rtc_ok = false;          // NVRTC + kernel sources: enough to compile into the on-disk cache (no GPU needed)
  std::string cache_dir;        // compiled cubins, keyed by (plan shape, kernel sources, compiler options)
  std::string build_cache_dir;  // the library's own jit_cache (filled at build time): also searched, never written when
                                // B2_JIT_CACHE_DIR points elsewhere (the installed tree may be read-only)
  unsigned long long src_hash = 0;
};

unsigned long long fnv1a(const void* p, size_t n, unsigned long long h = 1469598103934665603ull) {
  const unsigned char* c = (const unsigned char*)p;
  for (size_t i = 0; i < n; ++i) { h ^= c[i]; h *= 1099511628211ull; }
  return h;
}
bool read_file(const std::string& path, std::string* out) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  char buf[65536];
  size_t n;
  out->clear();
  while ((n = fread(buf, 1, sizeof(buf), f)) > 0) out->append(buf, n);
  fclose(f);
  return true;
}

template <class F>
bool sym(void* lib, const char* name, F* out) {
  *out = reinterpret_cast<F>(dlsym(lib, name));
  return *out != nullptr;
}

Api& api() {
  static Api a;
  static std::once_flag once;
  std::call_once(once, [] {
    void* rtc = nullptr;
    for (const char* n : {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so"})
      if ((rtc = dlopen(n, RTLD_NOW | RTLD_GLOBAL))) break;
    void* drv = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!rtc) { a.why = "libnvrtc not found"; return; }
    bool ok = sym(rtc, "nvrtcCreateProgram", &a.CreateProgram) && sym(rtc, "nvrtcCompileProgram", &a.CompileProgram) &&
              sym(rtc, "nvrtcGetProgramLogSize", &a.GetProgramLogSize) && sym(rtc, "nvrtcGetProgramLog", &a.GetProgramLog) &&
              sym(rtc, "nvrtcGetCUBINSize", &a.GetCUBINSize) && sym(rtc, "nvrtcGetCUBIN", &a.GetCUBIN) && sym(rtc, "nvrtcDestroyProgram", &a.DestroyProgram);
    if (!ok) { a.why = "nvrtc entry point missing"; return; }
    Dl_info info;
    if (!dladdr(reinterpret_cast<void*>(static_cast<bool (*)(std::string*)>(&jit_available)), &info) || !info.dli_fname) { a.why = "cannot locate the shared object"; return; }
    std::string so = info.dli_fname;
    size_t slash = so.rfind('/');
    std::string dir = slash == std::string::npos ? "." : so.substr(0, slash);
    a.csrc_dir = dir + "/../csrc";
    // the sources a specialised kernel is built from: their content is part of the cache key
    unsigned long long h = 1469598103934665603ull;
    for (const char* f : {"/scan_kernel.cuh", "/fast_kernel.cuh", "/kernels.cuh", "/b2_device.h", "/../../include/b2_copr.h"}) {
      std::string text;
      if (!read_file(a.csrc_dir + f, &text)) { a.why = std::string("kernel sources not found next to the library (") + a.csrc_dir + f + ")"; return; }
      h = fnv1a(text.data(), text.size(), h);
    }
    a.src_hash = h;
    const char* cd = getenv("B2_JIT_CACHE_DIR");
    a.build_cache_dir = dir + "/jit_cache";
    a.cache_dir = cd && *cd ? std::string(cd) : a.build_cache_dir;
    a.rtc_ok = true;
    if (!drv) { a.why = "libcuda.so.1 not found"; return; }
    ok = sym(drv, "cuModuleLoadData", &a.ModuleLoadData) && sym(drv, "cuModuleGetFunction", &a.ModuleGetFunction) &&
         sym(drv, "cuFuncSetAttribute", &a.FuncSetAttribute) &&
         sym(drv, "cuOccupancyMaxActiveBlocksPerMultiprocessor", &a.OccupancyMaxActiveBlocksPerMultiprocessor) && sym(drv, "cuLaunchKernel", &a.LaunchKernel);
    if (!ok) { a.why = "driver entry point missing"; return; }
    a.ok = true;
  });
  return a;
}

struct Entry {
  std::shared_future<JitKernel*> fut;
};
std::mutex g_mu;
// leaked on purpose: a static destructor would block process exit on compilations still in flight
std::map<std::string, Entry>& g_cache = *new std::map<std::string, Entry>();

// What a plan-specialised kernel is compiled from: the plan without its launch parameters (ScanArgs carries those) and the
// variant it needs
struct JitSpec {
  std::string literal;
  int mode;       // scan_body<mode>
  bool ext_sigs;  // the rarer scalar functions (b2_device.h)
  int fast;       // bit 0: the lean kernel too, bit 1: table scan (no index-row decoder)
};
JitSpec jit_spec(const DevPlan& plan) {
  DevPlan p = plan;
  p.read_ts = 0; p.isolation = 0; p.limit = 0;
  return JitSpec{plan_literal(p), scan_kernel_mode(plan), plan_uses_ext_sigs(plan), (plan_has_fast_kernel(plan) ? 1 : 0) | (plan.idx_cols == 0 ? 2 : 0)};
}

// ---- on-disk cache of compiled cubins ------------------------------------------------------------------------------
// One file per (plan shape, kernel instantiation, compiler options, kernel sources): <dir>/<hash>.cubin plus <hash>.key
// holding the full key (a hash collision or a stale file is detected by comparing it).  Written atomically (rename).
std::atomic<unsigned long long> g_nvrtc_compiles{0}, g_cache_hits{0};
std::string cache_key(const JitSpec& j) {
  return "b2jit6|sm_90a|mode" + std::to_string(j.mode) + "|ext" + std::to_string((int)j.ext_sigs) + "|fast" + std::to_string(j.fast) + "|src" + std::to_string(api().src_hash) + "|" + j.literal;
}
std::string cache_path(const std::string& key, const std::string& dir = api().cache_dir) {
  char name[32];
  snprintf(name, sizeof(name), "%016llx", fnv1a(key.data(), key.size()));
  return dir + "/" + name;
}
bool cache_load(const std::string& key, std::vector<char>* cubin) {
  for (const std::string* dir : {&api().cache_dir, &api().build_cache_dir}) {
    std::string path = cache_path(key, *dir), k, c;
    if (!read_file(path + ".key", &k) || k != key || !read_file(path + ".cubin", &c) || c.empty()) continue;
    cubin->assign(c.begin(), c.end());
    return true;
  }
  return false;
}
void cache_store(const std::string& key, const std::vector<char>& cubin) {
  mkdir(api().cache_dir.c_str(), 0755);
  std::string path = cache_path(key), tmp = path + ".tmp" + std::to_string((long)getpid()) + "." + std::to_string((unsigned long long)(uintptr_t)&cubin);
  for (int pass = 0; pass < 2; ++pass) {
    const std::string dst = path + (pass ? ".key" : ".cubin");
    FILE* f = fopen(tmp.c_str(), "wb");
    if (!f) return;
    const char* p = pass ? key.data() : cubin.data();
    size_t n = pass ? key.size() : cubin.size();
    bool ok = fwrite(p, 1, n, f) == n;
    ok = fclose(f) == 0 && ok;
    if (!ok || rename(tmp.c_str(), dst.c_str()) != 0) { remove(tmp.c_str()); return; }
  }
}

// NVRTC only (no CUDA context): plan literal -> sm_90a cubin
bool compile_cubin(const JitSpec& j, std::vector<char>* cubin, std::string* error) {
  Api& a = api();
  std::string defs;
  if (j.fast & 2) defs += "#define B2_NO_IDX 1\n";  // a table scan's kernel carries none of the index-row decoder
  // Plans with the rarer scalar functions (wide projections over DIV / MOD / CASE ...) compile several times faster with the
  // general-path decoders out of line; everything else keeps them inline, on the hot path of the common plans
  if (j.ext_sigs) defs += "#define B2_COLD_OUTLINE 1\n";
  std::string src = defs + "#define B2_NVRTC 1\n#define B2_JIT_PLAN 1\n#include \"fast_kernel.cuh\"\nnamespace b2 { __constant__ const DevPlan kJitPlan =\n" + j.literal +
                    ";\n}\nextern \"C\" __global__ void __launch_bounds__(b2::TILE + 64, 2) b2_scan_jit(const __grid_constant__ b2::ScanArgs A) {\n"
                    "  b2::scan_body<" + std::to_string(j.mode) + ">(b2::kJitPlan, A);\n}\n";
  if (j.fast & 1)
    src += "extern \"C\" __global__ void __launch_bounds__(b2::FK_THREADS, 3) b2_fast_jit(const __grid_constant__ b2::ScanArgs A) {\n"
           "  b2::fast_body<" + std::to_string(j.mode) + ">(b2::kJitPlan, A);\n}\n";
  if (j.mode == PM_TOPN)  // the limit is a launch parameter: every TopN module also carries the large-limit variant
    src += "extern \"C\" __global__ void __launch_bounds__(b2::TILE + 64, 2) b2_scan_topn_hbm_jit(const __grid_constant__ b2::ScanArgs A) {\n"
           "  b2::scan_body<" + std::to_string(j.mode) + ", true>(b2::kJitPlan, A);\n}\n";
  nvrtcProgram prog;
  if (a.CreateProgram(&prog, src.c_str(), "b2_scan_jit.cu", 0, nullptr, nullptr) != NVRTC_SUCCESS) { *error = "nvrtcCreateProgram failed"; return false; }
  std::string inc = "-I" + a.csrc_dir;
  const char* opts[] = {"--gpu-architecture=sm_90a", "--std=c++17", "-lineinfo", "-DB2_NVRTC=1", "-default-device", inc.c_str(), "-I/usr/local/cuda/include",
                        j.ext_sigs ? "-DB2_EXT_SIGS=1" : "-DB2_EXT_SIGS=0", "--split-compile=0"};
  nvrtcResult rc = a.CompileProgram(prog, (int)(sizeof(opts) / sizeof(opts[0])), opts);
  g_nvrtc_compiles++;
  if (rc != NVRTC_SUCCESS) {
    size_t n = 0;
    a.GetProgramLogSize(prog, &n);
    std::string log(n, 0);
    if (n) a.GetProgramLog(prog, &log[0]);
    *error = "nvrtc: " + log.substr(0, 2000);
    a.DestroyProgram(&prog);
    return false;
  }
  size_t n = 0;
  a.GetCUBINSize(prog, &n);
  cubin->resize(n);
  a.GetCUBIN(prog, cubin->data());
  a.DestroyProgram(&prog);
  return true;
}

JitKernel* compile(int device, const JitSpec& j) {
  Api& a = api();
  JitKernel* k = new JitKernel();
  cudaSetDevice(device);
  cudaFree(nullptr);  // make sure the primary context exists and is current on this thread
  const std::string key = cache_key(j);
  std::vector<char> cubin;
  if (cache_load(key, &cubin)) g_cache_hits++;
  else {
    if (!compile_cubin(j, &cubin, &k->error)) return k;
    cache_store(key, cubin);
  }
  CUmodule mod;
  if (a.ModuleLoadData(&mod, cubin.data()) != CUDA_SUCCESS) { k->error = "cuModuleLoadData failed"; return k; }
  CUfunction fn;
  if (a.ModuleGetFunction(&fn, mod, "b2_scan_jit") != CUDA_SUCCESS) { k->error = "kernel symbol missing"; return k; }
  k->fn = fn;
  if (j.fast & 1) {
    CUfunction ff;
    if (a.ModuleGetFunction(&ff, mod, "b2_fast_jit") != CUDA_SUCCESS) { k->error = "lean kernel symbol missing"; return k; }
    k->fn_fast = ff;
  }
  if (j.mode == PM_TOPN) {
    CUfunction fh;
    if (a.ModuleGetFunction(&fh, mod, "b2_scan_topn_hbm_jit") != CUDA_SUCCESS) { k->error = "large-limit TopN kernel symbol missing"; return k; }
    k->fn_topn_hbm = fh;
  }
  k->ok = true;
  return k;
}

}  // namespace

bool jit_available(std::string* why) {
  Api& a = api();
  if (!a.ok && why) *why = a.why;
  return a.ok;
}

// Compilations still in flight when the process exits are waited for (this handler is registered after the CUDA runtime's
// own teardown, so it runs before it): a compile thread must not touch a runtime that is being destroyed.
static void jit_wait_all_at_exit() {
  std::vector<std::shared_future<JitKernel*>> pending;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    for (auto& kv : g_cache) pending.push_back(kv.second.fut);
  }
  for (auto& f : pending) f.wait();
}

std::shared_future<JitKernel*> jit_get(int device, const DevPlan& plan) {
  static std::once_flag at_exit_once;
  std::call_once(at_exit_once, [] { std::atexit(jit_wait_all_at_exit); });
  JitSpec j = jit_spec(plan);
  std::string key = std::to_string(device) + "|" + j.literal;
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_cache.find(key);
  if (it != g_cache.end()) return it->second.fut;
  std::shared_future<JitKernel*> fut = std::async(std::launch::async, [device, j] { return compile(device, j); }).share();
  g_cache[key].fut = fut;
  return fut;
}

bool plan_has_fast_kernel(const DevPlan& plan) {
  if (plan.fast_n <= 0 || plan.expr_refs) return false;  // (the lean kernels do not track a row's HBM address: LIKE / Decimal operands need it)
  if (plan.mode == PM_TOPN) return true;
  if (plan.mode != PM_AGG || plan.n_group > 1) return false;
  for (int a = 0; a < plan.n_aggs; ++a)
    if ((plan.aggs[a].kind == 1 || plan.aggs[a].kind == 2) && plan.aggs[a].arg_et == 1) return false;  // exact Real sums: 67 words per group
  return true;
}

// Compile the kernel of `plan` into the on-disk cache without touching a GPU (build machines, ahead-of-time warm-up).
// 0 = compiled now, 1 = was cached already, negative = failure (message in *error).
int jit_precompile(const DevPlan& plan, std::string* error) {
  Api& a = api();
  if (!a.rtc_ok) { *error = a.why; return -1; }
  const JitSpec j = jit_spec(plan);
  const std::string key = cache_key(j);
  std::vector<char> cubin;
  if (cache_load(key, &cubin)) return 1;
  if (!compile_cubin(j, &cubin, error)) return -1;
  cache_store(key, cubin);
  return 0;
}
void jit_counters(unsigned long long* nvrtc_compiles, unsigned long long* disk_hits) { *nvrtc_compiles = g_nvrtc_compiles.load(); *disk_hits = g_cache_hits.load(); }

static CUfunction entry_fn(const JitKernel* k, JitEntry e) { return (CUfunction)(e == JIT_FAST ? k->fn_fast : e == JIT_TOPN_HBM ? k->fn_topn_hbm : k->fn); }
static size_t& entry_smem(const JitKernel* k, JitEntry e) { return e == JIT_FAST ? k->max_dyn_smem_fast : e == JIT_TOPN_HBM ? k->max_dyn_smem_topn_hbm : k->max_dyn_smem; }

int jit_max_blocks_per_sm(const JitKernel* k, size_t smem, JitEntry entry) {
  int n = 0;
  const bool fast = entry == JIT_FAST;
  CUfunction fn = entry_fn(k, entry);
  size_t& lim = entry_smem(k, entry);
  if (smem > lim) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (smem > lim && api().FuncSetAttribute(fn, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem) == CUDA_SUCCESS) lim = smem;
  }
  if (api().OccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, fast ? (int)FK_THREADS_HOST : TILE + 64, smem) != CUDA_SUCCESS || n < 1) n = 1;
  return n;
}

cudaError_t jit_launch(const JitKernel* k, const ScanArgs& a, int grid, size_t smem, cudaStream_t s, JitEntry entry) {
  if (a.c_hi <= a.c_lo) return cudaSuccess;
  uint32_t n_tiles = (a.c_hi - a.c_lo + TILE - 1) / TILE;
  if ((uint32_t)grid > n_tiles) grid = (int)n_tiles;
  void* params[] = {const_cast<ScanArgs*>(&a)};
  const bool fast = entry == JIT_FAST;
  CUfunction fn = entry_fn(k, entry);
  size_t& lim = entry_smem(k, entry);
  if (smem > lim) {  // opt in to large dynamic shared memory (the limit excludes the kernel's static part)
    std::lock_guard<std::mutex> lk(g_mu);
    if (smem > lim) {
      if (api().FuncSetAttribute(fn, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem) != CUDA_SUCCESS) return cudaErrorInvalidValue;
      lim = smem;
    }
  }
  CUresult rc = api().LaunchKernel(fn, (unsigned)grid, 1, 1, fast ? (unsigned)FK_THREADS_HOST : TILE + 64, 1, 1, (unsigned)smem, (CUstream)s, params, nullptr);
  if (rc != CUDA_SUCCESS) fprintf(stderr, "b2copr: cuLaunchKernel of the plan-specialised kernel failed: CUresult %d\n", (int)rc);
  return rc == CUDA_SUCCESS ? cudaSuccess : cudaErrorLaunchFailure;
}

}  // namespace b2
