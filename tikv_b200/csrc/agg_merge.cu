// Final merge of gathered partial aggregation tables (b2_agg_merge, engine.cu): rows of `key_words` key words, a NULL
// mask byte and `acc_words` state words are grouped by (NULL mask, key words) and each group's words are reduced with
// their B2_MERGE_* op.  The groups come out in the order torch.unique(dim=0) gives them -- ascending by the NULL mask, then by
// the key words as signed int64 -- and no op depends on the order of its operands (FIRST breaks ties by input order), so
// the result equals the torch merge of dist.py bit for bit.
//
// Order: stable LSD radix sorts of the row indices, by the last key word first and by the NULL mask last (cub sorts
// int64 keys in signed order).  Groups: a head flag per sorted row, an inclusive scan of the flags, the first sorted row
// of every group.  Reduce: one warp per group over its rows in sorted order, which is input order within the group.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "kernels.cuh"

namespace b2 {

namespace {

// key word `word` (or the NULL mask, word == key_words) of the rows in the order of `perm`; perm == nullptr: input order,
// and `perm_out` receives that order
__global__ void agg_merge_gather_kernel(AggMergeArgs a, uint32_t word, const unsigned int* perm, unsigned int* perm_out, long long* keys_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  unsigned int r = i;
  if (perm) r = perm[i];
  else perm_out[i] = i;
  long long v;
  if (word == a.key_words) v = a.key_null[r];
  else if (a.key_words == 1 && a.key_null[r]) v = 0;  // one key word: a NULL row's key bits do not count
  else v = a.keys[(size_t)r * a.keys_stride + word];
  keys_out[i] = v;
}

__device__ __forceinline__ bool agg_merge_same_ident(const AggMergeArgs& a, unsigned int r, unsigned int q) {
  if (a.key_null[r] != a.key_null[q]) return false;
  if (a.key_words == 1 && a.key_null[r]) return true;
  for (uint32_t k = 0; k < a.key_words; ++k)
    if (a.keys[(size_t)r * a.keys_stride + k] != a.keys[(size_t)q * a.keys_stride + k]) return false;
  return true;
}

// flags[i] = 1 when sorted row i starts a group
__global__ void agg_merge_heads_kernel(AggMergeArgs a, const unsigned int* perm, unsigned int* flags) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  flags[i] = i == 0 || !agg_merge_same_ident(a, perm[i], perm[i - 1]);
}

// gid: inclusive sums of the head flags (group id + 1).  starts[g] = first sorted row of group g, starts[n_groups] = n
__global__ void agg_merge_starts_kernel(const unsigned int* gid, uint32_t n, unsigned int* starts, unsigned int* n_groups) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned int g = gid[i];
  if (g != (i ? gid[i - 1] : 0u)) starts[g - 1] = i;
  if (i == n - 1) { starts[g] = n; *n_groups = g; }
}

__device__ __forceinline__ uint32_t agg_merge_part_of(const unsigned long long* part_offs, uint32_t n_parts, unsigned int r) {
  uint32_t lo = 0, hi = n_parts;  // largest p with part_offs[p] <= r
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (part_offs[mid] <= r) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ unsigned long long agg_merge_op(unsigned char op, unsigned long long x, unsigned long long y) {
  if (op == B2_MERGE_ADD) return x + y;
  if (op == B2_MERGE_MAX) return x > y ? x : y;
  if (op == B2_MERGE_OR) return x | y;
  return x ^ y;
}

// One warp per group (grid-stride): the lanes stride over the group's sorted rows and the words reduce across the warp.
// ADD (modulo 2^64), MAX, OR and XOR do not depend on the order of their operands; FIRST picks the row of largest
// (part preference, unsigned key, sorted position), so a tie inside a part goes to the last such row in input order.
__global__ void agg_merge_reduce_kernel(AggMergeArgs a, const unsigned int* perm, const unsigned int* starts, const unsigned int* n_groups) {
  const uint32_t lane = threadIdx.x & 31, n_warps = gridDim.x * blockDim.x / 32, ng = *n_groups;
  for (uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) / 32; g < ng; g += n_warps) {
    const uint32_t lo = starts[g], hi = starts[g + 1];
    if (lane == 0) {
      const long long* first = a.keys + (size_t)perm[lo] * a.keys_stride;
      const unsigned char mask = a.key_null[perm[lo]];
      for (uint32_t k = 0; k < a.key_words; ++k) a.out_keys[(size_t)g * a.key_words + k] = (a.key_words == 1 && mask != 0) ? 0 : first[k];
      a.out_null[g] = mask;
    }
    long long* out = a.out_acc + (size_t)g * a.acc_words;
    for (uint32_t w = 0; w < a.acc_words; ++w) {
      const long long* col = a.acc + w;
      const unsigned char op = a.ops[w];
      if (op == B2_MERGE_FIRST_VALUE) continue;  // written with its key word
      if (op == B2_MERGE_FIRST_KEY) {
        // preference: the earliest part holding a nonzero key wins, the latest when desc
        uint32_t has = 0, pref = 0, pos = 0;
        unsigned long long key = 0;
        for (uint32_t j = lo + lane; j < hi; j += 32) {
          const unsigned long long k = (unsigned long long)col[(size_t)perm[j] * a.acc_stride];
          if (k == 0) continue;
          const uint32_t p = agg_merge_part_of(a.part_offs, a.n_parts, perm[j]), pr = a.desc ? p : a.n_parts - 1 - p;
          if (!has || pr > pref || (pr == pref && k >= key)) { has = 1; pref = pr; key = k; pos = j; }
        }
        for (int off = 16; off; off >>= 1) {
          const uint32_t h2 = __shfl_down_sync(0xffffffffu, has, off), p2 = __shfl_down_sync(0xffffffffu, pref, off), j2 = __shfl_down_sync(0xffffffffu, pos, off);
          const unsigned long long k2 = __shfl_down_sync(0xffffffffu, key, off);
          if (h2 && (!has || p2 > pref || (p2 == pref && (k2 > key || (k2 == key && j2 > pos))))) { has = 1; pref = p2; key = k2; pos = j2; }
        }
        if (lane == 0) {
          out[w] = has ? (long long)key : 0;
          out[w + 1] = has ? col[(size_t)perm[pos] * a.acc_stride + 1] : 0;
        }
        continue;
      }
      unsigned long long acc = 0;  // the identity of every op (MAX is unsigned)
      for (uint32_t j = lo + lane; j < hi; j += 32) acc = agg_merge_op(op, acc, (unsigned long long)col[(size_t)perm[j] * a.acc_stride]);
      for (int off = 16; off; off >>= 1) acc = agg_merge_op(op, acc, __shfl_down_sync(0xffffffffu, acc, off));
      if (lane == 0) out[w] = (long long)acc;
    }
  }
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace

cudaError_t launch_agg_merge(const AggMergeArgs& a, void* tmp, size_t* tmp_bytes, cudaStream_t s) {
  const uint32_t n = a.n;
  // scratch: two key buffers, two index buffers, the group ids, the group starts, then cub's temporary storage
  const size_t keys_b = align256((size_t)n * 8), idx_b = align256((size_t)n * 4), starts_b = align256(((size_t)n + 1) * 4);
  const size_t fixed = 2 * keys_b + 3 * idx_b + starts_b;
  cub::DoubleBuffer<long long> kq(nullptr, nullptr);
  cub::DoubleBuffer<unsigned int> vq(nullptr, nullptr);
  if (!tmp) {  // (the queries cost host time: a run takes what is left after the fixed part as cub's storage)
    size_t sort_key_b = 0, sort_mask_b = 0, scan_b = 0;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, sort_key_b, kq, vq, (int)n, 0, 64, s);
    if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(nullptr, sort_mask_b, kq, vq, (int)n, 0, (int)a.key_words, s);
    if (e == cudaSuccess) e = cub::DeviceScan::InclusiveSum(nullptr, scan_b, (unsigned int*)nullptr, (unsigned int*)nullptr, (int)n, s);
    *tmp_bytes = fixed + std::max(std::max(sort_key_b, sort_mask_b), scan_b);
    return e;
  }
  if (*tmp_bytes < fixed) return cudaErrorInvalidValue;
  const size_t cub_b = *tmp_bytes - fixed;
  cudaError_t e = cudaSuccess;
  if (n == 0) return cudaMemsetAsync(a.n_groups, 0, 4, s);

  char* p = (char*)tmp;
  long long* k0 = (long long*)p; p += keys_b;
  long long* k1 = (long long*)p; p += keys_b;
  unsigned int* v0 = (unsigned int*)p; p += idx_b;
  unsigned int* v1 = (unsigned int*)p; p += idx_b;
  unsigned int* gid = (unsigned int*)p; p += idx_b;
  unsigned int* starts = (unsigned int*)p; p += starts_b;
  void* cub_tmp = p;
  kq = cub::DoubleBuffer<long long>(k0, k1);
  vq = cub::DoubleBuffer<unsigned int>(v0, v1);
  const int threads = 256, blocks = (int)((n + threads - 1) / threads);
  for (uint32_t pass = 0; pass <= a.key_words; ++pass) {
    const uint32_t word = pass < a.key_words ? a.key_words - 1 - pass : a.key_words;  // NULL mask in the last pass
    agg_merge_gather_kernel<<<blocks, threads, 0, s>>>(a, word, pass ? vq.Current() : nullptr, vq.Current(), kq.Current());
    size_t b = cub_b;
    e = cub::DeviceRadixSort::SortPairs(cub_tmp, b, kq, vq, (int)n, 0, word == a.key_words ? (int)a.key_words : 64, s);
    if (e != cudaSuccess) return e;
  }
  const unsigned int* perm = vq.Current();
  agg_merge_heads_kernel<<<blocks, threads, 0, s>>>(a, perm, gid);
  size_t b = cub_b;
  e = cub::DeviceScan::InclusiveSum(cub_tmp, b, gid, gid, (int)n, s);
  if (e != cudaSuccess) return e;
  agg_merge_starts_kernel<<<blocks, threads, 0, s>>>(gid, n, starts, a.n_groups);
  const int reduce_blocks = (int)(((size_t)n * 32 + threads - 1) / threads < 4096 ? ((size_t)n * 32 + threads - 1) / threads : 4096);
  agg_merge_reduce_kernel<<<reduce_blocks, threads, 0, s>>>(a, perm, starts, a.n_groups);
  return cudaGetLastError();
}

}  // namespace b2
