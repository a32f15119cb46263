// The per-entry rules of b2_sst_merge (sst.cu): the internal-key order, the staging checks of one entry and the verdict
// of one merged position.  __host__ __device__ so that the same code is built for the CPU in tests/sst_merge_emul.cpp.
//
// A staged key is  user key | fixed64 LE footer  with footer = seq << 8 | type.  The order is RocksDB's
// InternalKeyComparator: user key bytewise ascending, then the footer descending (the newest version first).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define B2M_HD __host__ __device__ __forceinline__
#else
#define B2M_HD inline
#endif

namespace b2merge {

enum : uint32_t { kDeletion = 0, kValue = 1, kSingleDeletion = 7 };
enum : uint32_t { kOk = 0, kCorrupt = 1, kUnsupported = 2 };                   // the decoder's error codes (SST_*)
enum : uint32_t { kInvisible = 0, kOut = 1, kDeleted = 2, kHidden = 3 };      // the verdict of one merged position
constexpr uint64_t kMaxSeq = (1ull << 56) - 1;

B2M_HD uint64_t footer_of(const uint8_t* key, uint32_t len) {  // (len >= 8)
  uint64_t f = 0;
  for (int i = 7; i >= 0; --i) f = (f << 8) | key[len - 8 + i];
  return f;
}

// Staged keys shorter than the footer (a corrupted run, reported by stage_check) compare as if their user key were
// empty; the footer is then read from the 8 bytes at the key's start, which the staged heap's padding keeps readable.
B2M_HD uint32_t body_len(uint32_t len) { return len < 8 ? 0 : len - 8; }

// -1, 0, 1: the user keys of a and b (body lengths la, lb)
B2M_HD int user_key_cmp(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  const uint32_t m = la < lb ? la : lb;
  for (uint32_t i = 0; i < m; ++i)
    if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
  return la == lb ? 0 : (la < lb ? -1 : 1);
}

// -1, 0, 1: a against b in internal-key order
B2M_HD int ikey_cmp(const uint8_t* a, uint32_t len_a, const uint8_t* b, uint32_t len_b) {
  const uint32_t la = body_len(len_a), lb = body_len(len_b);
  const int c = user_key_cmp(a, la, b, lb);
  if (c) return c;
  const uint64_t fa = footer_of(a + la, 8), fb = footer_of(b + lb, 8);
  return fa == fb ? 0 : (fa > fb ? -1 : 1);
}

// One entry of run r as decoded (key with its footer), given the entry before it in the same run (prev == nullptr for the
// run's first).  Returns kOk, kCorrupt (key shorter than its footer, the run not strictly ascending, or a stored seq
// other than 0 under a global seqno) or kUnsupported (a type other than Value / Deletion / SingleDeletion); *eff is the
// footer the merge orders by: the stored one, or global_seq << 8 | type for an ingested run.
B2M_HD uint32_t stage_check(const uint8_t* key, uint32_t len, const uint8_t* prev, uint32_t prev_len, uint64_t global_seq, uint64_t* eff) {
  *eff = 0;
  if (len < 8 || (prev && prev_len < 8)) return kCorrupt;
  const uint64_t f = footer_of(key, len);
  const uint32_t type = (uint32_t)(f & 0xff);
  if (type != kDeletion && type != kValue && type != kSingleDeletion) return kUnsupported;
  if (global_seq && (f >> 8)) return kCorrupt;
  if (prev && ikey_cmp(prev, prev_len, key, len) >= 0) return kCorrupt;
  *eff = global_seq ? (global_seq << 8 | type) : f;
  return kOk;
}

// The verdict of the merged position holding footer f, whose predecessor in merged order has footer pf and the same user
// key (same_key; false for position 0).  Within one user key the newest entry comes first, so the first visible one is
// the one whose predecessor is another user key or invisible.
B2M_HD uint32_t verdict(uint64_t f, bool same_key, uint64_t pf, uint64_t snapshot_seq) {
  if ((f >> 8) > snapshot_seq) return kInvisible;
  if (same_key && (pf >> 8) <= snapshot_seq) return kHidden;
  return (f & 0xff) == kValue ? kOut : kDeleted;
}

}  // namespace b2merge
