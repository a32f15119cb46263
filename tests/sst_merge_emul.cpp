// TEST INFRASTRUCTURE: the per-entry rules of b2_sst_merge (tikv_b200/csrc/sst_merge.h) built for the CPU and run under
// AddressSanitizer: stage_check over every entry of every run, then the entries ordered by ikey_cmp with the id as the
// tie-break (the device's comparator, here through std::sort), then verdict at every merged position.  Every key lives
// in an allocation of exactly its size.
//
//   sst_merge_emul <case> <result>
//   case   := u32 n_runs | u64 snapshot_seq | run*            run := u64 global_seq | u32 n | (u32 len | len key bytes)*
//   result := u32 status | (u32 id | u32 verdict)*   ids number the entries of all runs in order; the pairs follow the
//                                                  merged order and are written only when status == 0
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../tikv_b200/csrc/sst_merge.h"

struct Key { uint8_t* p; uint32_t len; };

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: %s case result\n", argv[0]); return 2; }
  FILE* in = fopen(argv[1], "rb");
  FILE* out = fopen(argv[2], "wb");
  if (!in || !out) { perror("open"); return 2; }
  uint32_t n_runs;
  uint64_t snap;
  if (fread(&n_runs, 4, 1, in) != 1 || fread(&snap, 8, 1, in) != 1) return 2;
  std::vector<Key> keys;
  uint32_t status = b2merge::kOk;
  for (uint32_t r = 0; r < n_runs; ++r) {
    uint64_t gs;
    uint32_t n;
    if (fread(&gs, 8, 1, in) != 1 || fread(&n, 4, 1, in) != 1) return 2;
    for (uint32_t i = 0; i < n; ++i) {
      uint32_t len;
      if (fread(&len, 4, 1, in) != 1) return 2;
      uint8_t* p = (uint8_t*)malloc(len ? len : 1);
      if (len && fread(p, 1, len, in) != len) return 2;
      uint64_t eff;
      const Key* prev = i ? &keys.back() : nullptr;
      const uint32_t st = b2merge::stage_check(p, len, prev ? prev->p : nullptr, prev ? prev->len : 0, gs, &eff);
      if (st > status) status = st;
      if (st == b2merge::kOk)
        for (int q = 0; q < 8; ++q) p[len - 8 + q] = (uint8_t)(eff >> (8 * q));
      keys.push_back({p, len});
    }
  }
  fwrite(&status, 4, 1, out);
  if (status == b2merge::kOk) {
    std::vector<uint32_t> ids(keys.size());
    for (uint32_t i = 0; i < ids.size(); ++i) ids[i] = i;
    std::sort(ids.begin(), ids.end(), [&](uint32_t a, uint32_t b) {
      const int c = b2merge::ikey_cmp(keys[a].p, keys[a].len, keys[b].p, keys[b].len);
      return c ? c < 0 : a < b;
    });
    for (uint32_t i = 0; i < ids.size(); ++i) {
      const Key& k = keys[ids[i]];
      const uint32_t bl = b2merge::body_len(k.len);
      bool same = false;
      uint64_t pf = 0;
      if (i) {
        const Key& pk = keys[ids[i - 1]];
        const uint32_t pbl = b2merge::body_len(pk.len);
        same = b2merge::user_key_cmp(pk.p, pbl, k.p, bl) == 0;
        pf = b2merge::footer_of(pk.p + pbl, 8);
      }
      const uint32_t v = b2merge::verdict(b2merge::footer_of(k.p + bl, 8), same, pf, snap);
      fwrite(&ids[i], 4, 1, out);
      fwrite(&v, 4, 1, out);
    }
  }
  for (Key& k : keys) free(k.p);
  fclose(in);
  fclose(out);
  return 0;
}
