// TEST INFRASTRUCTURE — CPU oracle of the merging read over sorted runs, not product code.
//
// What a RocksDB DBIter over a MergingIterator yields at a snapshot sequence number, restated from RocksDB's published
// semantics (RocksDB is not under the reference tree; TiKV reaches it through librocksdb behind components/engine_rocks):
//   - InternalKeyComparator: user key bytewise ascending, then the packed footer seq << 8 | type descending;
//   - MergingIterator: a min-heap of child iterators under that comparator; children whose current keys compare equal
//     come out in child order (the heap is built over the children newest first: memtable, L0 newest first, L1 .. Ln);
//   - DBIter (forward, no prefix / timestamps): entries with seq > snapshot are skipped; the first remaining entry of a
//     user key decides: kTypeValue yields it, kTypeDeletion / kTypeSingleDeletion yield nothing, and every later entry
//     of that user key is skipped;
//   - an ingested file carries sequence number 0 in its keys and a file-level global seqno that replaces it
//     (ExternalSstFileIngestionJob; TiKV ingests Raft snapshots, components/raftstore/src/store/snap/io.rs:388, and
//     imports, components/sst_importer/src/util.rs:213).
// Each run is read by the oracle's block iterator (oracle/orc_sst.h) keeping the footer (key_suffix_len 0).
// This is a heap merge of cursors, deliberately not the device's merge rounds over entry ids.
#include <cstdint>
#include <cstring>
#include <queue>
#include <string>
#include <vector>

#include "../oracle/orc_sst.h"

namespace {

struct Run {
  std::string keys, vals;
  std::vector<uint32_t> koff, voff;
  uint32_t n() const { return (uint32_t)koff.size() - 1; }
  std::string user(uint32_t i) const { return keys.substr(koff[i], koff[i + 1] - koff[i] - 8); }
  uint64_t footer(uint32_t i) const { uint64_t f; memcpy(&f, keys.data() + koff[i + 1] - 8, 8); return f; }
};

// a < b in internal-key order
bool ikey_less(const std::string& ua, uint64_t fa, const std::string& ub, uint64_t fb) {
  const int c = ua.compare(ub);
  if (c) return c < 0;
  return fa > fb;
}

struct Out { std::string keys, vals; std::vector<uint32_t> koff{0}, voff{0}; uint64_t counts[5] = {0, 0, 0, 0, 0}; };

}  // namespace

extern "C" {

// counts: n_in, n_out, n_invisible, n_hidden, n_deletions.  Returns 0 ok, 1 corrupted (a block, a key shorter than its
// footer, a run out of order, a nonzero stored seq under a global seqno), 2 unsupported (a block the iterator does
// not read, a value type other than 0 / 1 / 7); *out holds the output (free with orc_sst_merge_free).
int orc_sst_merge(const uint8_t* const* data, const uint64_t* const* block_offs, const uint32_t* n_blocks, const uint32_t* trailer_len, const uint64_t* global_seqs,
                  uint32_t n_runs, uint32_t key_prefix_len, uint64_t snapshot, void** out) {
  auto* o = new Out();
  *out = o;
  std::vector<Run> runs(n_runs);
  for (uint32_t r = 0; r < n_runs; ++r) {
    const int rc = orc::sst_decode(data[r], block_offs[r], n_blocks[r], trailer_len[r], key_prefix_len, 0, &runs[r].keys, &runs[r].koff, &runs[r].vals, &runs[r].voff);
    if (rc) return rc;
  }
  int verdict = 0;
  for (uint32_t r = 0; r < n_runs; ++r) {
    Run& R = runs[r];
    const uint64_t gs = global_seqs ? global_seqs[r] : 0;
    for (uint32_t i = 0; i < R.n(); ++i) {
      if (R.koff[i + 1] - R.koff[i] < 8) { verdict = verdict > 1 ? verdict : 1; continue; }
      const uint64_t f = R.footer(i);
      const uint32_t t = (uint32_t)(f & 0xff);
      if (t != 0 && t != 1 && t != 7) { verdict = 2; continue; }
      if (gs && (f >> 8)) verdict = verdict > 1 ? verdict : 1;
      if (i && R.koff[i] - R.koff[i - 1] >= 8 && !ikey_less(R.user(i - 1), R.footer(i - 1), R.user(i), f)) verdict = verdict > 1 ? verdict : 1;
    }
    if (gs)  // the ingested file's keys as its reader presents them
      for (uint32_t i = 0; i < R.n(); ++i) {
        const uint64_t f = gs << 8 | (R.footer(i) & 0xff);
        memcpy(&R.keys[R.koff[i + 1] - 8], &f, 8);
      }
  }
  if (verdict) return verdict;
  // MergingIterator
  struct Cur { uint32_t run, i; };
  auto later = [&](const Cur& a, const Cur& b) {  // priority_queue keeps the greatest on top: "later" is the lesser priority
    const std::string ua = runs[a.run].user(a.i), ub = runs[b.run].user(b.i);
    const uint64_t fa = runs[a.run].footer(a.i), fb = runs[b.run].footer(b.i);
    if (ikey_less(ua, fa, ub, fb)) return false;
    if (ikey_less(ub, fb, ua, fa)) return true;
    return a.run > b.run;
  };
  std::priority_queue<Cur, std::vector<Cur>, decltype(later)> heap(later);
  for (uint32_t r = 0; r < n_runs; ++r) {
    o->counts[0] += runs[r].n();
    if (runs[r].n()) heap.push({r, 0});
  }
  // DBIter
  bool have = false;  // a visible entry of `cur_user` was seen
  std::string cur_user;
  while (!heap.empty()) {
    const Cur c = heap.top();
    heap.pop();
    if (c.i + 1 < runs[c.run].n()) heap.push({c.run, c.i + 1});
    const Run& R = runs[c.run];
    const std::string u = R.user(c.i);
    const uint64_t f = R.footer(c.i);
    if (u != cur_user) { cur_user = u; have = false; }
    if ((f >> 8) > snapshot) { ++o->counts[2]; continue; }
    if (have) { ++o->counts[3]; continue; }
    have = true;
    if ((f & 0xff) == 1) {
      ++o->counts[1];
      o->keys += u;
      o->vals.append(R.vals, R.voff[c.i], R.voff[c.i + 1] - R.voff[c.i]);
      o->koff.push_back((uint32_t)o->keys.size());
      o->voff.push_back((uint32_t)o->vals.size());
    } else ++o->counts[4];
  }
  return 0;
}

// the output of orc_sst_merge as a host b2_cf_block's fields and its counts
void orc_sst_merge_result(void* h, const uint8_t** keys, const uint32_t** koff, const uint8_t** vals, const uint32_t** voff, uint32_t* n, uint64_t* counts) {
  auto* o = (Out*)h;
  *keys = (const uint8_t*)o->keys.data(); *koff = o->koff.data(); *vals = (const uint8_t*)o->vals.data(); *voff = o->voff.data();
  *n = (uint32_t)o->koff.size() - 1;
  memcpy(counts, o->counts, sizeof(o->counts));
}

void orc_sst_merge_free(void* h) { delete (Out*)h; }

}  // extern "C"
