// The lean kernels of the order-free pipelines: aggregation (no / one group-by expression), TopN and checksum.
//
// scan_body (scan_kernel.cuh) carries everything the reference's executors can meet — version walks, Lock / Rollback
// records, CF_DEFAULT lookups, every row layout, lazy errors — and pays for it on every row: ~900 warp instructions per
// 32 rows, CTA-wide votes per tile, 96 registers.  fast_body keeps only what a plain table needs and hands the rest over:
//
//   * one thread per CF_WRITE entry, 8 decoding warps + 1 TMA producer warp per CTA, no CTA-wide barrier on the row path
//     (TopN keeps one per tile for its shared candidate buffer);
//   * a branch-free front end per lane (b2_device.h: key_tail_load, fast_write_kind, fast_row_v2) and warp ballots for
//     the version runs (fast_lane_decide): plain runs — newer versions above the snapshot, then a Put with an inline
//     value or a Delete — are committed here; every other run (Lock / Rollback records, long values, gc fences, rows that
//     need the general decoder, evaluation errors, odd keys, RcCheckTs conflicts) has its first entry appended to
//     ScanArgs::slow_list, exactly once, and nothing of it is committed;
//   * scan_body then runs in list mode over those entries (engine.cu launches it right behind, it reads the count on the
//     device), so each run is processed by exactly one of the two kernels and statistics / results simply add up;
//   * aggregation without GROUP BY accumulates in registers (no atomics per row); with GROUP BY the CTA table is sized
//     for the group count, hashed with one multiply, and warp pre-aggregation is only tried while the table is tiny;
//   * checksum uses the linearity of CRC-64 (b2_device.h): one 8-byte table step per KV for the handle, plain XORs for
//     the value words, the table walks over value bytes once per warp at the end.
#pragma once
#include "scan_kernel.cuh"

namespace b2 {

enum { FK_STAGES = 2, FK_THREADS = TILE + 32, CK_WORDS = 16 /* value bytes / 8 the checksum kernel folds in registers */ };

__device__ __forceinline__ unsigned int hash32(unsigned long long k) { return ((unsigned int)k ^ (unsigned int)(k >> 32)) * 0x9E3779B1u; }

// a stage's tile and what the decoding warps need of its unit (read from shared memory per tile, not held in registers)
struct FastTileMeta : TileMeta {
  uint32_t unit, e0, e_lo, c_hi;  // the unit's index, the tile's first entry, the unit's first entry and end
  unsigned long long entry_base;
  const uint8_t* gvals;
};

template <int MODE>
__device__ __forceinline__ void fast_body(const DevPlan& P, const ScanArgs& A) {
  static_assert(MODE == PM_AGG || MODE == PM_TOPN || MODE == PM_CHECKSUM, "order-free pipelines only");
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  const unsigned int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint32_t n_tiles = A.n_unit_tiles;

  __shared__ __align__(8) unsigned long long s_full[FK_STAGES], s_empty[FK_STAGES];
  __shared__ FastTileMeta s_meta[FK_STAGES];
  __shared__ unsigned int s_tbl_used, s_tbl_miss, s_tbl_off;
  __shared__ unsigned int s_top_cnt, s_top_have_thr, s_top_next_sync;
  __shared__ TopItem s_top_thr;

  // ---- mode state in dynamic shared memory (before the stages) ----
  // PM_AGG with GROUP BY: the CTA table is addressed by the group key itself — slot k holds the accumulators of key k for
  // 0 <= k < slots (status codes, type ids, small dictionaries: the low-cardinality GROUP BY worth keeping on chip); no
  // hashing, no probing, no key compare.  occ[k] says whether key k was seen.  Every other key (and NULL) goes to the HBM
  // table.  Flushed into the HBM table once, at the end.
  SmemTable st;
  st.slots = 0; st.keys = nullptr; st.acc = nullptr;
  unsigned int* occ = nullptr;
  if (MODE == PM_AGG && P.has_group && A.smem_slots) {
    st.slots = A.smem_slots;
    st.acc = reinterpret_cast<unsigned long long*>(dyn_smem);
    occ = reinterpret_cast<unsigned int*>(st.acc + (size_t)st.slots * P.acc_words);
    for (unsigned int i = tid; i < st.slots; i += FK_THREADS) occ[i] = 0;
    for (unsigned int i = tid; i < st.slots * P.acc_words; i += FK_THREADS) st.acc[i] = 0;
  }
  const TopBuf tb = topbuf_make(MODE == PM_TOPN && A.topn_work ? A.topn_work + (size_t)blockIdx.x * A.topn_work_stride : dyn_smem, MODE == PM_TOPN ? A.topn_cap : 0u, P);
  if (MODE == PM_TOPN)
    for (unsigned int i = tid; i < A.topn_cap; i += FK_THREADS) tb.idx[i] = (unsigned short)i;
  unsigned long long* crc_tab = reinterpret_cast<unsigned long long*>(dyn_smem);  // PM_CHECKSUM: slicing-by-8 tables, then kacc[256]
  unsigned long long* kacc = crc_tab + 8 * 256;
  if (MODE == PM_CHECKSUM) {
    for (unsigned int i = tid; i < 256; i += FK_THREADS) { crc_tab[i] = crc64_table_entry(i); kacc[i] = 0; }
    __syncthreads();
    for (unsigned int i = tid; i < 256; i += FK_THREADS) {
      unsigned long long t = crc_tab[i];
      for (int kk = 1; kk < 8; ++kk) { t = crc_tab[(uint32_t)t & 0xffu] ^ (t >> 8); crc_tab[kk * 256 + i] = t; }
    }
  }
  if (tid == 0) {
    s_tbl_used = 0; s_tbl_miss = 0; s_tbl_off = 0; s_top_cnt = 0; s_top_have_thr = 0; s_top_next_sync = 0;
    if (MODE == PM_TOPN && A.topn_seed && A.limit > 0 && *A.topn_seed_cnt >= (unsigned int)A.limit) { s_top_thr = A.topn_seed[A.limit - 1]; s_top_have_thr = 1; }
    for (int i = 0; i < FK_STAGES; ++i) { mbar_init(&s_full[i], 1); mbar_init(&s_empty[i], TILE / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  unsigned char* stage_base = dyn_smem + A.stage_off;
  const uint32_t STAGE_KEY_CAP = A.stage_key_cap, STAGE_VAL_CAP = A.stage_val_cap;
  const uint32_t STAGE_BYTES = STAGE_KEY_CAP + STAGE_VAL_CAP + 2 * STAGE_OFF_CAP;

  // ---- producer warp: claims tiles of the unit table from one counter (so no CTA is left with a tail of its own), and
  // issues bulk copies of each tile's key / value bytes and offset slices, FK_STAGES tiles ahead.  Software-pipelined by
  // one tile: the claim and the four bounding offsets of tile k+1 are fetched while the producer waits for a free stage ----
  if (wid == TILE / 32) {
    if (lane == 0) {
      uint32_t u = 0;  // cursor into the unit table: claims only increase
      uint32_t nx_tile, nx_e0 = 0, nx_wlo = 0, nx_whi = 0, nx_k0 = 0, nx_k1 = 0, nx_v0 = 0, nx_v1 = 0;
      auto claim = [&]() {
        nx_tile = atomicAdd(A.tile_ctr, 1u);
        if (nx_tile < n_tiles) {
          while (u + 1 < A.n_units && A.units[u + 1].tile_lo <= nx_tile) ++u;
          const UnitDesc& d = A.units[u];
          nx_e0 = d.c_lo + (nx_tile - d.tile_lo) * TILE;
          nx_whi = nx_e0 + TILE < d.c_hi ? nx_e0 + TILE : d.c_hi;
          nx_wlo = nx_e0 > d.e_lo ? nx_e0 - 1 : nx_e0;
          nx_k0 = d.blk.koff[nx_wlo]; nx_k1 = d.blk.koff[nx_whi]; nx_v0 = d.blk.voff[nx_wlo]; nx_v1 = d.blk.voff[nx_whi];
        }
      };
      claim();
      for (uint32_t k = 0;; ++k) {
        const int slot = (int)(k % FK_STAGES);
        FastTileMeta m;
        m.tile = nx_tile;
        m.staged = 0; m.w_lo = 0; m.w_hi = 0; m.keys_adj = 0; m.vals_adj = 0; m.koff_adj = 0; m.voff_adj = 0;
        m.unit = 0; m.e0 = 0; m.e_lo = 0; m.c_hi = 0; m.entry_base = 0; m.gvals = nullptr;
        uint32_t tx = 0;
        const uint32_t w_lo = nx_wlo, w_hi = nx_whi, k0 = nx_k0, k1 = nx_k1, v0 = nx_v0, v1 = nx_v1;
        const BlockView blk = A.units[u].blk;
        if (m.tile < n_tiles) {
          const UnitDesc& d = A.units[u];
          m.unit = u; m.e0 = nx_e0; m.e_lo = d.e_lo; m.c_hi = d.c_hi; m.entry_base = d.entry_base; m.gvals = d.blk.vals;
        }
        mbar_wait_sleep(&s_empty[slot], ((k / FK_STAGES) & 1) ^ 1);
        if (m.tile < n_tiles) {
          unsigned long long ka = (unsigned long long)(blk.keys + k0), va = (unsigned long long)(blk.vals + v0);
          unsigned long long oa = (unsigned long long)(blk.koff + w_lo), ob = (unsigned long long)(blk.voff + w_lo);
          uint32_t kpad = (uint32_t)(ka & 15), vpad = (uint32_t)(va & 15), opad = (uint32_t)(oa & 15), qpad = (uint32_t)(ob & 15);
          uint32_t kbytes = (kpad + (k1 - k0) + 15) & ~15u, vbytes = (vpad + (v1 - v0) + 15) & ~15u;
          uint32_t obytes = (opad + (w_hi - w_lo + 1) * 4 + 15) & ~15u, qbytes = (qpad + (w_hi - w_lo + 1) * 4 + 15) & ~15u;
          if (kbytes + 16 <= STAGE_KEY_CAP && vbytes + 16 <= STAGE_VAL_CAP && obytes <= STAGE_OFF_CAP && qbytes <= STAGE_OFF_CAP) {
            m.staged = 1; m.w_lo = w_lo; m.w_hi = w_hi;
            m.keys_adj = (long long)kpad - (long long)k0; m.vals_adj = (long long)vpad - (long long)v0;
            m.koff_adj = (int)(opad / 4) - (int)w_lo; m.voff_adj = (int)(qpad / 4) - (int)w_lo;
            s_meta[slot] = m;
            unsigned char* stg = stage_base + (size_t)slot * STAGE_BYTES;
            tx = kbytes + vbytes + obytes + qbytes;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(&s_full[slot], tx);
            bulk_g2s(stg, (const void*)(ka - kpad), kbytes, &s_full[slot]);
            bulk_g2s(stg + STAGE_KEY_CAP, (const void*)(va - vpad), vbytes, &s_full[slot]);
            bulk_g2s(stg + STAGE_KEY_CAP + STAGE_VAL_CAP, (const void*)(oa - opad), obytes, &s_full[slot]);
            bulk_g2s(stg + STAGE_KEY_CAP + STAGE_VAL_CAP + STAGE_OFF_CAP, (const void*)(ob - qpad), qbytes, &s_full[slot]);
          }
        }
        if (!tx) {
          s_meta[slot] = m;
          asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&s_full[slot])) : "memory");
        }
        if (m.tile >= n_tiles) break;
        claim();
      }
    }
    return;
  }

  // ---- decoding warps ----
  unsigned long long n_keys = 0, n_size = 0, n_live = 0;
  unsigned int n_keys32 = 0, n_size32 = 0;  // per-lane counts (folded into the 64-bit ones before they could wrap)
  unsigned int n_newer = 0, n_last = 0, n_warn = 0;
  // PM_AGG without GROUP BY: accumulators in registers
  unsigned long long r_cnt[MAX_AGGS], r_lo[MAX_AGGS], r_hi[MAX_AGGS];
#pragma unroll
  for (int a = 0; a < MAX_AGGS; ++a) { r_cnt[a] = 0; r_lo[a] = 0; r_hi[a] = 0; }
  // PM_CHECKSUM: right-aligned XOR of the values, parity word, counters
  unsigned long long vacc[MODE == PM_CHECKSUM ? CK_WORDS : 1], ck_par = 0, ck_kvs = 0, ck_bytes = 0;
#pragma unroll
  for (int j = 0; j < (MODE == PM_CHECKSUM ? CK_WORDS : 1); ++j) vacc[j] = 0;
  const bool rc_check = A.isolation == B2_ISO_RC_CHECK_TS;
  // rows returned and the last of them are per unit (its range's row count, its block's entry_base): the warp hands them
  // over whenever its tile's unit changes (warp-uniform) and at the end
  uint32_t w_unit = ~0u;
  auto flush_unit = [&]() {
    n_keys += n_keys32; n_keys32 = 0;
    for (int off = 16; off > 0; off >>= 1) {
      n_keys += __shfl_xor_sync(0xffffffffu, n_keys, off);
      n_last = max(n_last, __shfl_xor_sync(0xffffffffu, n_last, off));
    }
    if (lane == 0) {
      const UnitDesc& d = A.units[w_unit];
      if (n_keys) atomicAdd(&A.ctr->processed_keys, n_keys);
      if (n_keys && d.range_rows) atomicAdd(d.range_rows, n_keys);
      if (n_last) atomicMax(&A.ctr->last_row, d.entry_base + n_last);
    }
    n_keys = 0; n_last = 0;
  };

  for (uint32_t k = 0;; ++k) {
    const int cur = (int)(k % FK_STAGES);
    mbar_wait_sleep(&s_full[cur], (k / FK_STAGES) & 1);  // suspended by the hardware until the stage lands: polling cost 6 % of the kernel's issue slots
    const uint32_t tile = s_meta[cur].tile;
    if (tile >= n_tiles) break;
    if (s_meta[cur].unit != w_unit) {
      if (w_unit != ~0u) flush_unit();
      w_unit = s_meta[cur].unit;
    }
    const uint32_t e_raw = s_meta[cur].e0 + tid;
    const bool valid = e_raw < s_meta[cur].c_hi;
    const uint32_t e = valid ? e_raw : s_meta[cur].c_hi - 1;
    bool push = false, live = false, cand = false;
    uint32_t push_e = e_raw;
    // per-mode values computed before the hand-over decision (an evaluation error turns the commit into a push)
    Value gk; gk.bits = 0; gk.null = false;
    Value av[MAX_AGGS];
    TopItem item;
    uint32_t rlen = 0;
    const uint8_t* rowp = nullptr;
    unsigned long long kw_a = 0, kw_b = 0;

    if (!s_meta[cur].staged) {
      push = valid;  // the tile did not fit the stage: every entry goes to the general walk (it skips the non-starts itself)
    } else {
      const unsigned char* stg = stage_base + (size_t)cur * STAGE_BYTES;
      SmemView sv;
      sv.skeys = stg + s_meta[cur].keys_adj;
      sv.svals = stg + STAGE_KEY_CAP + s_meta[cur].vals_adj;
      sv.skoff = reinterpret_cast<const uint32_t*>(stg + STAGE_KEY_CAP + STAGE_VAL_CAP) + s_meta[cur].koff_adj;
      sv.svoff = reinterpret_cast<const uint32_t*>(stg + STAGE_KEY_CAP + STAGE_VAL_CAP + STAGE_OFF_CAP) + s_meta[cur].voff_adj;
      sv.gvals = s_meta[cur].gvals;
      const uint32_t ko = sv.skoff[e], kl = sv.skoff[e + 1] - ko, vo = sv.svoff[e], vl = sv.svoff[e + 1] - vo;
      const uint8_t* kp = sv.skeys + ko;
      const uint8_t* vp = sv.svals + vo;
      KeyTail t;
      const bool k35 = kl == 35;
      const bool kok = key_tail_load(kp, &t) && k35;
      const uint64_t cts = key_tail_commit_ts(t);  // (only kept when the plan reads the commit-ts column)
      const bool vis = k35 && key_tail_visible(t, ~A.read_ts);
      // the entry before: its key words travel up one lane; lane 0 reads them itself
      unsigned int pa_lo = __shfl_up_sync(0xffffffffu, (unsigned int)t.a, 1), pa_hi = __shfl_up_sync(0xffffffffu, (unsigned int)(t.a >> 32), 1);
      unsigned int pb_lo = __shfl_up_sync(0xffffffffu, (unsigned int)t.b, 1);
      unsigned int px = __shfl_up_sync(0xffffffffu, ((unsigned int)(t.b >> 32) & 0xffffffu) | (k35 ? 1u << 24 : 0u) | (vis ? 1u << 25 : 0u), 1);
      // (on the clamped index: in a unit of one entry the lanes past the end hold that entry too, and looking one entry back
      //  from it would index the offsets with -1)
      const bool first = e == s_meta[cur].e_lo;
      if (lane == 0 && !first) {
        KeyTail q;
        const bool q35 = sv.klen(e - 1) == 35;
        key_tail_load(sv.kptr(e - 1), &q);
        pa_lo = (unsigned int)q.a; pa_hi = (unsigned int)(q.a >> 32); pb_lo = (unsigned int)q.b;
        px = ((unsigned int)(q.b >> 32) & 0xffffffu) | (q35 ? 1u << 24 : 0u) | ((q35 && key_tail_visible(q, ~A.read_ts)) ? 1u << 25 : 0u);
      }
      const bool same = valid && !first && k35 && ((px >> 24) & 1u) && (unsigned int)t.a == pa_lo && (unsigned int)(t.a >> 32) == pa_hi &&
                        (unsigned int)t.b == pb_lo && (((unsigned int)(t.b >> 32) ^ px) & 0xffffffu) == 0;
      const bool pvis = (px >> 25) & 1u;
      const bool chosen = vis && (!same || !pvis);
      uint32_t roff = 0;
      const uint32_t kind = fast_write_kind(vp, vl, &roff, &rlen);
      const unsigned int start_m = __ballot_sync(0xffffffffu, valid && !same), chosen_m = __ballot_sync(0xffffffffu, valid && chosen);
      const unsigned int valid_m = __ballot_sync(0xffffffffu, valid);
      uint32_t push_back = 0;
      const uint32_t act = fast_lane_decide(lane, start_m, chosen_m, valid_m, valid, same, chosen, kok, kind, vis, rc_check, &push_back);
      n_newer |= (valid && k35 && !vis) ? 1u : 0u;
      push = (act & FA_PUSH) != 0;
      push_e = e_raw - push_back;
      bool commit = (act & FA_COMMIT) != 0;
      rowp = vp + roff;
      kw_a = t.a; kw_b = t.b;
      if (MODE == PM_CHECKSUM) {
        if (commit && rlen > 8u * CK_WORDS) { commit = false; push = true; }
        live = commit;
      } else if (commit) {
        Row row;
        Cells cells;
        uint64_t cell_cache[8];
        row.cv = cell_cache;
        row.enc_key = kp; row.enc_key_len = 27; row.commit_ts = cts; row.imms = A.imms;
        bool ok = fast_row_v2(P, rowp, rlen, row);
        bool keep = false;
        if (ok) {
          row.filled = P.fast_filled;
#ifdef B2_JIT_PLAN
          fast_fill_cells(P, row, P.fast_need);  // every stored column an expression reads, once (compile-time positions)
#endif
          ok = eval_conds(P, row, cells, &keep) == 0;
        }
        if (ok && keep) {
          if (MODE == PM_AGG) {
            if (P.has_group) {
              ok = eval_expr(P, P.group, row, cells, &gk, nullptr) == 0;
              if (gk.null) gk.bits = 0;
              else if (P.group_et == 1 && bits_f64(gk.bits) == 0.0) gk.bits = 0;  // -0.0 and 0.0 are one group
            }
#pragma unroll
            for (int a = 0; a < MAX_AGGS; ++a)
              if (a < P.n_aggs && ok) ok = eval_expr(P, P.aggs[a].arg, row, cells, &av[a], nullptr) == 0;
          } else {
            // most rows lose against the CTA's threshold on their first sort key alone (the threshold only changes inside a
            // CTA-wide compaction, so reading it here is race-free).  When a later key can fail or warn, every row evaluates
            // all of them: a request's error and warning count must not depend on which rows the bound let through.
            Value v0;
            ok = eval_expr(P, P.order[0].e, row, cells, &v0, nullptr) == 0;
            cand = ok && (P.topn_all_keys || !s_top_have_thr || first_key_may_beat(P, v0, s_top_thr));
            const unsigned long long id = s_meta[cur].entry_base + e;
            if (cand) ok = make_item(P, row, cells, A.desc ? ~id : id, &item, &v0) == 0;
          }
        }
        if (!ok) { push = true; commit = false; }  // the general decoder / evaluator owns this run (and raises its error)
        live = commit && keep;
        if (commit) n_warn += row.warn;
      }
      if (commit) { n_keys32 += 1; n_size32 += 27u + rlen; n_last = e + 1; }
    }

    // ---- hand-over list: one atomic per warp ----
    const unsigned int pm = __ballot_sync(0xffffffffu, push);
    if (pm) {
      unsigned int base = 0;
      if (lane == 0) base = atomicAdd(A.slow_count + w_unit, (unsigned int)__popc(pm));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (push) A.slow_list[A.units[w_unit].slow_off + base + __popc(pm & ((1u << lane) - 1u))] = push_e;
    }
    n_live += live ? 1u : 0u;
    if ((k & 0xfffu) == 0xfffu) { n_keys += n_keys32; n_size += n_size32; n_keys32 = 0; n_size32 = 0; }  // (a lane adds < 2^20 per 4096 tiles)

    // ---- commit ----
    if (MODE == PM_AGG) {
      if (!P.has_group) {
        if (live) {
#pragma unroll
          for (int a = 0; a < MAX_AGGS; ++a) {
            if (a < P.n_aggs) {
              const DevAgg g = P.aggs[a];
              const bool has = !av[a].null;
              r_cnt[a] += has ? 1u : 0u;
              if (agg_is_extremum(g.kind)) {
                const unsigned long long key = has ? extremum_key(av[a].bits, g.arg_et, g.arg_unsigned, g.kind == AGG_MIN) : 0ull;
                r_lo[a] = key > r_lo[a] ? key : r_lo[a];
              } else if (g.kind == AGG_FIRST) {  // r_lo / r_hi: the lane's (key, value) pair
                const unsigned long long key = first_agg_key(s_meta[cur].entry_base + e, A.desc, !has);
                if (key > r_lo[a]) { r_lo[a] = key; r_hi[a] = has ? av[a].bits : 0ull; }
              } else if (agg_is_bit(g.kind)) {
                const unsigned long long x = bit_agg_word(g.kind, has, av[a].bits);
                r_lo[a] = g.kind == AGG_BIT_XOR ? r_lo[a] ^ x : r_lo[a] | x;
              } else if (g.kind != AGG_COUNT && has) {
                r_lo[a] += (uint32_t)av[a].bits;
                r_hi[a] += g.arg_unsigned ? (unsigned long long)(uint32_t)(av[a].bits >> 32) : (unsigned long long)(long long)(int32_t)(av[a].bits >> 32);
              }
            }
          }
        }
      } else {
        const unsigned int active = __ballot_sync(0xffffffffu, live);
        // warp pre-aggregation only pays while the CTA has met a handful of groups (few, hot accumulators): uniform switch
        const bool preagg = st.slots && *(volatile unsigned int*)&s_tbl_used <= 8u;
        if (live) {
          const bool direct = st.slots && !gk.null && gk.bits < (unsigned long long)st.slots;
          unsigned int peers = 1u << lane;
          if (preagg) {
            const unsigned int nm = __ballot_sync(active, gk.null);
            peers = __match_any_sync(active, gk.bits) & (gk.null ? nm : ~nm);
          }
          const bool leader = !preagg || (unsigned int)(__ffs(peers) - 1) == lane;
          const bool solo = !preagg || (peers & (peers - 1)) == 0;
          unsigned long long* acc = nullptr;
          if (leader) {
            if (direct) {
              const unsigned int slot = (unsigned int)gk.bits;
              if (*(volatile unsigned int*)&occ[slot] == 0 && atomicExch(&occ[slot], 1u) == 0) atomicAdd(&s_tbl_used, 1u);
              acc = st.acc + (size_t)slot * P.acc_words;
            } else {
              const unsigned int gslot = table_find_or_insert(A.tbl, gk.bits, gk.null);
              if (gslot == 0xffffffffu) atomicExch(&A.ctr->agg_overflow, 1u);
              else acc = A.tbl.acc + (size_t)gslot * P.acc_words;
            }
          }
#pragma unroll
          for (int a = 0; a < MAX_AGGS; ++a) {
            if (a < P.n_aggs) {
              const DevAgg g = P.aggs[a];
              const bool has = !av[a].null;
              const unsigned int cnt = solo ? (has ? 1u : 0u) : __reduce_add_sync(peers, has ? 1u : 0u);
              unsigned long long* w = acc + g.acc_off;
              const bool commit_w = leader && acc != nullptr && cnt != 0;
              if (g.kind == AGG_COUNT) {
                if (commit_w) atomicAdd(&w[0], (unsigned long long)cnt);
              } else if (agg_is_extremum(g.kind)) {
                unsigned long long key = has ? extremum_key(av[a].bits, g.arg_et, g.arg_unsigned, g.kind == AGG_MIN) : 0ull;
                if (!solo)
                  for (unsigned int mm = peers & (peers - 1); mm; mm &= mm - 1) {
                    unsigned long long other = __shfl_sync(peers, key, __ffs(mm) - 1);
                    key = other > key ? other : key;
                  }
                if (commit_w) { atomicAdd(&w[0], (unsigned long long)cnt); atomicMax(&w[1], key); }
              } else if (g.kind == AGG_FIRST) {
                unsigned long long key = first_agg_key(s_meta[cur].entry_base + e, A.desc, !has), val = has ? av[a].bits : 0ull;
                if (!solo)
                  for (unsigned int mm = peers & (peers - 1); mm; mm &= mm - 1) {
                    const unsigned long long ok2 = __shfl_sync(peers, key, __ffs(mm) - 1), ov = __shfl_sync(peers, val, __ffs(mm) - 1);
                    if (ok2 > key) { key = ok2; val = ov; }
                  }
                if (leader && acc != nullptr) first_agg_update(w, key, val);
              } else if (agg_is_bit(g.kind)) {
                unsigned long long x = bit_agg_word(g.kind, has, av[a].bits);
                if (!solo) {
                  const unsigned int lo = g.kind == AGG_BIT_XOR ? __reduce_xor_sync(peers, (unsigned int)x) : __reduce_or_sync(peers, (unsigned int)x);
                  const unsigned int hi = g.kind == AGG_BIT_XOR ? __reduce_xor_sync(peers, (unsigned int)(x >> 32)) : __reduce_or_sync(peers, (unsigned int)(x >> 32));
                  x = ((unsigned long long)hi << 32) | lo;
                }
                if (leader && acc != nullptr && x) { if (g.kind == AGG_BIT_XOR) atomicXor(&w[0], x); else atomicOr(&w[0], x); }
              } else {
                const uint32_t lo = has ? (uint32_t)av[a].bits : 0u, hi = has ? (uint32_t)(av[a].bits >> 32) : 0u;
                unsigned long long lo_sum, hi_sum;
                if (solo) {
                  lo_sum = lo;
                  hi_sum = g.arg_unsigned ? (unsigned long long)hi : (unsigned long long)(long long)(int32_t)hi;
                } else {
                  const unsigned int s0 = __reduce_add_sync(peers, lo & 0xffffu), s1 = __reduce_add_sync(peers, lo >> 16);
                  lo_sum = (unsigned long long)s0 + ((unsigned long long)s1 << 16);
                  const unsigned int t0 = __reduce_add_sync(peers, hi & 0xffffu);
                  if (g.arg_unsigned) hi_sum = (unsigned long long)t0 + ((unsigned long long)__reduce_add_sync(peers, hi >> 16) << 16);
                  else hi_sum = (unsigned long long)((long long)__reduce_add_sync(peers, (int)hi >> 16) * 65536ll + (long long)t0);
                }
                if (commit_w) { atomicAdd(&w[0], (unsigned long long)cnt); atomicAdd(&w[1], lo_sum); atomicAdd(&w[2], hi_sum); }
              }
            }
          }
        }
      }
    } else if (MODE == PM_TOPN) {
      if (live && cand && (!s_top_have_thr || item_less(item, s_top_thr, P))) {
        const unsigned int pos = atomicAdd(&s_top_cnt, 1u);
        topbuf_put(tb, tb.idx[pos], item);  // pos < topn_cap: see the rendezvous schedule below
      }
      // CTA rendezvous only as often as the buffer could fill up: at most TILE candidates arrive per tile, so after a
      // rendezvous that left `cnt` of them the next one is due (cap - cnt) / TILE tiles later
      if (k == s_top_next_sync) {
        cta256_sync();
        if (s_top_cnt + 2 * TILE > A.topn_cap) cta_topn_compact(tb, (unsigned int)A.limit, &s_top_cnt, &s_top_have_thr, &s_top_thr, P);
        if (tid == 0) { const unsigned int room = (A.topn_cap - s_top_cnt) / TILE; s_top_next_sync = k + (room > 1 ? room - 1 : 1); }
        cta256_sync();
      }
    } else {  // PM_CHECKSUM
      const unsigned int cm = __ballot_sync(0xffffffffu, live);
      if (cm) {
        const unsigned long long ck = live ? crc_step8(crc_tab, A.units[w_unit].ck_key_state, key_tail_handle_le(kw_a, kw_b)) : 0ull;
        // the key states are folded per value length (the zero-byte advance by that length happens once, at the end)
        const uint32_t lead_len = __shfl_sync(0xffffffffu, rlen, __ffs(cm) - 1);
        if (__all_sync(0xffffffffu, !live || rlen == lead_len)) {
          const unsigned int xl = __reduce_xor_sync(0xffffffffu, (unsigned int)ck), xh = __reduce_xor_sync(0xffffffffu, (unsigned int)(ck >> 32));
          if (lane == 0) atomicXor(&kacc[lead_len], ((unsigned long long)xh << 32) | xl);
        } else if (live) atomicXor(&kacc[rlen], ck);
        if (live) {
          ck_par ^= ~0ull; ck_kvs += 1; ck_bytes += 19ull + rlen + A.ck_old_prefix_len - A.ck_new_prefix_len;
        }
        // value words, right-aligned: word j = the 8 bytes ending 8j bytes before the value's end (lanes past their own
        // length read earlier stage bytes and mask them away)
        const uint32_t max_len = __reduce_max_sync(0xffffffffu, live ? rlen : 0u);
        const uint8_t* vend = rowp + rlen;
#pragma unroll
        for (int j = 0; j < CK_WORDS; ++j) {
          if (8u * j < max_len) {
            const unsigned long long w = ld64(vend - 8 * (j + 1));
            const uint32_t have = rlen > 8u * j ? rlen - 8u * j : 0u;  // value bytes at or after this word's start
            const unsigned long long m = !live || have == 0 ? 0ull : (have >= 8 ? ~0ull : (~0ull << (64 - 8 * have)));
            vacc[j] ^= w & m;
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&s_empty[cur])) : "memory");
  }

  // ---- epilogue ----
  if (MODE == PM_CHECKSUM) {
    // Lin(XOR of the values): fold the warp's accumulator words, then one table walk per warp
#pragma unroll
    for (int j = CK_WORDS - 1; j >= 0; --j) {
      const unsigned int lo = __reduce_xor_sync(0xffffffffu, (unsigned int)vacc[j]), hi = __reduce_xor_sync(0xffffffffu, (unsigned int)(vacc[j] >> 32));
      vacc[j] = ((unsigned long long)hi << 32) | lo;
    }
    unsigned long long x = ((unsigned long long)__reduce_xor_sync(0xffffffffu, (unsigned int)(ck_par >> 32)) << 32) | __reduce_xor_sync(0xffffffffu, (unsigned int)ck_par);
    if (lane == 0) {
      unsigned long long lin = 0;
#pragma unroll 1
      for (int j = CK_WORDS - 1; j >= 0; --j) lin = crc_step8(crc_tab, lin, vacc[j]);
      x ^= lin;
    }
    for (int off = 16; off > 0; off >>= 1) { ck_kvs += __shfl_xor_sync(0xffffffffu, ck_kvs, off); ck_bytes += __shfl_xor_sync(0xffffffffu, ck_bytes, off); }
    cta256_sync();  // every warp's key states are in kacc
    unsigned long long y = kacc[tid];
    if (y) y = crc_advance_zeros(crc_tab, y, tid);
    y = ((unsigned long long)__reduce_xor_sync(0xffffffffu, (unsigned int)(y >> 32)) << 32) | __reduce_xor_sync(0xffffffffu, (unsigned int)y);
    if (lane == 0) {
      if (x ^ y) atomicXor(&A.ctr->checksum, x ^ y);
      if (ck_kvs) { atomicAdd(&A.ctr->total_kvs, ck_kvs); atomicAdd(&A.ctr->total_bytes, ck_bytes); }
    }
  }
  if (MODE == PM_TOPN) {
    cta256_sync();
    cta_topn_compact(tb, (unsigned int)A.limit, &s_top_cnt, &s_top_have_thr, &s_top_thr, P);
    const unsigned int keep = s_top_cnt;
    for (unsigned int i = tid; i < keep; i += TILE) A.topn.items[(size_t)blockIdx.x * A.topn.stride + i] = topbuf_get(tb, tb.idx[i]);
    if (tid == 0) A.topn.counts[blockIdx.x] = keep;
  }
  if (MODE == PM_AGG) {
    if (!P.has_group) {
#pragma unroll
      for (int a = 0; a < MAX_AGGS; ++a) {
        if (a < P.n_aggs) {
          const DevAgg g = P.aggs[a];
          for (int off = 16; off > 0; off >>= 1) {
            r_cnt[a] += __shfl_xor_sync(0xffffffffu, r_cnt[a], off);
            const unsigned long long o_lo = __shfl_xor_sync(0xffffffffu, r_lo[a], off), o_hi = __shfl_xor_sync(0xffffffffu, r_hi[a], off);
            if (agg_is_extremum(g.kind)) r_lo[a] = o_lo > r_lo[a] ? o_lo : r_lo[a];
            else if (g.kind == AGG_FIRST) { if (o_lo > r_lo[a]) { r_lo[a] = o_lo; r_hi[a] = o_hi; } }
            else if (g.kind == AGG_BIT_XOR) r_lo[a] ^= o_lo;
            else if (agg_is_bit(g.kind)) r_lo[a] |= o_lo;
            else r_lo[a] += o_lo;
            if (g.kind != AGG_FIRST) r_hi[a] += o_hi;
          }
          unsigned long long* w = A.tbl.acc + g.acc_off;
          if (lane == 0 && g.kind == AGG_FIRST && r_lo[a]) first_agg_update(w, r_lo[a], r_hi[a]);
          else if (lane == 0 && agg_is_bit(g.kind) && r_lo[a]) { if (g.kind == AGG_BIT_XOR) atomicXor(&w[0], r_lo[a]); else atomicOr(&w[0], r_lo[a]); }
          else if (lane == 0 && r_cnt[a] && g.kind < AGG_FIRST) {
            atomicAdd(&w[0], r_cnt[a]);
            if (agg_is_extremum(g.kind)) atomicMax(&w[1], r_lo[a]);
            else if (g.kind != AGG_COUNT) { atomicAdd(&w[1], r_lo[a]); atomicAdd(&w[2], r_hi[a]); }
          }
        }
      }
    } else if (st.slots) {
      cta256_sync();
      for (unsigned int s = tid; s < st.slots; s += TILE) {
        if (occ[s] == 0) continue;
        const unsigned int gslot = table_find_or_insert(A.tbl, (unsigned long long)s, false);
        if (gslot == 0xffffffffu) { atomicExch(&A.ctr->agg_overflow, 1u); continue; }
        for (int a = 0; a < P.n_aggs; ++a) {
          const DevAgg g = P.aggs[a];
          const unsigned long long* src = st.acc + (size_t)s * P.acc_words + g.acc_off;
          unsigned long long* dst = A.tbl.acc + (size_t)gslot * P.acc_words + g.acc_off;
          if (src[0] == 0) continue;
          if (g.kind == AGG_FIRST) { first_agg_update(dst, src[0], src[1]); continue; }
          if (agg_is_bit(g.kind)) { if (g.kind == AGG_BIT_XOR) atomicXor(&dst[0], src[0]); else atomicOr(&dst[0], src[0]); continue; }
          atomicAdd(&dst[0], src[0]);
          if (g.kind == AGG_COUNT) continue;
          if (agg_is_extremum(g.kind)) atomicMax(&dst[1], src[1]);
          else { atomicAdd(&dst[1], src[1]); atomicAdd(&dst[2], src[2]); }
        }
      }
    }
  }
  // statistics
  if (w_unit != ~0u) flush_unit();
  n_size += n_size32;
  for (int off = 16; off > 0; off >>= 1) {
    n_size += __shfl_xor_sync(0xffffffffu, n_size, off);
    n_live += __shfl_xor_sync(0xffffffffu, n_live, off);
    n_newer |= __shfl_xor_sync(0xffffffffu, n_newer, off);
    n_warn += __shfl_xor_sync(0xffffffffu, n_warn, off);
  }
  if (lane == 0) {
    if (n_size) atomicAdd(&A.ctr->processed_size, n_size);
    if (n_live) atomicAdd(&A.ctr->live_rows, n_live);
    if (n_newer) atomicOr(&A.ctr->met_newer, 1u);
    if (n_warn) atomicAdd(&A.ctr->warn_div0, (unsigned long long)n_warn);
  }
}

}  // namespace b2
