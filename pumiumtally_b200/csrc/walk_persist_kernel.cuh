// The persistent walk kernel, included three times by walk_persist.cuh: as walk_persist_kernel (PTB_PERSIST_CU false, the
// parameters KernelParams<NS, TM>), as walk_persist_current_kernel (true, CurrentWalkParams: the walks with face
// currents) and as walk_persist_current_mu_kernel (PTB_PERSIST_MU true as well: face currents with cosine bins).  The
// face-current kernels get names of their own so that their instantiations stay apart from the others, and the text
// is shared, not wrapped, so that the others compile to exactly the code they had before.
template <int BLOCK, int FETCH, int MINB, int REFILL_T, int STAGING, int NS = 0, bool TM = false, bool MO = false>
__global__ void __launch_bounds__(BLOCK, MINB) PTB_PERSIST_NAME(const PTB_PERSIST_PARAMS P) {
  constexpr bool CU = PTB_PERSIST_CU;
  constexpr bool MU = PTB_PERSIST_MU;
  constexpr bool GATHER = STAGING == 1;
  constexpr bool PACKED = STAGING == 2;
  constexpr int WARPS = BLOCK / 32;
  constexpr bool kBulkTets = FETCH == kFetchBulk;
  constexpr bool kRows = FETCH == kFetchBulk;
  __shared__ ParticleStage stages[WARPS][2];
  __shared__ __align__(8) unsigned long long bars[WARPS][3];
  __shared__ __align__(128) unsigned char rows[kRows ? WARPS : 1][kRows ? 32 * kRowBytes : 16];
  // The timed walk keeps the per-lane L1 fetch in the binned kernel: with the cooperative one it ran 19 % slower, and
  // still 12 % slower once that fetch was issued without branches (DESIGN section 4.1, item 6).
  constexpr bool kCoop = FETCH == kFetchCoopL1 && !TM;
  __shared__ __align__(16) unsigned char coop_rows[kCoop ? WARPS : 1][kCoop ? kCoopWarpBytes : 16];
  constexpr bool kEdge = FETCH == kFetchEdge;
  // each lane's ray target (plane_step, edge_persist_step) and particle id (plane_step); the whole-record
  // and lean steps keep their own
  constexpr bool kTargetSlot = !kRows && FETCH != kFetchLean && FETCH != kFetchLeanL1;
  __shared__ double targets[kTargetSlot ? BLOCK : 1][3];
  __shared__ int32_t lane_ids[kTargetSlot ? BLOCK : 1];
  __shared__ SchedFixed sched_fixed[WARPS];
  __shared__ SchedCursor sched_cursor[WARPS];
  __shared__ int32_t ticket_ids[GATHER ? WARPS : 1][2][kClaimRun * kChunk];  // gather mode: current and next ticket
  static_assert(NS == 0 || (!kEdge && !kRows), "scored walks run on the plane records");
  static_assert(!TM || NS > 0, "the timed walk is a scored walk");
  static_assert(!CU || NS > 0, "face currents run on the tallied walk");
  __shared__ double score_wl[kLaneSlots<NS, TM, CU, MU>][NS > 0 ? BLOCK : 1];  // scored walk: ScoreLane::wl of each lane
  __shared__ int32_t time_bin[TM ? BLOCK : 1];                          // timed walk: TimeLane::bin of each lane
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t bar0 = smem_u32(&bars[warp][0]);
  const uint32_t bar_row = bar0 + 16;
  const uint32_t row = smem_u32(&rows[kRows ? warp : 0][kRows ? lane * kRowBytes : 0]);
  if (lane == 0) {
    mbar_init(bar0, GATHER ? 32 : 1);
    mbar_init(bar0 + 8, GATHER ? 32 : 1);
    mbar_init(bar_row, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();
  // The L2 policies are made where they are used (one createpolicy each): none is held across the loop.
  SchedFixed fx;
  SchedCursor s;
  fx.total = (GATHER || PACKED) ? (int)__ldg(P.work_count) : P.end - P.begin;
  fx.nchunks = (fx.total + kChunk - 1) / kChunk;
  // Gather mode: a ticket is a run of kClaimRun chunks = 64 particles whose ids are copied to the
  // warp's ticket_ids.  The *next* ticket is claimed, and its ids requested, one run ahead, so the
  // id copies are never waited for.
  static_assert(kClaimRun * kChunk == 64, "two ids per lane cover the largest ticket");
  fx.claim_run = GATHER ? min(max(P.claim_run, 1), kClaimRun) : 1;
  s.run_base = s.run_next = s.run_end = 0;
  s.pend_base = -1;
  s.tk = 0;
  // Die split (sorted modes only).  On a GPU whose L2 is two partitions that each cache the lines their own SMs
  // touch, a line only the other partition holds costs a longer trip.  When all SMs
  // work through the sorted particles front to back, both partitions hold the same window of the mesh.  Here
  // the SMs of partition 0 take chunks from the front of the sequence and those of partition 1 from its own
  // start further back (the sequence is cut in proportion to the SM counts), so each partition caches only its
  // own window; a partition that runs out of chunks helps the other finish.
  constexpr bool kSplit = GATHER || PACKED;
  constexpr int kNoChunk = 0x3fffffff;
  s.split_phase = 2;
  fx.own_lo = fx.own_hi = fx.oth_lo = fx.oth_hi = 0;
  fx.own_cnt = fx.oth_cnt = P.work_counter;
  if constexpr (kSplit) {
    if (P.die0_sms > 0 && P.die0_sms < P.nsms) {
      unsigned sm;
      asm("mov.u32 %0, %%smid;" : "=r"(sm));
      const int die = (P.die_mask[(sm >> 5) & 7] >> (sm & 31)) & 1;
      const int mid = (int)((long long)fx.nchunks * P.die0_sms / P.nsms) & ~(kClaimRun - 1);  // tickets never straddle it
      fx.own_lo = die ? mid : 0; fx.own_hi = die ? fx.nchunks : mid;
      fx.oth_lo = die ? 0 : mid; fx.oth_hi = die ? mid : fx.nchunks;
      fx.own_cnt = die ? P.work_counter2 : P.work_counter;
      fx.oth_cnt = die ? P.work_counter : P.work_counter2;
      s.split_phase = 0;
    }
  }
  // next ticket of `run` chunks: its first chunk, or a value >= nchunks when nothing is left (warp-uniform)
  auto take = [&](int run) -> int {
    int c = 0;
    if constexpr (kSplit) {
      if (s.split_phase < 2) {
        if (lane == 0) {
          c = kNoChunk;
          if (s.split_phase == 0) {
            c = fx.own_lo + (int)atomicAdd(fx.own_cnt, (unsigned)run);
            if (c >= fx.own_hi) { c = kNoChunk; s.split_phase = 1; }
          }
          if (c == kNoChunk) {
            c = fx.oth_lo + (int)atomicAdd(fx.oth_cnt, (unsigned)run);
            if (c >= fx.oth_hi) { c = kNoChunk; s.split_phase = 3; }
          }
        }
        s.split_phase = __shfl_sync(0xffffffffu, s.split_phase, 0);
        return __shfl_sync(0xffffffffu, c, 0);
      }
      if (s.split_phase == 3) return kNoChunk;
    }
    if (lane == 0) c = (int)atomicAdd(P.work_counter, (unsigned)run);
    return __shfl_sync(0xffffffffu, c, 0);
  };
  // claims the next ticket and starts the copies of its ids into ticket_ids[warp][s.tk ^ 1]
  auto fetch_ticket = [&]() {
    s.pend_base = take(fx.claim_run);
    const long long p0 = (long long)s.pend_base * kChunk + lane, p1 = p0 + 32;
    const long long pe = min((long long)fx.total, ((long long)s.pend_base + fx.claim_run) * kChunk);
    int32_t *ids = ticket_ids[GATHER ? warp : 0][s.tk ^ 1];
    if (p0 < pe) cp_async_4(smem_u32(ids + lane), P.order + p0);
    if (p1 < pe) cp_async_4(smem_u32(ids + lane + 32), P.order + p1);
    cp_async_commit();
  };
  auto load_stage = [&](int chunk, ParticleStage *st, uint32_t bar) {
    if constexpr (PACKED) {
      // one bulk copy: the chunk's rows are contiguous and every row is 64 bytes, ragged tail included
      if (lane == 0) {
        const uint32_t bytes = 64u * (uint32_t)min(kChunk, fx.total - chunk * kChunk);
        mbar_expect_tx(bar, bytes);
        bulk_g2s_hint(smem_u32(st), P.rows + (size_t)chunk * kChunk, bytes, bar, l2_policy_stream_now());
      }
    } else if constexpr (GATHER) {
      const int k = chunk - s.run_base;  // chunk's position in the current ticket (warp-uniform)
      const int id = ticket_ids[warp][s.tk][k * kChunk + (lane & (kChunk - 1))];
      stage_gather(P, id, min(kChunk, fx.total - chunk * kChunk), st, bar, lane, l2_policy_stream_now());
    } else if constexpr (FETCH == kFetchPlain) {
      stage_load(P, chunk, st, bar, lane);
    } else {
      stage_load_hint(P, chunk, st, bar, lane, l2_policy_stream_now());
    }
  };
  auto claim = [&]() -> int {
    int c = 0;
    if constexpr (GATHER) {
      if (s.run_next >= s.run_end) {
        if (s.pend_base < 0) fetch_ticket();
        s.run_base = s.run_next = s.pend_base;
        s.run_end = s.pend_base + fx.claim_run;
        s.tk ^= 1;
        cp_async_wait_ids();  // this lane's copies of the ticket's ids have landed...
        __syncwarp();         // ...and every lane's are visible to the warp
        fetch_ticket();
      }
      c = s.run_next++;
    } else {
      c = take(1);
    }
    return c < fx.nchunks ? c : -1;
  };

  s.cur = s.cursor = s.cur_count = 0;
  s.parity = 0;
  s.chunk_cur = claim();
  if (s.chunk_cur >= 0) load_stage(s.chunk_cur, &stages[warp][0], bar0);
  s.chunk_next = s.chunk_cur >= 0 ? claim() : -1;
  if (s.chunk_next >= 0) load_stage(s.chunk_next, &stages[warp][1], bar0 + 8);
  if (s.chunk_cur >= 0) {
    mbar_wait(bar0, 0);
    s.parity ^= 1u;
    s.cur_count = min(kChunk, fx.total - s.chunk_cur * kChunk);
  }
  if (lane == 0) {
    sched_fixed[warp] = fx;
    sched_cursor[warp] = s;
  }
  __syncwarp();

  Counters c;
  Ray r;
  EdgeRay g;  // only live in the compact-layout instantiation
  g.dv = 0;
  r.stage = kStageDone;
  int my_i = 0;
  uint32_t row_parity = 0;  // phase parity of the tet-row barrier (kBulkTets)
  double *const tgt = &targets[kTargetSlot ? threadIdx.x : 0][0];
  for (;;) {
    unsigned idle = __ballot_sync(0xffffffffu, r.stage == kStageDone);
    if ((int)__popc(idle) >= REFILL_T && sched_cursor[warp].cur_count > 0) {
      fx = sched_fixed[warp];
      s = sched_cursor[warp];
      while (s.cur_count > 0 && (int)__popc(idle) >= REFILL_T) {
        const int slot = s.cursor + __popc(idle & ((1u << lane) - 1u));
        if (r.stage == kStageDone && slot < s.cur_count) {
          if constexpr (PACKED) {
            const auto sl = walk_lane<NS, BLOCK, TM>(P, &score_wl[0][0], &time_bin[0]);
            my_i = begin_from_row<NS, TM, MO, CU, MU>(P, reinterpret_cast<const PackedRow *>(&stages[warp][s.cur]) + slot,
                                                      r, c, NS > 0 ? &sl : nullptr);
          } else {
            my_i = GATHER ? stages[warp][s.cur].id[slot] : P.begin + s.chunk_cur * kChunk + slot;
            const auto sl = walk_lane<NS, BLOCK, TM>(P, &score_wl[0][0], &time_bin[0]);
            begin_from_stage<NS, TM, MO, CU, MU>(P, &stages[warp][s.cur], slot, r, c, my_i, NS > 0 ? &sl : nullptr);
          }
          if constexpr (FETCH == kFetchEdge) g.dv = 0;
          if constexpr (kTargetSlot) {
            if (r.stage != kStageDone) {
              tgt[0] = r.tx; tgt[1] = r.ty; tgt[2] = r.tz;
              lane_ids[threadIdx.x] = my_i;
            }
          }
        }
        __syncwarp();
        s.cursor += __popc(idle);
        if (s.cursor >= s.cur_count) {
          // every slot of this stage has been handed out: recycle it for the chunk after next
          const int recycled = s.cur;
          s.chunk_cur = s.chunk_next;
          s.cur ^= 1;
          s.cursor = 0;
          s.cur_count = 0;
          s.chunk_next = -1;
          if (s.chunk_cur >= 0) {
            mbar_wait(bar0 + 8 * s.cur, (s.parity >> s.cur) & 1u);
            s.parity ^= 1u << s.cur;
            s.cur_count = min(kChunk, fx.total - s.chunk_cur * kChunk);
            s.chunk_next = claim();
            if (s.chunk_next >= 0) {
              if (lane == 0) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
              load_stage(s.chunk_next, &stages[warp][recycled], bar0 + 8 * recycled);
            }
          }
        }
        idle = __ballot_sync(0xffffffffu, r.stage == kStageDone);
      }
      // write back what this mode can have changed (the rest need not stay live through the branch)
      __syncwarp();
      if (lane == 0) {
        SchedCursor &d = sched_cursor[warp];
        d.cur = s.cur; d.cursor = s.cursor; d.cur_count = s.cur_count;
        d.chunk_cur = s.chunk_cur; d.chunk_next = s.chunk_next; d.parity = s.parity;
        if constexpr (GATHER) {
          d.run_base = s.run_base; d.run_next = s.run_next; d.run_end = s.run_end;
          d.pend_base = s.pend_base; d.tk = s.tk;
        }
        if constexpr (kSplit) d.split_phase = s.split_phase;
      }
      __syncwarp();
    }
    if (idle == 0xffffffffu) break;  // no lane active and nothing left to hand out
    if constexpr (kBulkTets) {
      const unsigned act = ~idle;
      if (lane == __ffs(act) - 1) mbar_expect_tx(bar_row, 128u * __popc(act));
      if (r.stage != kStageDone) bulk_g2s_hint(row, P.tets + r.e, 128u, bar_row, l2_policy_keep_now());
      mbar_wait(bar_row, row_parity);
      row_parity ^= 1u;
    }
    if constexpr (kCoop) {  // warp-collective: the idle lanes help fetch the active lanes' records
      const auto sl = walk_lane<NS, BLOCK, TM>(P, &score_wl[0][0], &time_bin[0]);
      coop_plane_step<NS, TM, MO, CU, MU>(P, r, c, ~idle, smem_u32(&coop_rows[warp][0]), tgt, &lane_ids[threadIdx.x],
                                          NS > 0 ? &sl : nullptr);
    } else if (r.stage != kStageDone) {
      if constexpr (FETCH == kFetchEdge) {
        edge_persist_step(P, my_i, r, g, c, l2_policy_keep_now(), tgt);
      } else if constexpr (kRows) {
        ExitScan sc;
        double raw[16];
#pragma unroll
        for (int j = 0; j < 8; ++j)
          asm volatile("ld.shared.v2.f64 {%0,%1}, [%2];"
                       : "=d"(raw[2 * j]), "=d"(raw[2 * j + 1])
                       : "r"(row + 16 * j));
        scan_record(raw, r.e, r.ox, r.oy, r.oz, r.ux, r.uy, r.uz, sc);
        advance(P, my_i, r, exit_parameter(sc), sc.nbr, sc.back, c, true);
      } else if constexpr (FETCH == kFetchLean || FETCH == kFetchLeanL1) {
        plane_step_lean<FETCH>(P, my_i, r, c, l2_policy_keep_now());
      } else {
        const auto sl = walk_lane<NS, BLOCK, TM>(P, &score_wl[0][0], &time_bin[0]);
        plane_step<FETCH == kFetchCoopL1 ? kFetchPolicyL1 : FETCH, NS, TM, MO, CU, MU>(
            P, r, c, FETCH != kFetchPlain ? l2_policy_keep_now() : 0, tgt, &lane_ids[kTargetSlot ? threadIdx.x : 0],
            NS > 0 ? &sl : nullptr);
      }
    }
  }
  flush_counters(P, c);
}
