// Host-side engine template instantiated once per curve (inst_*.cu): workspace management, plan
// selection, launches, error mapping.  No CPU compute path exists.
#pragma once
#include "context.h"
#include "msm.cuh"

namespace nmsm {

// ---------------------------------------------------------------------------------------------
// MSM driver
// ---------------------------------------------------------------------------------------------
inline unsigned int cdiv(uint64_t a, unsigned int b) { return (unsigned int)((a + b - 1) / b); }

#define EV(slot)                                                         \
  do {                                                                   \
    if (g_ctx.profiling) cudaEventRecord(C.ev[slot], C.stream);              \
  } while (0)

template <class Cv>
struct Engine {
  using G = typename Cv::G;

// Runs the pipeline on device-resident canonical inputs.  If d_out_acc != nullptr the raw
// accumulator is written there and no affine result is produced.
// `d_prepared` != nullptr: points were validated and prepared once by prepare_points() (device-resident
// handle, nmsm_points_upload); k_prepare is skipped.
// `table_c` != 0: d_prepared holds table_digits(table_c) levels of `table_points` points each (precompute_table).
static int run_msm(const uint32_t* d_pts, const uint32_t* d_scalars, uint64_t n, uint32_t* d_out_acc,
                   uint8_t* out_xy, int* out_is_inf, const uint32_t* d_prepared = nullptr, int table_c = 0,
                   uint64_t table_points = 0) {
  if (int r = submit_msm(d_pts, d_scalars, n, d_out_acc, d_prepared, table_c, table_points)) return r;
  return collect_msm(out_xy, out_is_inf);
}

// chunks per logical thread (quad) of a k_reduce2 pass over `chunks` chunks per window.  A pass that fits one block
// (the last one) spreads its chunks over as many of the 32 quads as it can: the serial part of the chain is 3 additions
// per chunk.  A multi-block pass takes 4 chunks per quad, or up to 16 when that leaves <= REDUCE2_MAX_SPLITS block
// results (one more pass then finishes; every pass is a latency-bound launch).
static int reduce2_r(uint64_t chunks) {
  if (chunks <= (uint64_t)REDUCE2_LOGICAL * 4) {  // single block
    int r = 1;
    while ((uint64_t)REDUCE2_LOGICAL * r < chunks) r *= 2;
    return r;
  }
  int r = REDUCE2_R;
  while (r < 16 && (chunks + (uint64_t)REDUCE2_LOGICAL * r - 1) / ((uint64_t)REDUCE2_LOGICAL * r) > (uint64_t)REDUCE2_MAX_SPLITS &&
         chunks <= (uint64_t)REDUCE2_LOGICAL * 16 * REDUCE2_MAX_SPLITS)
    r *= 2;
  return r;
}

static constexpr int SHARD_MIN_C = 8;  // sharded MSMs: at most ceil(257 / 8) = 33 windows (MAX_WINDOWS), one group each

// How many window groups to pipeline.  Overlapping the bucket reduction and Horner chains of finished groups with the
// accumulation of the rest does not shorten one MSM: the latency-bound tail kernels share every SM sub-partition with
// 4 accumulate warps and run several times slower, the accumulation loses the pipe time they take, and the last group's
// tail stays on the critical path.  So one group is the default; nmsm_set_window_groups keeps
// the pipelined form available, and sharded MSMs use one group per window because that is what lets a window's bucket
// exchange overlap the accumulation of the next windows.
static int choose_groups(const MsmPlan& plan, uint64_t max_entries) {
  (void)max_entries;
  if (plan.W <= 1) return 1;
  int ng = 1;
  if (g_ctx.forced_groups) ng = g_ctx.forced_groups < plan.W ? g_ctx.forced_groups : plan.W;
  if (g_ctx.profiling) ng = 1;  // per-kernel event times only mean something on a linear pipeline
  return ng;
}

// k_prepare (and, for host inputs, the H2D copy of the points) on the slot's prep_stream, beside the scalar copy and the
// digit passes on the main stream?  Not while profiling: per-kernel event times need the linear pipeline.
static bool prepare_on_side_stream(uint64_t n, bool prepared) { return !g_ctx.profiling && !prepared && n >= (1u << 14); }

// H2D of host inputs: scalars first on the main stream (the digit passes only need them), the 3x larger point array on
// prep_stream where k_prepare follows it — the digit count / scan / scatter overlap the point copy.
static int stage_host_inputs(Slot& C, const void* pts, const void* scalars, uint64_t n) {
  CK(C.in_pts.ensure(n * G::IN_WORDS * 4));
  CK(C.in_scalars.ensure(n * SCALAR_WORDS * 4));
  // h2d_any: pinned sources are one DMA each; large pageable ones are staged through pinned chunks by worker threads
  if (int r = h2d_any(C.in_scalars.p, scalars, n * SCALAR_WORDS * 4, C.stream)) return r;
  return h2d_any(C.in_pts.p, pts, n * G::IN_WORDS * 4, prepare_on_side_stream(n, false) ? C.prep_stream : C.stream);
}

// Enqueue the whole pipeline (and the small result D2H); no host sync.
//
// Single GPU, one window group (the default, see choose_groups): everything on the slot's main stream, except k_prepare
// (and the point H2D of host inputs) on prep_stream beside the digit passes:
//   prepare | count, scan, scatter -> k_accumulate -> k_stitch_tiles x2 -> k_reduce1 -> k_reduce2 levels
//   -> k_horner_step -> k_combine (inversion to affine) -> D2H
// With NG > 1 groups (nmsm_set_window_groups; windows [w_lo, w_hi), top windows first):
//       acc_stream[g % 8]  (low priority)  k_accumulate of the group                      -> ev_acc[g]
//       tail_stream[g % 4] (high priority) stitch tiles, k_reduce1, k_reduce2 levels      -> ev_tail[g]
//       horner_stream      (high priority) k_horner_step: hacc = 2^(c * windows) * hacc + group sum
// all accumulate launches are issued before any tail work (streams may share a hardware queue).
//
// Sharded (multi-GPU) MSM, `shard` != nullptr (SURVEY §8e, BASELINE north_star "allreduce of the per-window bucket
// accumulators"): every GPU accumulates its n_local terms into the full W x B bucket array with the GLOBAL window
// size; window w is owned by rank w % world.  Default (bulk form, one group):
//   main stream   one k_accumulate over all windows, k_stitch_tiles, k_bucket_finalize (dense buckets)   -> ev_fin
//   comm stream   direct form: a 4-byte ncclAllGather as the barrier "my dense buckets are complete"     -> ev_xchg
//                 (copy form, NMSM_DIST_P2P=0: grouped ncclSend / ncclRecv of the dense windows to their owners)
//   per owned window, on its own tail stream:
//                 k_bucket_fold_peers — the owner PULLS every peer's partial buckets over NVLink inside the fold kernel
//                 (EC addition is not an NCCL reduction operator: exchange + fold) — k_reduce1_dense, k_reduce2 levels,
//                 k_horner_step with the window's weight 2^(c w)                                          -> ev_tail[w]
//   comm stream   ncclAllGather of every rank's weighted window sums (+ its validation words); k_combine folds them.
// With nmsm_set_window_groups(> 1): one group per window, top window first, the exchange of window w overlapping the
// accumulation of windows w-1..0 (slower than the bulk form for the reason given at choose_groups: DESIGN.md §6).
static int submit_msm(const uint32_t* d_pts, const uint32_t* d_scalars, uint64_t n, uint32_t* d_out_acc,
                      const uint32_t* d_prepared, int table_c = 0, uint64_t table_points = 0,
                      const ShardArgs* shard = nullptr) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (C.pend.active) return fail(NMSM_ERR_ARG, "slot busy: collect the previous MSM first");
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  if (shard && (!g_dist.ready || d_out_acc || d_prepared))
    return fail(NMSM_ERR_ARG, shard && !g_dist.ready ? "nmsm_dist_init has not been called" : "sharded MSM: unsupported combination");
  const uint64_t n_plan = shard ? shard->n_total : n;
  if (shard && (n_plan >= (1ull << 31) || shard->offset + n > n_plan)) return fail(NMSM_ERR_ARG, "sharded MSM: bad shard bounds");
  const int RES_WORDS = G::IN_WORDS + 4;  // xy | inf | err_pt | err_sc | pad   (then 2 words: accumulator starts, profiling)
  CK(C.result.ensure((RES_WORDS + 4) * 4));
  uint32_t* d_res = (uint32_t*)C.result.p;
  unsigned int* d_err = (unsigned int*)(d_res + G::IN_WORDS + 1);

  C.pend = Pending();
  C.pend.curve = Cv::ID;
  C.pend.n = n;
  C.pend.partial = d_out_acc != nullptr;
  if (n_plan == 0) {  // curve.ts:878 — empty input returns the identity (sharded: empty on every rank, no exchange)
    if (d_out_acc) {
      typename G::Acc id = G::identity();
      CK(cudaMemcpyAsync(d_out_acc, &id, sizeof(id), cudaMemcpyHostToDevice, C.stream));
      CK(cudaStreamSynchronize(C.stream));
    }
    C.pend.empty = true;
    C.pend.active = true;
    return NMSM_OK;
  }

  MsmPlan plan = table_c ? make_table_plan<Cv>(table_points, table_c, g_ctx.sm_count)
                         : make_plan<Cv>(n_plan, g_ctx.forced_c, g_ctx.sm_count, shard ? (n ? n : 1) : 0, shard ? SHARD_MIN_C : 2);
  if (shard && plan.W > MAX_WINDOWS) return fail(NMSM_ERR_ARG, "window count exceeds MAX_WINDOWS");
  if (shard && g_ctx.forced_groups > 1) plan_one_wave_per_window<Cv>(plan, n, g_ctx.sm_count);  // pipelined sharded form
  const uint64_t max_entries = (n ? n : 1) * (uint64_t)plan.D * split_of<Cv>();
  if (max_entries >= (1ull << 32)) return fail(NMSM_ERR_ARG, "n * windows must be < 2^32");
  // bucket reduction levels: every k_reduce2 pass shrinks the per-window chunk count by REDUCE2_CHUNKS_PER_BLOCK
  // until ONE block per window is left (two passes for the ordinary plans)
  size_t blk_entries = 0;
  for (uint64_t m = plan.chunks;;) {
    const uint64_t sp = (m + (uint64_t)REDUCE2_LOGICAL * reduce2_r(m) - 1) / ((uint64_t)REDUCE2_LOGICAL * reduce2_r(m));
    blk_entries += sp;
    if (sp <= 1) break;
    m = sp;
  }
  const uint64_t nseg = (uint64_t)plan.W * plan.TPW;  // accumulate segments, TPW per window

  if (!d_prepared) CK(C.aff.ensure((n ? n : 1) * split_of<Cv>() * G::AFF_WORDS * 4));
  CK(C.counts.ensure((size_t)(plan.G + 1) * 4));
  CK(C.offsets.ensure((size_t)(plan.G + 1) * 4));
  CK(C.cursor.ensure((size_t)(plan.G + 1) * 4));
  CK(C.sorted.ensure(max_entries * 4));
  CK(C.buckets.ensure((size_t)plan.G * G::ACC_WORDS * 4));
  CK(C.heads.ensure(nseg * G::ACC_WORDS * 4));
  CK(C.tails.ensure(nseg * G::ACC_WORDS * 4));
  CK(C.chunk_out.ensure((size_t)plan.W * plan.chunks * G::ACC_WORDS * 4 * 2));
  CK(C.tile_sums.ensure((size_t)(plan.G / SCAN_TILE + 2) * 4));
  const uint64_t ntile1 = nseg / STITCH_FAN, ntile2 = ntile1 / STITCH_FAN;  // nseg is a multiple of 1024
  CK(C.tiles.ensure((ntile1 + ntile2) * G::ACC_WORDS * 4));
  CK(C.blk.ensure((size_t)plan.W * blk_entries * G::ACC_WORDS * 4 * 2));
  CK(C.window_out.ensure((size_t)plan.W * G::ACC_WORDS * 4));
  CK(C.hacc.ensure((size_t)G::ACC_WORDS * 4));

  uint32_t* aff = d_prepared ? const_cast<uint32_t*>(d_prepared) : (uint32_t*)C.aff.p;
  unsigned int* counts = (unsigned int*)C.counts.p;
  uint32_t* offsets = (uint32_t*)C.offsets.p;
  unsigned int* cursor = (unsigned int*)C.cursor.p;
  uint32_t* sorted = (uint32_t*)C.sorted.p;
  uint32_t* buckets = (uint32_t*)C.buckets.p;
  uint32_t* heads = (uint32_t*)C.heads.p;
  uint32_t* tails = (uint32_t*)C.tails.p;
  uint32_t* sums = (uint32_t*)C.chunk_out.p;
  uint32_t* wsums = sums + (size_t)plan.W * plan.chunks * G::ACC_WORDS;
  uint32_t* tile_sums = (uint32_t*)C.tile_sums.p;
  uint32_t* tile1 = (uint32_t*)C.tiles.p;
  uint32_t* tile2 = tile1 + ntile1 * G::ACC_WORDS;
  uint32_t* window_out = (uint32_t*)C.window_out.p;
  uint32_t* hacc = (uint32_t*)C.hacc.p;
  cudaStream_t st = C.stream;
  const uint32_t n32 = (uint32_t)n;
  // sharded: one group per window (the exchange of window w overlaps the accumulation of the rest) or, the default, ONE
  // group (bulk: one accumulate launch at full efficiency, one exchange step for all windows).
  int NG = choose_groups(plan, max_entries);
  if (shard) {
    NG = g_ctx.forced_groups ? (g_ctx.forced_groups >= plan.W ? plan.W : g_ctx.forced_groups) : 1;
    if (NG > 1) NG = plan.W;  // pipelined form: exactly one window per group
  }
  static const int quad_env = getenv("NMSM_QUAD_REDUCE1") ? atoi(getenv("NMSM_QUAD_REDUCE1")) : 0;  // tuning experiment
  const bool quad_reduce1 = (quad_env == 1 && NG > 1) || quad_env == 2 || (quad_env == 0 && NG == 1 && reduce1_quad_form(plan));
  const bool prof = g_ctx.profiling && !shard;
  // sharded: which windows this rank owns, where their peers' buckets land, and the gather layout
  const int world = shard ? g_dist.world : 1, rank = shard ? g_dist.rank : 0;
  const int slots = (plan.W + world - 1) / world;                    // owned windows per rank (upper bound)
  const size_t WB = (size_t)plan.B * G::ACC_WORDS;                   // words of one window's dense bucket array
  const int gather_words = slots * G::ACC_WORDS + 4;                 // per rank: weighted window sums | err_pt err_sc off_lo off_hi
  uint32_t *recv = nullptr, *gsend = nullptr, *grecv = nullptr;
  bool p2p = shard && g_dist.p2p && world > 1;
  PeerPtrs peer_ptrs = {};
  if (shard) {
    if (p2p) {  // (re)map the peers' bucket arrays when this slot's own array moved (same call on every rank)
      if (int r = dist_map_peer_buckets(g_ctx.cur, C.buckets.p, C.comm_stream)) return r;
      p2p = g_dist.p2p;  // a peer that cannot be mapped turns the direct form off on every rank
      for (int r = 0; r < world && p2p; r++) peer_ptrs.p[r] = (const uint32_t*)g_dist.mapped[g_ctx.cur][r];
    }
    if (!p2p) CK(C.recv.ensure((size_t)slots * (world - 1) * WB * 4 + 16));
    CK(C.gsend.ensure((size_t)gather_words * 4));
    CK(C.grecv.ensure((size_t)gather_words * 4 * world + 256 + 4 * world));  // + scratch of the 4-byte barrier all-gathers
    recv = (uint32_t*)C.recv.p;
    gsend = (uint32_t*)C.gsend.p;
    grecv = (uint32_t*)C.grecv.p;
  }
  int launches = 0;
#define PEV(slot)                                   \
  do {                                              \
    if (prof) cudaEventRecord(C.ev[slot], st);      \
  } while (0)

  CK(cudaEventRecord(C.ev_t0, st));
  PEV(0);
  CK(cudaMemsetAsync(d_err, 0xff, 8, st));
  CK(cudaMemsetAsync(counts, 0, (size_t)(plan.G + 1) * 4, st));
  // k_prepare only feeds k_accumulate: outside profiling it runs on its own stream beside the digit passes
  const bool prep_aside = prepare_on_side_stream(n, d_prepared != nullptr);
  if (!d_prepared && n) {
    cudaStream_t sp = prep_aside ? C.prep_stream : st;
    if (prep_aside) {
      CK(cudaEventRecord(C.ev_start, st));
      CK(cudaStreamWaitEvent(sp, C.ev_start, 0));
    }
    k_prepare<Cv><<<cdiv(n, 128), 128, 0, sp>>>(d_pts, n32, aff, d_err);
    if (prep_aside) CK(cudaEventRecord(C.ev_prep, sp));
    launches++;
  }
  PEV(1);
  if (n) k_digits<Cv, false><<<cdiv(n, 256), 256, 0, st>>>(d_scalars, n32, plan, counts, nullptr, d_err);
  PEV(2);
  {
    const unsigned int tiles = cdiv(plan.G, SCAN_TILE);
    k_scan_tiles<<<tiles, SCAN_THREADS, 0, st>>>(counts, (uint32_t)plan.G, tile_sums);
    k_scan_apply<<<tiles, SCAN_THREADS, 0, st>>>(counts, (uint32_t)plan.G, tile_sums, offsets, cursor);
  }
  PEV(3);
  if (n) k_digits<Cv, true><<<cdiv(n, 256), 256, 0, st>>>(d_scalars, n32, plan, cursor, sorted, d_err);
  launches += 4;
  PEV(4);
  if (prof) {  // accounting only (not part of the timed kernels: between the scatter and the accumulate events)
    CK(cudaMemsetAsync(d_res + RES_WORDS, 0, 16, st));
    const uint64_t items = nseg > (uint64_t)plan.G ? nseg : (uint64_t)plan.G;
    k_count_starts<<<cdiv(items, 256), 256, 0, st>>>(offsets, plan, (unsigned long long*)(d_res + RES_WORDS));
    cudaEventRecord(C.ev[4], st);  // restart the accumulate interval after the counting kernel
  }
  if (shard) { k_set_identity<Cv><<<1, 32, 0, st>>>(gsend, slots); launches++; }
  if (prep_aside) CK(cudaStreamWaitEvent(st, C.ev_prep, 0));
  if (NG > 1) CK(cudaEventRecord(C.ev_fork, st));
  const bool trace = g_ctx.trace && (NG > 1 || shard);
  if (trace) cudaEventRecord(C.tr_fork, st);

  const int per = (plan.W + NG - 1) / NG;  // windows per group
  // Pass 1: every group's accumulate launch, top windows first.  They are issued before any tail work so that, should
  // two of the library's streams share a hardware work queue (CUDA_DEVICE_MAX_CONNECTIONS), an accumulate launch never
  // sits behind a tail kernel that is still waiting for an earlier group.
  int ngroups = 0;
  for (int w_hi = plan.W; w_hi > 0; w_hi -= per, ngroups++) {
    const int w_lo = w_hi > per ? w_hi - per : 0;
    const uint32_t nw = (uint32_t)(w_hi - w_lo);
    cudaStream_t sa = NG > 1 ? C.acc_stream[ngroups % ACC_STREAMS] : st;
    if (NG > 1 && ngroups < ACC_STREAMS) CK(cudaStreamWaitEvent(sa, C.ev_fork, 0));
    k_accumulate<Cv><<<cdiv((uint64_t)nw * plan.TPW, 128), 128, 0, sa>>>(aff, sorted, offsets, plan, (uint32_t)w_lo, buckets,
                                                                         heads, tails);
    if (NG > 1) CK(cudaEventRecord(C.ev_acc[ngroups], sa));
    if (trace) cudaEventRecord(C.tr_acc[ngroups], sa);
  }
  // Pass 2 (sharded): per group — dense buckets, exchange with the window owners, owner fold + reduction + weight
  if (shard) {
    const size_t smem2 = (REDUCE2_THREADS / 32) * G::ACC_WORDS * 4;
    int g = 0;
    for (int w_hi = plan.W; w_hi > 0; w_hi -= per, g++) {
      const int w_lo = w_hi > per ? w_hi - per : 0;
      cudaStream_t stl = NG > 1 ? C.tail_stream[g % TAIL_STREAMS] : st;
      if (NG > 1) CK(cudaStreamWaitEvent(stl, C.ev_acc[g], 0));
      {  // tile sums for buckets spanning many accumulate segments (no-ops for ordinary inputs), then the dense bucket arrays
        const uint32_t a0 = (uint32_t)((uint64_t)w_lo * plan.TPW / STITCH_FAN), a1 = (uint32_t)((uint64_t)w_hi * plan.TPW / STITCH_FAN);
        k_stitch_tiles<Cv><<<cdiv((uint64_t)(a1 - a0) * 32, 128), 128, 0, stl>>>(offsets, plan, STITCH_FAN, a0, a1, heads, tile1);
        const uint32_t b0 = a0 / STITCH_FAN, b1 = a1 / STITCH_FAN;
        k_stitch_tiles<Cv><<<cdiv((uint64_t)(b1 - b0) * 32, 128), 128, 0, stl>>>(offsets, plan, STITCH_FAN * STITCH_FAN, b0, b1,
                                                                                tile1, tile2);
        k_bucket_finalize<Cv><<<cdiv((uint64_t)(w_hi - w_lo) * plan.B, 128), 128, 0, stl>>>(
            offsets, buckets, heads, tails, tile1, tile2, plan, (uint32_t)w_lo * plan.B, (uint32_t)w_hi * plan.B);
        launches += 3;
      }
      if (world > 1 && p2p) {
        // direct exchange: the owners pull the peers' partial buckets inside k_bucket_fold_peers.  All that has to cross
        // the ranks here is "my dense buckets of this group are complete": a 4-byte all-gather as the barrier.
        CK(cudaEventRecord(C.ev_fin[g], stl));
        CK(cudaStreamWaitEvent(C.comm_stream, C.ev_fin[g], 0));
        if (nccl_all_gather(grecv + (size_t)gather_words * world + 16, grecv + (size_t)gather_words * world + 32, 4, C.comm_stream))
          return NMSM_ERR_CUDA;
        CK(cudaEventRecord(C.ev_xchg[g], C.comm_stream));
        if (trace) cudaEventRecord(C.tr_h[g], C.comm_stream);
      } else if (world > 1) {  // copies: the window owners receive every peer's partial buckets; everybody else sends
        CK(cudaEventRecord(C.ev_fin[g], stl));
        CK(cudaStreamWaitEvent(C.comm_stream, C.ev_fin[g], 0));
        if (nccl_group_start()) return NMSM_ERR_CUDA;
        for (int w = w_hi - 1; w >= w_lo; w--) {
          const int own_rank = w % world;
          if (own_rank == rank) {
            uint32_t* wrecv = recv + (size_t)(w / world) * (world - 1) * WB;
            for (int r = 0, k = 0; r < world; r++)
              if (r != rank && nccl_recv(wrecv + (size_t)(k++) * WB, WB * 4, r, C.comm_stream)) return NMSM_ERR_CUDA;
          } else if (nccl_send(buckets + (size_t)w * WB, WB * 4, own_rank, C.comm_stream)) {
            return NMSM_ERR_CUDA;
          }
        }
        if (nccl_group_end()) return NMSM_ERR_CUDA;
        CK(cudaEventRecord(C.ev_xchg[g], C.comm_stream));
        if (trace) cudaEventRecord(C.tr_h[g], C.comm_stream);
      } else {
        CK(cudaEventRecord(C.ev_xchg[g], stl));
      }
      if (trace) cudaEventRecord(C.tr_tail[g], stl);
      // owned windows of the group: independent chains on the tail streams
      for (int w = w_hi - 1; w >= w_lo; w--) {
        if (w % world != rank) continue;
        const int slot = w / world;
        cudaStream_t so = C.tail_stream[slot % TAIL_STREAMS];
        CK(cudaStreamWaitEvent(so, C.ev_xchg[g], 0));
        uint32_t* wb = buckets + (size_t)w * WB;
        if (world > 1 && p2p) {
          k_bucket_fold_peers<Cv><<<cdiv((uint64_t)plan.B * 4, 128), 128, 0, so>>>(wb, peer_ptrs, (size_t)w * WB, world, rank,
                                                                                (uint32_t)plan.B);
          launches++;
        } else if (world > 1) {
          k_bucket_fold<Cv><<<cdiv((uint64_t)plan.B * 4, 128), 128, 0, so>>>(wb, recv + (size_t)slot * (world - 1) * WB, world - 1, WB,
                                                                          (uint32_t)plan.B);
          launches++;
        }
        const uint32_t id0 = (uint32_t)w * plan.chunks, id1 = id0 + plan.chunks;
        k_reduce1_dense<Cv><<<cdiv((uint64_t)(id1 - id0) * 4, REDUCE1_THREADS), REDUCE1_THREADS, 0, so>>>(buckets, plan, id0, id1, sums,
                                                                                                    wsums);
        launches++;
        MsmPlan pl = plan;
        const uint32_t *S = sums, *T = wsums;
        uint32_t* base = (uint32_t*)C.blk.p;
        for (;;) {
          const int R2 = reduce2_r(pl.chunks), per_block = REDUCE2_LOGICAL * R2;
          const int splits = (pl.chunks + per_block - 1) / per_block;
          uint32_t* blkP = base;
          uint32_t* blkQ = base + (size_t)plan.W * splits * G::ACC_WORDS;
          base = blkQ + (size_t)plan.W * splits * G::ACC_WORDS;
          k_reduce2<Cv><<<dim3(splits, 1), REDUCE2_THREADS, smem2, so>>>(S, T, pl, R2, (uint32_t)w, blkP, blkQ,
                                                                         splits == 1 ? window_out : nullptr);
          launches++;
          if (splits == 1) break;
          S = blkQ;
          T = blkP;
          pl.chunks = splits;
          pl.K *= per_block;
        }
        // weighted window sum 2^(c w) S_w straight into its gather slot
        k_horner_step<Cv><<<1, 32, 0, so>>>(window_out, plan, w, w + 1, 1, 1, gsend + (size_t)slot * G::ACC_WORDS);
        launches++;
        CK(cudaEventRecord(C.ev_tail[w], so));
        if (trace && w < 16) cudaEventRecord(C.tr_acc[17 + w], so);
      }
    }
    ngroups = g;
  }
  // Pass 2 (single GPU): per group, the bucket reduction and the Horner step
  int g = 0;
  for (int w_hi = plan.W; w_hi > 0 && !shard; w_hi -= per, g++) {
    const int w_lo = w_hi > per ? w_hi - per : 0;
    const uint32_t nw = (uint32_t)(w_hi - w_lo);
    cudaStream_t stl = NG > 1 ? C.tail_stream[g % TAIL_STREAMS] : st;
    cudaStream_t sh = NG > 1 ? C.horner_stream : st;
    if (NG > 1) CK(cudaStreamWaitEvent(stl, C.ev_acc[g], 0));
    PEV(5);
    {  // tile sums for buckets spanning many accumulate segments (no-ops for ordinary inputs)
      const uint32_t a0 = (uint32_t)((uint64_t)w_lo * plan.TPW / STITCH_FAN), a1 = (uint32_t)((uint64_t)w_hi * plan.TPW / STITCH_FAN);
      k_stitch_tiles<Cv><<<cdiv((uint64_t)(a1 - a0) * 32, 128), 128, 0, stl>>>(offsets, plan, STITCH_FAN, a0, a1, heads, tile1);
      const uint32_t b0 = a0 / STITCH_FAN, b1 = a1 / STITCH_FAN;
      k_stitch_tiles<Cv><<<cdiv((uint64_t)(b1 - b0) * 32, 128), 128, 0, stl>>>(offsets, plan, STITCH_FAN * STITCH_FAN, b0, b1,
                                                                              tile1, tile2);
    }
    PEV(6);
    {
      const uint32_t id0 = (uint32_t)w_lo * plan.chunks, id1 = (uint32_t)w_hi * plan.chunks;
      if (quad_reduce1 && w_lo == 0)  // last group: its chain is the critical path, run it in the latency form
        k_reduce1<Cv, true><<<cdiv((uint64_t)(id1 - id0) * 4, REDUCE1_THREADS), REDUCE1_THREADS, 0, stl>>>(
            offsets, buckets, heads, tails, tile1, tile2, plan, id0, id1, sums, wsums);
      else
        k_reduce1<Cv, false><<<cdiv(id1 - id0, REDUCE1_THREADS), REDUCE1_THREADS, 0, stl>>>(offsets, buckets, heads, tails,
                                                                                           tile1, tile2, plan, id0, id1, sums, wsums);
    }
    PEV(7);
    launches += 4;
    {
      // msm.cuh "Bucket reduction": P/Q of one level are the T/S of the next (chunks := splits, K := K * Mb)
      const size_t smem2 = (REDUCE2_THREADS / 32) * G::ACC_WORDS * 4;
      MsmPlan pl = plan;
      const uint32_t *S = sums, *T = wsums;
      uint32_t* base = (uint32_t*)C.blk.p;
      for (;;) {
        const int R2 = reduce2_r(pl.chunks), per_block = REDUCE2_LOGICAL * R2;
        const int splits = (pl.chunks + per_block - 1) / per_block;
        uint32_t* blkP = base;
        uint32_t* blkQ = base + (size_t)plan.W * splits * G::ACC_WORDS;
        base = blkQ + (size_t)plan.W * splits * G::ACC_WORDS;
        k_reduce2<Cv><<<dim3(splits, nw), REDUCE2_THREADS, smem2, stl>>>(S, T, pl, R2, (uint32_t)w_lo, blkP, blkQ,
                                                                         splits == 1 ? window_out : nullptr);
        launches++;
        if (splits == 1) break;
        S = blkQ;
        T = blkP;
        pl.chunks = splits;
        pl.K *= per_block;
      }
    }
    PEV(8);
    if (NG > 1) {
      CK(cudaEventRecord(C.ev_tail[g], stl));
      CK(cudaStreamWaitEvent(sh, C.ev_tail[g], 0));
    }
    if (trace) cudaEventRecord(C.tr_tail[g], stl);
    k_horner_step<Cv><<<1, 32, 0, sh>>>(window_out, plan, w_lo, w_hi, g == 0 ? 1 : 0, 0, hacc);
    if (trace) cudaEventRecord(C.tr_h[g], sh);
    launches++;
  }
  if (shard) g = ngroups;
  if (shard) {
    cudaStream_t sc = world > 1 ? C.comm_stream : st;
    for (int w = rank; w < plan.W; w += world) CK(cudaStreamWaitEvent(sc, C.ev_tail[w], 0));  // every owned window's chain
    k_pack_shard_tail<<<1, 32, 0, sc>>>(gsend + (size_t)slots * G::ACC_WORDS, d_err, shard->offset);
    if (world > 1) {
      if (nccl_all_gather(gsend, grecv, (size_t)gather_words * 4, sc)) return NMSM_ERR_CUDA;
      CK(cudaEventRecord(C.ev_gather, sc));
      CK(cudaStreamWaitEvent(st, C.ev_gather, 0));
    } else {
      CK(cudaMemcpyAsync(grecv, gsend, (size_t)gather_words * 4, cudaMemcpyDeviceToDevice, sc));
      if (sc != st) {
        CK(cudaEventRecord(C.ev_gather, sc));
        CK(cudaStreamWaitEvent(st, C.ev_gather, 0));
      }
    }
    k_combine<Cv, true><<<1, 32, 0, st>>>(grecv, world * slots, slots, gather_words, d_res, d_res + G::IN_WORDS);
    launches += 2;
    CK(cudaMemcpyAsync(C.h_gather, grecv, (size_t)gather_words * 4 * world, cudaMemcpyDeviceToHost, st));
  } else {
    if (NG > 1) {
      CK(cudaEventRecord(C.ev_horner, C.horner_stream));
      CK(cudaStreamWaitEvent(st, C.ev_horner, 0));
    }
    if (d_out_acc)
      k_combine<Cv, false><<<1, 32, 0, st>>>(hacc, 1, 1, 0, d_out_acc, nullptr);
    else
      k_combine<Cv, true><<<1, 32, 0, st>>>(hacc, 1, 1, 0, d_res, d_res + G::IN_WORDS);
    launches++;
  }
  PEV(9);
#undef PEV
  CK(cudaEventRecord(C.ev_t1, st));
  CK(cudaGetLastError());
  // one small D2H: result + error slots (+ entry count for accounting)
  CK(cudaMemcpyAsync(C.h_result, d_res, RES_WORDS * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(C.h_result + RES_WORDS, offsets + plan.G, 4, cudaMemcpyDeviceToHost, st));
  if (prof) CK(cudaMemcpyAsync(C.h_result + RES_WORDS + 2, d_res + RES_WORDS, 16, cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(C.done, st));
  C.pend.plan = MsmPlanLite{plan.c, plan.W, plan.B, plan.G, plan.L, plan.K, plan.chunks, plan.D, plan.TPW};
  C.pend.profiled = prof;
  C.pend.sharded = shard != nullptr;
  C.pend.gather_words = gather_words;
  C.pend.groups = g;
  C.pend.launches = launches;
  C.pend.active = true;
  return NMSM_OK;
}

// Wait for the slot's MSM, map device-side validation errors, hand out the result and the timings.
static int collect_msm(uint8_t* out_xy, int* out_is_inf) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (!C.pend.active) return fail(NMSM_ERR_ARG, "nothing submitted on this slot");
  C.pend.active = false;
  if (C.pend.empty) {
    if (!C.pend.partial) {
      memset(out_xy, 0, G::IN_WORDS * 4);
      if (G::IS_EDWARDS) out_xy[G::COORD_WORDS * 4] = 1;  // (0, 1)
      *out_is_inf = 1;
    }
    return NMSM_OK;
  }
  const int RES_WORDS = G::IN_WORDS + 4;
  CK(cudaEventSynchronize(C.done));
  MsmPlan plan;
  plan.c = C.pend.plan.c; plan.W = C.pend.plan.W; plan.B = C.pend.plan.B; plan.G = C.pend.plan.G;
  plan.L = C.pend.plan.L; plan.K = C.pend.plan.K; plan.chunks = C.pend.plan.chunks; plan.D = C.pend.plan.D;
  const bool partial = C.pend.partial;

  uint64_t err_pt = C.h_result[G::IN_WORDS + 1], err_sc = C.h_result[G::IN_WORDS + 2];
  if (err_pt == 0xffffffffu) err_pt = ~0ull;
  if (err_sc == 0xffffffffu) err_sc = ~0ull;
  if (C.pend.sharded) {  // every rank's validation words came with the gather: report the smallest GLOBAL index
    err_pt = err_sc = ~0ull;
    const int slots_words = C.pend.gather_words - 4;
    for (int r = 0; r < g_dist.world; r++) {
      const uint32_t* t = C.h_gather + (size_t)r * C.pend.gather_words + slots_words;
      const uint64_t off = (uint64_t)t[2] | ((uint64_t)t[3] << 32);
      if (t[0] != 0xffffffffu && off + t[0] < err_pt) err_pt = off + t[0];
      if (t[1] != 0xffffffffu && off + t[1] < err_sc) err_sc = off + t[1];
    }
  }
  // the reference validates all points before any scalar (curve.ts:871-872)
  if (err_pt != ~0ull) return fail(NMSM_ERR_POINT, "invalid point at index " + std::to_string(err_pt), (long long)err_pt);
  if (err_sc != ~0ull) return fail(NMSM_ERR_SCALAR, "invalid scalar at index " + std::to_string(err_sc), (long long)err_sc);

  const uint64_t entries = C.h_result[RES_WORDS];
  C.last_info.c = plan.c;
  C.last_info.windows = plan.W;
  C.last_info.buckets_per_window = plan.B;
  C.last_info.entries_per_thread = plan.L;
  C.last_info.reduce_chunk = plan.K;
  C.last_info.sorted_entries = entries;
  C.last_info.modmul_equiv = plan_modmuls<Cv>(plan, entries);
  C.last_info.bucket_starts = C.pend.profiled ? ((uint64_t)C.h_result[RES_WORDS + 2] | ((uint64_t)C.h_result[RES_WORDS + 3] << 32)) : 0;
  C.last_info.bucket_pairs = (C.pend.profiled && NMSM_PAIRED && !G::IS_EDWARDS)
                                 ? ((uint64_t)C.h_result[RES_WORDS + 4] | ((uint64_t)C.h_result[RES_WORDS + 5] << 32)) : 0;
  C.last_info.accumulate_threads = C.pend.profiled ? (entries + plan.L - 1) / plan.L : 0;
  C.last_info.launches = C.pend.launches;
  C.last_info.window_groups = C.pend.groups;
  memset(C.last_ms, 0, sizeof(C.last_ms));
  if (C.pend.profiled)  // events were recorded at submit (not: whatever the profiling switch says now)
    for (int k = 0; k < 9; k++)
      if (cudaEventElapsedTime(&C.last_ms[k], C.ev[k], C.ev[k + 1]) != cudaSuccess) C.last_ms[k] = 0;
  if (cudaEventElapsedTime(&C.last_ms[NMSM_T_TOTAL], C.ev_t0, C.ev_t1) != cudaSuccess) C.last_ms[NMSM_T_TOTAL] = 0;
  (void)cudaGetLastError();
  if (g_ctx.trace && (C.pend.groups > 1 || C.pend.sharded)) {
    float f = 0, a = 0, t = 0, h = 0, tot = C.last_ms[NMSM_T_TOTAL];
    cudaEventElapsedTime(&f, C.ev_t0, C.tr_fork);
    fprintf(stderr, "[nmsm trace%s rank %d] fork %.3f total %.3f |", C.pend.sharded ? " sharded" : "", g_dist.rank, f, tot);
    for (int k = 0; k < C.pend.groups; k++) {
      a = t = h = -1;
      cudaEventElapsedTime(&a, C.ev_t0, C.tr_acc[k]);
      cudaEventElapsedTime(&t, C.ev_t0, C.tr_tail[k]);
      if (!C.pend.sharded || g_dist.world > 1) cudaEventElapsedTime(&h, C.ev_t0, C.tr_h[k]);
      fprintf(stderr, " g%d acc %.3f %s %.3f %s %.3f |", k, a, C.pend.sharded ? "dense" : "tail", t, C.pend.sharded ? "xchg" : "horner", h);
    }
    if (C.pend.sharded)
      for (int w = g_dist.rank; w < C.pend.plan.W && w < 16; w += g_dist.world) {
        a = -1;
        cudaEventElapsedTime(&a, C.ev_t0, C.tr_acc[17 + w]);
        fprintf(stderr, " own w%d done %.3f |", w, a);
      }
    fprintf(stderr, "\n");
    (void)cudaGetLastError();
  }
  memcpy(g_ctx.last_ms, C.last_ms, sizeof(C.last_ms));
  g_ctx.last_info = C.last_info;
  if (!partial) {
    memcpy(out_xy, C.h_result, G::IN_WORDS * 4);
    *out_is_inf = (int)C.h_result[G::IN_WORDS];
  }
  return NMSM_OK;
}

// single-kernel calls (multiply batches): device time of the kernel between ev[0] and ev[1] -> NMSM_T_TOTAL
static void note_kernel_time(Slot& C) {
  if (!g_ctx.profiling) return;  // same lock-protected call that recorded ev[0] / ev[1]
  memset(C.last_ms, 0, sizeof(C.last_ms));
  if (cudaEventElapsedTime(&C.last_ms[NMSM_T_TOTAL], C.ev[0], C.ev[1]) != cudaSuccess) (void)cudaGetLastError();
  memcpy(g_ctx.last_ms, C.last_ms, sizeof(C.last_ms));
}

// C-ABI asynchronous halves (nmsm_msm_submit / nmsm_msm_collect)
static int submit_any(const void* pts, const void* scalars, uint64_t n, int inputs_on_device, void* d_out_acc,
                      const ShardArgs* shard) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (C.pend.active) return fail(NMSM_ERR_ARG, "slot busy: collect the previous MSM first");
  if (d_out_acc && !inputs_on_device) return fail(NMSM_ERR_ARG, "raw-accumulator output needs device-resident inputs");
  if (inputs_on_device || n == 0)
    return submit_msm((const uint32_t*)pts, (const uint32_t*)scalars, n, (uint32_t*)d_out_acc, nullptr, 0, 0, shard);
  if (int r = stage_host_inputs(C, pts, scalars, n)) return r;
  return submit_msm((const uint32_t*)C.in_pts.p, (const uint32_t*)C.in_scalars.p, n, nullptr, nullptr, 0, 0, shard);
}

// Upload + validate + prepare a point set once (fixed-base reuse; the device-resident analogue of the
// reference's captured tables in interleavedMSMUnsafe, curve.ts:937-959).  Returns a device buffer.
static int prepare_points(const uint8_t* pts, uint64_t n, uint32_t** out_dev) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (n == 0 || n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be in [1, 2^31)");
  uint32_t* d_aff = nullptr;
  CK(cudaMalloc((void**)&d_aff, n * split_of<Cv>() * G::AFF_WORDS * 4));
  cudaError_t e1 = C.in_pts.ensure(n * G::IN_WORDS * 4);
  cudaError_t e2 = C.result.ensure((G::IN_WORDS + 4) * 4);
  if (e1 != cudaSuccess || e2 != cudaSuccess) { cudaFree(d_aff); return cuda_fail(e1 != cudaSuccess ? e1 : e2, "workspace"); }
  unsigned int* d_err = (unsigned int*)C.result.p;
  cudaMemcpyAsync(C.in_pts.p, pts, n * G::IN_WORDS * 4, cudaMemcpyHostToDevice, C.stream);
  cudaMemsetAsync(d_err, 0xff, 8, C.stream);
  k_prepare<Cv><<<cdiv(n, 128), 128, 0, C.stream>>>((const uint32_t*)C.in_pts.p, (uint32_t)n, d_aff, d_err);
  unsigned int err[2] = {0, 0};
  cudaMemcpyAsync(err, d_err, 8, cudaMemcpyDeviceToHost, C.stream);
  cudaError_t e = cudaStreamSynchronize(C.stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { cudaFree(d_aff); return cuda_fail(e, "prepare_points"); }
  if (err[0] != 0xffffffffu) {
    cudaFree(d_aff);
    return fail(NMSM_ERR_POINT, "invalid point at index " + std::to_string(err[0]), err[0]);
  }
  *out_dev = d_aff;
  return NMSM_OK;
}

// MSM of host scalars against a prepared point set (scalars beyond the set are an error; fewer
// scalars use the first n_scalars points, like interleavedMSMUnsafe's trailing zeros).
static int run_msm_prepared(const uint32_t* d_prepared, uint64_t n_points, int table_c, const uint8_t* scalars,
                            uint64_t n, uint8_t* out_xy, int* out_is_inf) {
  if (int r = submit_prepared(d_prepared, n_points, table_c, scalars, n, 0)) return r;
  return collect_msm(out_xy, out_is_inf);
}

// asynchronous half (nmsm_msm_points_submit): scalars from the host (copied on the slot's stream) or the device
static int submit_prepared(const uint32_t* d_prepared, uint64_t n_points, int table_c, const void* scalars, uint64_t n,
                           int scalars_on_device) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (C.pend.active) return fail(NMSM_ERR_ARG, "slot busy: collect the previous MSM first");
  if (n > n_points) return fail(NMSM_ERR_LENGTH, "array of scalars must not be larger than array of points");
  if (Cv::GLV && n != n_points)
    return fail(NMSM_ERR_ARG, "this curve's prepared sets interleave P and phi(P): pass one scalar per point");
  const uint32_t* d_scalars = (const uint32_t*)scalars;
  if (n && !scalars_on_device) {
    CK(C.in_scalars.ensure(n * SCALAR_WORDS * 4));
    CK(cudaMemcpyAsync(C.in_scalars.p, scalars, n * SCALAR_WORDS * 4, cudaMemcpyHostToDevice, C.stream));
    d_scalars = (const uint32_t*)C.in_scalars.p;
  }
  return submit_msm(nullptr, d_scalars, n, nullptr, d_prepared, table_c, n_points);
}

// Fixed-base table for a prepared set: levels j = 0..D-1 hold 2^(c*j) * P_i (and 2^(c*j) * phi(P_i) for the GLV
// curves), each level in the prepared affine layout.  The device-resident counterpart of the per-point wNAF
// tables interleavedMSMUnsafe captures (curve.ts:937-959) and of Point.precompute (curve.ts:532-577): built once,
// every later MSM over the set needs one bucket window instead of W and no Horner doublings.
static int precompute_table(uint32_t** d_prepared, uint64_t n_points, int c_req, int* out_c, int* out_levels) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  const uint64_t terms = n_points * split_of<Cv>();
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if (c_req != 0 && (c_req < 4 || c_req > MAX_TABLE_BITS))
    return fail(NMSM_ERR_ARG, "table window bits must be 0 (automatic) or in [4, 22]");
  // the request is an upper bound on the digit width; the scalar bits are then spread evenly over the digits
  const int c = c_req ? canonical_table_bits<Cv>(c_req) : choose_table_bits<Cv>(n_points, g_ctx.sm_count, 0.5 * (double)free_b);
  const MsmPlan tp = make_table_plan<Cv>(n_points, c, g_ctx.sm_count);
  const int D = tp.D;
  if (terms * (uint64_t)D >= (1ull << 31)) return fail(NMSM_ERR_ARG, "points * levels must be < 2^31");
  const size_t level_bytes = (size_t)terms * G::AFF_WORDS * 4;
  uint32_t* tbl = nullptr;
  CK(cudaMalloc((void**)&tbl, level_bytes * D));
  cudaMemcpyAsync(tbl, *d_prepared, level_bytes, cudaMemcpyDeviceToDevice, C.stream);
  for (int j = 1; j < D; j++)
    k_table_level<Cv><<<cdiv(terms, 128), 128, 0, C.stream>>>(tbl + (size_t)(j - 1) * terms * G::AFF_WORDS,
                                                               tbl + (size_t)j * terms * G::AFF_WORDS, (uint32_t)terms,
                                                               digit_width(tp, j - 1));
  cudaError_t e = cudaStreamSynchronize(C.stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { cudaFree(tbl); return cuda_fail(e, "precompute_table"); }
  cudaFree(*d_prepared);
  *d_prepared = tbl;
  *out_c = c;
  *out_levels = D;
  return NMSM_OK;
}

// Fixed-point table (nmsm_point_table_create): validate P, level 0 = d*P (d <= 2^15), then levels 2^(16 j).
static int build_point_table(const uint8_t* point_xy, uint32_t** out_tbl, int* out_levels) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  constexpr int LV = point_table_levels<Cv>();
  uint32_t in[G::IN_WORDS];
  memcpy(in, point_xy, sizeof(in));
  if (!G::input_in_range(in)) return fail(NMSM_ERR_POINT, "invalid point at index 0", 0);
  CK(C.in_pts.ensure(G::IN_WORDS * 4));
  CK(C.aff.ensure((size_t)split_of<Cv>() * G::AFF_WORDS * 4));
  CK(C.result.ensure((G::IN_WORDS + 4) * 4));
  unsigned int* d_err = (unsigned int*)C.result.p;
  uint32_t* tbl = nullptr;
  const size_t level_words = (size_t)PT_HALF * G::AFF_WORDS;
  CK(cudaMalloc((void**)&tbl, level_words * 4 * LV));
  cudaStream_t st = C.stream;
  cudaMemcpyAsync(C.in_pts.p, point_xy, G::IN_WORDS * 4, cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(d_err, 0xff, 8, st);
  k_prepare<Cv><<<1, 1, 0, st>>>((const uint32_t*)C.in_pts.p, 1u, (uint32_t*)C.aff.p, d_err);
  k_table_base<Cv><<<cdiv(PT_HALF, 128), 128, 0, st>>>((const uint32_t*)C.aff.p, tbl);
  for (int j = 1; j < LV; j++)
    k_table_level<Cv><<<cdiv(PT_HALF, 128), 128, 0, st>>>(tbl + (size_t)(j - 1) * level_words, tbl + (size_t)j * level_words,
                                                           PT_HALF, PT_BITS);
  cudaError_t e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { cudaFree(tbl); return cuda_fail(e, "build_point_table"); }
  *out_tbl = tbl;
  *out_levels = LV;
  return NMSM_OK;
}

// out[i] = scalars[i] * P through the table: the batch form of a precomputed point's multiply / multiplyUnsafe.
static int table_mul_batch(const uint32_t* tbl, const uint8_t* scalars, uint64_t n, int allow_zero, uint8_t* out_xy,
                           uint8_t* out_is_inf) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  CK(C.in_scalars.ensure(n * SCALAR_WORDS * 4));
  CK(C.mul_out.ensure(n * (G::IN_WORDS + 1) * 4 + 16));
  CK(C.result.ensure(64));
  unsigned int* d_err = (unsigned int*)C.result.p;
  uint32_t* d_xy = (uint32_t*)C.mul_out.p;
  uint32_t* d_inf = d_xy + n * G::IN_WORDS;
  cudaStream_t st = C.stream;
  CK(cudaMemcpyAsync(C.in_scalars.p, scalars, n * SCALAR_WORDS * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_err, 0xff, 8, st));
  EV(0);
  k_table_mul<Cv><<<cdiv(n, 128), 128, 0, st>>>(tbl, (const uint32_t*)C.in_scalars.p, (uint32_t)n, allow_zero, d_xy,
                                                   d_inf, d_err);
  EV(1);
  CK(cudaGetLastError());
  std::vector<uint32_t> inf(n);
  unsigned int err[2];
  CK(cudaMemcpyAsync(err, d_err, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(out_xy, d_xy, n * G::IN_WORDS * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(inf.data(), d_inf, n * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  note_kernel_time(C);
  if (err[1] != 0xffffffffu)
    return fail(NMSM_ERR_SCALAR, "invalid scalar: out of range (index " + std::to_string(err[1]) + ")", err[1]);
  for (uint64_t i = 0; i < n; i++) out_is_inf[i] = (uint8_t)inf[i];
  return NMSM_OK;
}

// out_ok[i] = (n * P_i == O): the batch form of isTorsionFree
static int run_torsion(const uint8_t* pts, uint64_t n, uint8_t* out_ok) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  CK(C.in_pts.ensure(n * G::IN_WORDS * 4));
  CK(C.mul_out.ensure(n + 16));
  CK(C.result.ensure(64));
  unsigned int* d_err = (unsigned int*)C.result.p;
  cudaStream_t st = C.stream;
  CK(cudaMemcpyAsync(C.in_pts.p, pts, n * G::IN_WORDS * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_err, 0xff, 8, st));
  EV(0);
  k_torsion<Cv><<<cdiv(n, 128), 128, 0, st>>>((const uint32_t*)C.in_pts.p, (uint32_t)n, (uint8_t*)C.mul_out.p, d_err);
  EV(1);
  CK(cudaGetLastError());
  unsigned int err[2];
  CK(cudaMemcpyAsync(err, d_err, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(out_ok, C.mul_out.p, n, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  note_kernel_time(C);
  if (err[0] != 0xffffffffu) return fail(NMSM_ERR_POINT, "invalid point at index " + std::to_string(err[0]), err[0]);
  return NMSM_OK;
}

// out_ok[i] = 1 iff pts[i] satisfies the curve equation (assertValidity's isValidXY)
static int run_on_curve(const uint8_t* pts, uint64_t n, uint8_t* out_ok) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  CK(C.in_pts.ensure(n * G::IN_WORDS * 4));
  CK(C.mul_out.ensure(n + 16));
  cudaStream_t st = C.stream;
  CK(cudaMemcpyAsync(C.in_pts.p, pts, n * G::IN_WORDS * 4, cudaMemcpyHostToDevice, st));
  k_on_curve<Cv><<<cdiv(n, 128), 128, 0, st>>>((const uint32_t*)C.in_pts.p, (uint32_t)n, (uint8_t*)C.mul_out.p);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out_ok, C.mul_out.p, n, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return NMSM_OK;
}

static int run_msm_dev(const uint32_t* d_pts, const uint32_t* d_scalars, uint64_t n, uint32_t* d_out_acc,
                       uint8_t* out_xy, int* out_is_inf) {
  return run_msm(d_pts, d_scalars, n, d_out_acc, out_xy, out_is_inf, nullptr);
}

static int run_msm_host(const uint8_t* pts, const uint8_t* scalars, uint64_t n, uint8_t* out_xy, int* out_is_inf) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (C.pend.active) return fail(NMSM_ERR_ARG, "slot busy: collect the previous MSM first");
  if (n)
    if (int r = stage_host_inputs(C, pts, scalars, n)) return r;
  return run_msm((const uint32_t*)C.in_pts.p, (const uint32_t*)C.in_scalars.p, n, nullptr, out_xy, out_is_inf);
}

static int run_fold(const uint32_t* d_accs, int count, uint8_t* out_xy, int* out_is_inf) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  const int RES_WORDS = G::IN_WORDS + 4;
  CK(C.result.ensure(RES_WORDS * 4));
  uint32_t* d_res = (uint32_t*)C.result.p;
  k_fold<Cv><<<1, 32, 0, C.stream>>>(d_accs, count, d_res, d_res + G::IN_WORDS);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(C.h_result, d_res, RES_WORDS * 4, cudaMemcpyDeviceToHost, C.stream));
  CK(cudaStreamSynchronize(C.stream));
  memcpy(out_xy, C.h_result, G::IN_WORDS * 4);
  *out_is_inf = (int)C.h_result[G::IN_WORDS];
  return NMSM_OK;
}

// nmsm_accs_normalize: raw accumulators (host or device) -> canonical affine + infinity flags on the host
static int run_normalize(const void* accs, int on_device, uint64_t n, uint8_t* out_xy, uint8_t* out_is_inf) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  CK(C.mul_out.ensure(n * (G::IN_WORDS + 1) * 4 + 16));
  uint32_t* d_xy = (uint32_t*)C.mul_out.p;
  uint32_t* d_inf = d_xy + n * G::IN_WORDS;
  cudaStream_t st = C.stream;
  const uint32_t* d_accs = (const uint32_t*)accs;
  if (!on_device) {
    CK(C.in_pts.ensure(n * G::ACC_WORDS * 4));
    CK(cudaMemcpyAsync(C.in_pts.p, accs, n * G::ACC_WORDS * 4, cudaMemcpyHostToDevice, st));
    d_accs = (const uint32_t*)C.in_pts.p;
  }
  k_normalize_batch<Cv><<<cdiv(n, 128), 128, 0, st>>>(d_accs, (uint32_t)n, d_xy, d_inf);
  CK(cudaGetLastError());
  std::vector<uint32_t> inf(n);
  CK(cudaMemcpyAsync(out_xy, d_xy, n * G::IN_WORDS * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(inf.data(), d_inf, n * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (uint64_t i = 0; i < n; i++) out_is_inf[i] = (uint8_t)inf[i];
  return NMSM_OK;
}

static int run_mul_batch(const uint8_t* pts, const uint8_t* scalars, uint64_t n, int allow_zero, uint8_t* out_xy,
                         uint8_t* out_is_inf) {
  Slot& C = g_ctx.slot[g_ctx.cur];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  CK(C.in_pts.ensure(n * G::IN_WORDS * 4));
  CK(C.in_scalars.ensure(n * SCALAR_WORDS * 4));
  CK(C.mul_out.ensure(n * (G::IN_WORDS + 1) * 4 + 16));
  CK(C.result.ensure(64));
  unsigned int* d_err = (unsigned int*)C.result.p;
  uint32_t* d_xy = (uint32_t*)C.mul_out.p;
  uint32_t* d_inf = d_xy + n * G::IN_WORDS;
  cudaStream_t st = C.stream;
  CK(cudaMemcpyAsync(C.in_pts.p, pts, n * G::IN_WORDS * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(C.in_scalars.p, scalars, n * SCALAR_WORDS * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_err, 0xff, 8, st));
  EV(0);
  // one item per quad of lanes while that leaves the multiply pipe under-subscribed (<= 1.5 warps per sub-partition);
  // one item per thread wins once the pipe is full
  uint64_t quad_max = (uint64_t)g_ctx.sm_count * 4 * 12;
  if (const char* e = getenv("NMSM_MUL_QUAD_MAX")) quad_max = strtoull(e, nullptr, 10);  // tuning experiments
  if (n <= quad_max)
    k_mul_batch<Cv, true><<<cdiv(n * 4, 128), 128, 0, st>>>((const uint32_t*)C.in_pts.p, (const uint32_t*)C.in_scalars.p,
                                                            (uint32_t)n, allow_zero, d_xy, d_inf, d_err);
  else
    k_mul_batch<Cv, false><<<cdiv(n, 128), 128, 0, st>>>((const uint32_t*)C.in_pts.p, (const uint32_t*)C.in_scalars.p,
                                                          (uint32_t)n, allow_zero, d_xy, d_inf, d_err);
  EV(1);
  CK(cudaGetLastError());
  std::vector<uint32_t> inf(n);
  unsigned int err[2];
  CK(cudaMemcpyAsync(err, d_err, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(out_xy, d_xy, n * G::IN_WORDS * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(inf.data(), d_inf, n * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  note_kernel_time(C);
  if (err[0] != 0xffffffffu) return fail(NMSM_ERR_POINT, "invalid point at index " + std::to_string(err[0]), err[0]);
  if (err[1] != 0xffffffffu)
    return fail(NMSM_ERR_SCALAR, "invalid scalar: out of range (index " + std::to_string(err[1]) + ")", err[1]);
  for (uint64_t i = 0; i < n; i++) out_is_inf[i] = (uint8_t)inf[i];
  return NMSM_OK;
}
};


#define NMSM_DEFINE_ENGINE(FN, CURVE)                                                          \
  const EngineVTable* FN() {                                                                   \
    static const EngineVTable vt = {CURVE::G::IN_WORDS * 4,         CURVE::G::ACC_WORDS * 4,   \
                                    &Engine<CURVE>::run_msm_host,   &Engine<CURVE>::run_msm_dev,   \
                                    &Engine<CURVE>::run_fold,       &Engine<CURVE>::run_mul_batch,  \
                                    &Engine<CURVE>::prepare_points, &Engine<CURVE>::run_msm_prepared, \
                                    &Engine<CURVE>::precompute_table,                              \
                                    &Engine<CURVE>::build_point_table, &Engine<CURVE>::table_mul_batch, \
                                    &Engine<CURVE>::submit_any,     &Engine<CURVE>::collect_msm,    \
                                    &Engine<CURVE>::submit_prepared, &Engine<CURVE>::run_torsion,  \
                                    &Engine<CURVE>::run_on_curve,   &Engine<CURVE>::run_normalize};  \
    return &vt;                                                                                \
  }

}  // namespace nmsm
