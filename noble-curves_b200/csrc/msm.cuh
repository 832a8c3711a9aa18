// CUDA kernels (sm_90a) of the bucket-method multi-scalar multiplication and the batched scalar
// multiplication.  Thread bodies live in msm_body.cuh; this file is the launch geometry.
//
// Replaces /root/reference/src/abstract/curve.ts:863-905 `pippenger(c, points, scalars)`:
// same result point (compared as canonical affine), different schedule.  The reference walks
// unsigned c-bit windows MSB->LSB on one thread with complete projective additions; here
//
//   k_prepare      canonical affine -> Montgomery "prepared" affine, range validation     (N threads)
//   k_digits<0>    signed c-bit digit recoding + per-(window,bucket) histogram            (N threads)
//   k_scan_*       exclusive scan of the W*B histogram -> bucket offsets                  (2 passes)
//   k_digits<1>    counting-sort scatter of (point index | sign) into bucket order        (N threads)
//   k_accumulate   every thread folds exactly L consecutive sorted entries with mixed
//                  additions, emitting complete buckets or head/tail partials at bucket
//                  boundaries — constant work per thread whatever the bucket sizes are     (T/L threads)
//   k_stitch_tiles two levels of 32-way tile sums over the per-segment partials, only for buckets
//                  that span > 32 / > 1024 segments (degenerate inputs)                    (T/L/32 warps)
//   k_reduce1      per-chunk running sums (2 additions per bucket), stitching the partials
//                  of buckets that straddle accumulate segments on the fly                 (W*B/K threads)
//   k_reduce2      upper levels: suffix scan + reduction of chunk sums inside blocks of 32 quads
//                  (registers -> quad/warp shuffles -> shared memory), re-applied to its own
//                  block results until one block per window is left                        (W x splits blocks)
//   k_horner_step  Horner over the windows of one group (c doublings each), one warp whose lanes
//                  share each formula's independent multiplications; k_combine: inversion to affine (1 warp)
// The windows form groups that are accumulated top-first as separate launches; the reduction and Horner
// chains of finished groups run on high-priority side streams underneath the accumulation of the rest.
//
// No atomics touch curve points, so degenerate inputs (all scalars equal, all points equal —
// test/point.test.ts:842-853, benchmark/msm_timings.ts:45-63) stay correct; they only lengthen the
// stitch in k_reduce1 (bounded by the two tile levels).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "msm_body.cuh"
#include "validate.cuh"

namespace nmsm {

template <class Cv>
__global__ void k_prepare(const uint32_t* __restrict__ pts, uint32_t n, uint32_t* __restrict__ aff,
                          unsigned int* err) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) prepare_body<Cv>(i, n, pts, aff, err);
}

template <class Cv, bool SCATTER>
__global__ void k_digits(const uint32_t* __restrict__ scalars, uint32_t n, MsmPlan plan,
                         unsigned int* __restrict__ counts_or_cursor, uint32_t* __restrict__ sorted,
                         unsigned int* err) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) digits_body<Cv, SCATTER>(i, n, scalars, plan, counts_or_cursor, sorted, err);
}

// Exclusive scan of the G bucket counters in two coalesced passes over SCAN_TILE-element tiles:
//   k_scan_tiles   per-tile totals
//   k_scan_apply   tile prefix (every block sums the totals before it) + in-tile scan -> offsets, cursor
static constexpr int SCAN_THREADS = 256;
static constexpr int SCAN_PER_THREAD = 8;
static constexpr int SCAN_TILE = SCAN_THREADS * SCAN_PER_THREAD;

__device__ __forceinline__ uint32_t block_sum_256(uint32_t v, uint32_t* sh) {
  for (int d = 16; d >= 1; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t t = 0;
  for (int q = 0; q < SCAN_THREADS / 32; q++) t += sh[q];
  __syncthreads();
  return t;
}

static __global__ void __launch_bounds__(SCAN_THREADS)
k_scan_tiles(const unsigned int* __restrict__ counts, uint32_t G, uint32_t* __restrict__ tile_sums) {
  __shared__ uint32_t sh[SCAN_THREADS / 32];
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER_THREAD;
  uint32_t v = 0;
#pragma unroll
  for (int k = 0; k < SCAN_PER_THREAD; k++)
    if (base + k < G) v += counts[base + k];
  uint32_t t = block_sum_256(v, sh);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = t;
}

static __global__ void __launch_bounds__(SCAN_THREADS)
k_scan_apply(const unsigned int* __restrict__ counts, uint32_t G, const uint32_t* __restrict__ tile_sums,
             uint32_t* __restrict__ offsets, unsigned int* __restrict__ cursor) {
  __shared__ uint32_t sh[SCAN_THREADS / 32];
  __shared__ uint32_t warp_tot[SCAN_THREADS / 32];
  // prefix of the tiles before this one
  uint32_t pre = 0;
  for (uint32_t k = threadIdx.x; k < blockIdx.x; k += SCAN_THREADS) pre += tile_sums[k];
  const uint32_t tile_prefix = block_sum_256(pre, sh);
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER_THREAD;
  uint32_t c[SCAN_PER_THREAD];
  uint32_t mine = 0;
#pragma unroll
  for (int k = 0; k < SCAN_PER_THREAD; k++) {
    c[k] = (base + k < G) ? counts[base + k] : 0;
    mine += c[k];
  }
  // exclusive scan of `mine` across the block: warp inclusive scan + warp totals
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = mine;
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= (uint32_t)d) inc += o;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  uint32_t wpre = 0;
  for (uint32_t q = 0; q < warp; q++) wpre += warp_tot[q];
  uint32_t run = tile_prefix + wpre + inc - mine;
#pragma unroll
  for (int k = 0; k < SCAN_PER_THREAD; k++) {
    if (base + k < G) {
      offsets[base + k] = run;
      cursor[base + k] = run;
    }
    run += c[k];
  }
  // the thread that owns element G-1 also publishes the grand total
  if (base < G && base + SCAN_PER_THREAD >= G) offsets[G] = run;
}

// One field inversion per warp (Montgomery's trick across the lanes): every lane passes a non-zero z and gets
// 1/z.  Inclusive prefix and suffix products by shuffles (5 + 5 multiplications per lane), one inversion of the
// warp total computed redundantly in all lanes (same operand, no divergence), two more multiplications.
// All 32 lanes must call it.
template <class F>
__device__ __forceinline__ F shfl_field(const F& a, int src_lane) {
  F r;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&a);
  uint32_t* d = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int k = 0; k < (int)(sizeof(F) / 4); k++) d[k] = __shfl_sync(0xffffffffu, s[k], src_lane);
  return r;
}
template <class F>
__device__ __noinline__ F warp_batch_inverse(const F& z) {
  const int lane = threadIdx.x & 31;
  F pre = z, suf = z;
  for (int d = 1; d < 32; d <<= 1) {
    F a = shfl_field(pre, lane >= d ? lane - d : lane);
    F b = shfl_field(suf, lane + d < 32 ? lane + d : lane);
    if (lane >= d) pre = pre * a;
    if (lane + d < 32) suf = suf * b;
  }
  F r = inv(shfl_field(pre, 31));
  F left = shfl_field(pre, lane > 0 ? lane - 1 : 0);
  F right = shfl_field(suf, lane < 31 ? lane + 1 : 31);
  if (lane > 0) r = r * left;
  if (lane < 31) r = r * right;
  return r;
}

// NMSM_PAIRED=1 builds k_accumulate with paired accumulation (msm_body.cuh accumulate_pairs_pass1/2: same-bucket
// neighbours added in affine with one warp-shared inversion, 16 instead of 20 multiplications per two entries).  It is
// bit-exact (hostemu + all GPU parity tests) and executes 20 % fewer multiplications, but it was slower than the plain
// loop: one inversion plus 12 scan multiplications per warp amortise over only ~28 pairs per lane, pass 1 is a chain of
// dependent gathers with one multiplication each, and the extra live state spills.  Kept as a build option; the default
// is the plain mixed-addition loop.
#ifndef NMSM_PAIRED
#define NMSM_PAIRED 0
#endif
template <class Cv>
__global__ void __launch_bounds__(128, acc_blocks_per_sm<typename Cv::G>())
k_accumulate(const uint32_t* __restrict__ aff, const uint32_t* __restrict__ sorted,
             const uint32_t* __restrict__ offsets, MsmPlan plan, uint32_t w0, uint32_t* __restrict__ buckets,
             uint32_t* __restrict__ heads, uint32_t* __restrict__ tails) {
  // grid = (windows of the group) * TPW threads; TPW is a multiple of the block size, so a block never straddles windows
  const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t w = w0 + gid / plan.TPW, t = gid % plan.TPW;
#if NMSM_PAIRED
  if constexpr (!Cv::G::IS_EDWARDS) {
    // paired accumulation (msm_body.cuh): affine sums of same-bucket neighbours, ONE field inversion per warp
    using F = typename Cv::G::Field;
    F suf[MAX_PAIRS];
    int npairs;
    const F run = accumulate_pairs_pass1<Cv>(w, t, aff, sorted, offsets, plan, suf, npairs);
    const F inv_all = warp_batch_inverse(run);  // every lane of the warp, also the ones without a pair (run = 1)
    accumulate_pairs_pass2<Cv>(w, t, aff, sorted, offsets, plan, suf, npairs, inv_all, buckets, heads, tails);
    return;
  }
#endif
  accumulate_body<Cv>(w, t, aff, sorted, offsets, plan, buckets, heads, tails);
}

// ------------------------------------------------------------------------------------------------
// Bucket reduction.  These phases have little parallel work, and a field multiplication occupies
// the multiply pipe per WARP instruction, so every logical thread runs on a quad of 4 lanes
// (ec.cuh Par4: 4 multiplication levels per addition instead of 14 dependent multiplications).
//   sum_b (b+1) B_b  =  sum_k T_k + K * sum_k k * S_k        k over the M = B/K chunks   (k_reduce1)
//   per block of Mb chunks:  P_s = sum T_k + K * sum (k - s*Mb) S_k ,  Q_s = sum S_k        (k_reduce2)
//   window sum = sum_s P_s + K * Mb * sum_s s * Q_s                                          (k_reduce2, next level)
// The last line has the shape of the first (T := P, S := Q, K := K * Mb): k_reduce2 is applied again to its own outputs
// (with fewer chunks per quad) until ONE block per window is left, whose P_0 is the window sum.  Ordinary plans: two
// passes (4096 chunks -> 32 block results -> 1); fixed-base tables (one window of up to 2^21 buckets): three or four.
// ------------------------------------------------------------------------------------------------
template <class G>
__device__ __forceinline__ typename G::Acc shfl_down_acc(const typename G::Acc& a, int delta) {
  typename G::Acc r;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&a);
  uint32_t* d = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int k = 0; k < G::ACC_WORDS; k++) d[k] = __shfl_down_sync(0xffffffffu, s[k], delta);
  return r;
}

// One warp per tile of 32 consecutive partials (level 1: heads, span 32 segments; level 2: tile1,
// span 1024 segments).  Tiles that are not wholly inside one bucket exit after the bucket lookup,
// which is every tile for ordinary inputs; see msm_body.cuh "stitching".
template <class Cv>
__global__ void __launch_bounds__(128)
k_stitch_tiles(const uint32_t* __restrict__ offsets, MsmPlan plan, uint32_t span, uint32_t j0, uint32_t j1,
               const uint32_t* __restrict__ in, uint32_t* __restrict__ out) {
  using G = typename Cv::G;
  const uint32_t j = j0 + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;  // tiles [j0, j1)
  if (j >= j1) return;
  if (!tile_is_uniform(offsets, plan, (uint64_t)j * span, span)) return;  // warp-uniform
  typename G::Acc acc = load_acc<G>(in + ((size_t)j * STITCH_FAN + lane) * G::ACC_WORDS);
  for (int d = 16; d >= 1; d >>= 1) {
    typename G::Acc o = shfl_down_acc<G>(acc, d);
    nl_add<G>(acc, o);
  }
  if (lane == 0) save_acc<G>(out + (size_t)j * G::ACC_WORDS, acc);
}

// Two forms of the first reduction level.  Serial (one thread per chunk, out-of-line formulas): the throughput form —
// with >= 2 warps per SM sub-partition the multiply pipe is shared anyway.  Quad (one chunk per 4 lanes, ec.cuh Par4):
// the latency form for a group whose chain is on the critical path (the last window group: nothing left to overlap it
// with) — 4 multiplication levels per addition instead of 14 dependent multiplications.
static constexpr int REDUCE1_THREADS = 128;
#if defined(__CUDACC__)
template <class G>
struct QuadOps {
  __device__ static void add(typename G::Acc& p, const typename G::Acc& q) { G::template par_add<false>(p, q); }
  __device__ static void dbl(typename G::Acc& p) { G::template par_dbl<false>(p); }
  __device__ static void madd(typename G::Acc& p, const typename G::Affine& q) { G::template par_add<false>(p, G::from_affine(q)); }
};
#endif
template <class Cv, bool QUAD>
__global__ void __launch_bounds__(REDUCE1_THREADS)
k_reduce1(const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ buckets,
          const uint32_t* __restrict__ heads, const uint32_t* __restrict__ tails,
          const uint32_t* __restrict__ tile1, const uint32_t* __restrict__ tile2, MsmPlan plan, uint32_t id0,
          uint32_t id1, uint32_t* __restrict__ sums, uint32_t* __restrict__ wsums) {
  using G = typename Cv::G;
  const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t id = id0 + (QUAD ? gt >> 2 : gt);  // chunks [id0, id1) = the windows of one group
  if (id >= id1) return;  // whole quads leave together
  if (QUAD) reduce1_body<Cv, QuadOps<G>>(id, offsets, buckets, heads, tails, tile1, tile2, plan, sums, wsums);
  else reduce1_body<Cv, SerialOps<G>>(id, offsets, buckets, heads, tails, tile1, tile2, plan, sums, wsums);
}

// ---- multi-GPU bucket exchange (engine.cuh submit_msm, dist mode) -------------------------------------------
template <class Cv>
__global__ void __launch_bounds__(128)
k_bucket_finalize(const uint32_t* __restrict__ offsets, uint32_t* __restrict__ buckets, const uint32_t* __restrict__ heads,
                  const uint32_t* __restrict__ tails, const uint32_t* __restrict__ tile1, const uint32_t* __restrict__ tile2,
                  MsmPlan plan, uint32_t g0, uint32_t g1) {
  const uint32_t g = g0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (g < g1) bucket_finalize_body<Cv>(g, offsets, buckets, heads, tails, tile1, tile2, plan);
}
// Both run one logical thread per QUAD of lanes (ec.cuh Par4): an owner's fold and first reduction level sit on the
// critical path of a sharded MSM (one window = few thousand chains, the GPU is otherwise idle), so the latency form pays.
template <class Cv>
__global__ void __launch_bounds__(128)
k_bucket_fold(uint32_t* __restrict__ own, const uint32_t* __restrict__ recv, int npeers, size_t stride_words, uint32_t B) {
  const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  if (b < B) bucket_fold_body<Cv, QuadOps<typename Cv::G>>(b, own, recv, npeers, stride_words);
}
// Fused exchange + fold: the owner of a window reads every peer's partial bucket b straight from the peer's HBM over
// NVLink (peer pointers from CUDA IPC, `window_words` = offset of the window inside a bucket array) and adds it.
template <class Cv>
__global__ void __launch_bounds__(128)
k_bucket_fold_peers(uint32_t* __restrict__ own, PeerPtrs peers, size_t window_words, int world, int rank, uint32_t B) {
  const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  if (b >= B) return;
  const uint32_t* base[MAX_PEERS];
#pragma unroll
  for (int r = 0; r < MAX_PEERS; r++) base[r] = r < world && r != rank ? peers.p[r] + window_words : nullptr;
  bucket_fold_peers_body<Cv, QuadOps<typename Cv::G>>(b, own, base, world, rank);
}
template <class Cv>
__global__ void __launch_bounds__(REDUCE1_THREADS)
k_reduce1_dense(const uint32_t* __restrict__ buckets, MsmPlan plan, uint32_t id0, uint32_t id1, uint32_t* __restrict__ sums,
                uint32_t* __restrict__ wsums) {
  const uint32_t id = id0 + ((blockIdx.x * blockDim.x + threadIdx.x) >> 2);
  if (id < id1) reduce1_dense_body<Cv, QuadOps<typename Cv::G>>(id, buckets, plan, sums, wsums);
}
// tail of a rank's gather block: err_pt | err_sc (local indices, 0xffffffff = none) | shard offset (lo, hi)
static __global__ void k_pack_shard_tail(uint32_t* __restrict__ tail, const unsigned int* __restrict__ err, uint64_t offset) {
  if (threadIdx.x == 0) {
    tail[0] = err[0];
    tail[1] = err[1];
    tail[2] = (uint32_t)offset;
    tail[3] = (uint32_t)(offset >> 32);
  }
}
template <class Cv>
__global__ void __launch_bounds__(32)
k_set_identity(uint32_t* __restrict__ accs, int count) {
  using G = typename Cv::G;
  if ((int)threadIdx.x < count) save_acc<G>(accs + (size_t)threadIdx.x * G::ACC_WORDS, G::identity());
}

// shuffle by `dq` logical lanes (quads); every lane of the warp must be converged here
template <class G>
__device__ __forceinline__ typename G::Acc shfl_down_quads(const typename G::Acc& a, int dq) {
  typename G::Acc r;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&a);
  uint32_t* d = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int k = 0; k < G::ACC_WORDS; k++) d[k] = __shfl_down_sync(0xffffffffu, s[k], 4 * dq);
  return r;
}
template <class G>
__device__ __forceinline__ void smem_put(uint32_t* smem, uint32_t slot, const typename G::Acc& a) {
  const uint32_t* src = reinterpret_cast<const uint32_t*>(&a);
  for (int k = 0; k < G::ACC_WORDS; k++) smem[slot * G::ACC_WORDS + k] = src[k];
}
template <class G>
__device__ __forceinline__ typename G::Acc smem_get(const uint32_t* smem, uint32_t slot) {
  typename G::Acc a;
  uint32_t* dst = reinterpret_cast<uint32_t*>(&a);
  for (int k = 0; k < G::ACC_WORDS; k++) dst[k] = smem[slot * G::ACC_WORDS + k];
  return a;
}

static constexpr int REDUCE2_THREADS = 128;                   // 32 logical threads (quads), 4 warps
static constexpr int REDUCE2_LOGICAL = REDUCE2_THREADS / 4;
static constexpr int REDUCE2_MAX_SPLITS = 32;                 // block results per window the LAST pass (one block, R = 1) takes
static constexpr int REDUCE2_R = 4;                           // chunks per logical thread
static constexpr int REDUCE2_CHUNKS_PER_BLOCK = REDUCE2_LOGICAL * REDUCE2_R;

// grid (splits, W).  Logical thread lt owns R consecutive chunks; see the formulas above.
template <class Cv>
__global__ void __launch_bounds__(REDUCE2_THREADS)
k_reduce2(const uint32_t* __restrict__ sums, const uint32_t* __restrict__ wsums, MsmPlan plan, int R, uint32_t w0,
          uint32_t* __restrict__ blkP, uint32_t* __restrict__ blkQ, uint32_t* __restrict__ window_out) {
  using G = typename Cv::G;
  using Acc = typename G::Acc;
  extern __shared__ uint32_t smem[];  // one accumulator per warp
  const uint32_t s = blockIdx.x, w = w0 + blockIdx.y, splits = gridDim.x;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ql = lane >> 2;
  const uint32_t lt = threadIdx.x >> 2;
  constexpr uint32_t NW = REDUCE2_THREADS / 32;
  const uint32_t M = plan.chunks;
  const uint32_t Mb = REDUCE2_LOGICAL * R;
  const uint32_t base = s * Mb + lt * R;
  Acc S = G::identity(), WL = G::identity(), WT = G::identity();
  for (uint32_t k = base + R; k-- > base;) {
    if (k < M) {
      const size_t id = (size_t)w * M + k;
      G::template par_add<false>(WT, load_acc<G>(wsums + id * G::ACC_WORDS));
      G::template par_add<false>(S, load_acc<G>(sums + id * G::ACC_WORDS));
    }
    if (k > base) G::template par_add<false>(WL, S);  // after the loop: sum (k - base) * S_k
  }
  // inclusive suffix scan of S over the logical threads of the block
  Acc SS = S;
  for (int d = 1; d < 8; d <<= 1) {
    __syncwarp();
    Acc o = shfl_down_quads<G>(SS, d);
    if (ql + d < 8) G::template par_add<false>(SS, o);
  }
  __syncwarp();
  if (lane == 0) smem_put<G>(smem, warp, SS);  // warp totals
  __syncthreads();
  for (uint32_t q = warp + 1; q < NW; q++) G::template par_add<false>(SS, smem_get<G>(smem, q));
  __syncthreads();
  // per-thread contribution  WT + K * (WL + R * [lt >= 1] SS)
  Acc V = G::identity();
  if (lt >= 1) {
    V = SS;
    for (int r = 1; r < R; r <<= 1) G::template par_dbl<false>(V);
  }
  G::template par_add<false>(V, WL);
  for (int j = 1; j < plan.K; j <<= 1) G::template par_dbl<false>(V);
  G::template par_add<false>(V, WT);
  // block reduction of V
  for (int d = 4; d >= 1; d >>= 1) {
    __syncwarp();
    Acc o = shfl_down_quads<G>(V, d);
    G::template par_add<false>(V, o);
  }
  if (lane == 0) smem_put<G>(smem, warp, V);
  __syncthreads();
  if (warp == 0 && ql == 0) {
    for (uint32_t q = 1; q < NW; q++) G::template par_add<false>(V, smem_get<G>(smem, q));
    if (lane == 0) {
      if (window_out) {  // last level (one block per window): P_0 is the window sum, the s * Q_s term vanishes
        save_acc<G>(window_out + (size_t)w * G::ACC_WORDS, V);
      } else {
        save_acc<G>(blkP + ((size_t)w * splits + s) * G::ACC_WORDS, V);
        save_acc<G>(blkQ + ((size_t)w * splits + s) * G::ACC_WORDS, SS);  // SS of logical thread 0 = block total
      }
    }
  }
}

// One Horner step over the window sums of a window group (msm_body.cuh horner_step_body; curve.ts:901-902) by ONE warp
// whose lanes hold replicated state and split the independent multiplications of every point formula between them
// (ec.cuh Par4).  Runs on its own high-priority stream: the doubling chains of the upper windows overlap the
// accumulation of the lower ones (engine.cuh submit_msm).
template <class Cv>
__global__ void __launch_bounds__(32)
k_horner_step(const uint32_t* __restrict__ window_out, MsmPlan plan, int w_lo, int w_hi, int first, int shift,
              uint32_t* __restrict__ hacc) {
  using G = typename Cv::G;
  typename G::Acc acc = first ? G::identity() : load_acc<G>(hacc);
  for (int w = w_hi - 1; w >= w_lo; w--) {
    if (!(first && w == w_hi - 1))
      for (int j = 0; j < plan.c; j++) G::template par_dbl<true>(acc);
    G::template par_add<true>(acc, load_acc<G>(window_out + (size_t)w * G::ACC_WORDS));
  }
  if (shift)
    for (int j = 0; j < plan.c * w_lo; j++) G::template par_dbl<true>(acc);
  if (threadIdx.x == 0) save_acc<G>(hacc, acc);
}

// Sum of the `count` group accumulators; AFFINE_OUT: canonical affine + infinity flag, else the raw accumulator
// (multi-GPU partial, folded later by k_fold).
// The accumulators sit in blocks of `per_block` consecutive ones, `block_stride` words apart (the all-gathered layout of
// a sharded MSM: every rank's weighted window sums followed by its validation words).
template <class Cv, bool AFFINE_OUT>
__global__ void __launch_bounds__(32)
k_combine(const uint32_t* __restrict__ accs, int count, int per_block, int block_stride, uint32_t* __restrict__ out,
          uint32_t* __restrict__ out_inf) {
  using G = typename Cv::G;
  // the 8 quads of the warp each sum every 8th accumulator, then a 3-level tree over the quads: 1 + 3 lane-parallel
  // additions for the 8 weighted window sums of an 8-GPU MSM instead of 8 dependent ones
  const uint32_t lane = threadIdx.x, ql = lane >> 2;
  typename G::Acc acc = G::identity();
  for (int i = (int)ql; i < count; i += 8)
    G::template par_add<false>(acc, load_acc<G>(accs + (size_t)(i / per_block) * block_stride + (size_t)(i % per_block) * G::ACC_WORDS));
  for (int d = 4; d >= 1; d >>= 1) {
    __syncwarp();
    typename G::Acc o = shfl_down_quads<G>(acc, d);
    G::template par_add<false>(acc, o);
  }
  if (ql != 0) return;  // quad 0 holds the total
  if (AFFINE_OUT) {
    uint32_t xy[G::IN_WORDS];
    uint32_t inf;
    nl_to_affine<G>(acc, xy, &inf);
    if (lane == 0) {
      for (int k = 0; k < G::IN_WORDS; k++) out[k] = xy[k];
      *out_inf = inf;
    }
  } else if (lane == 0) {
    save_acc<G>(out, acc);
  }
}

template <class Cv>
__global__ void __launch_bounds__(32)
k_fold(const uint32_t* __restrict__ accs, int count, uint32_t* __restrict__ out, uint32_t* __restrict__ out_inf) {
  using G = typename Cv::G;
  typename G::Acc acc = G::identity();
  for (int i = 0; i < count; i++) G::template par_add<true>(acc, load_acc<G>(accs + (size_t)i * G::ACC_WORDS));
  uint32_t xy[G::IN_WORDS];
  uint32_t inf;
  nl_to_affine<G>(acc, xy, &inf);
  if (threadIdx.x == 0) {
    for (int k = 0; k < G::IN_WORDS; k++) out[k] = xy[k];
    *out_inf = inf;
  }
}

// Fixed-base tables: level j+1 = 2^c * level j for every point of the set (nmsm_points_precompute).
template <class Cv>
__global__ void __launch_bounds__(128)
k_table_level(const uint32_t* __restrict__ prev, uint32_t* __restrict__ next, uint32_t count, int c) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) table_level_body<Cv>(i, prev, next, c);
}

// Fixed-point multiplication tables (nmsm_point_table_*): level 0 = d * P, then k_table_level per level.
template <class Cv>
__global__ void __launch_bounds__(128)
k_table_base(const uint32_t* __restrict__ p_aff, uint32_t* __restrict__ level0) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < PT_HALF) table_base_body<Cv>(i, p_aff, level0);
}

// out[i] = scalars[i] * P: `levels` gathered mixed additions per thread, then canonical affine.
template <class Cv>
__global__ void __launch_bounds__(128)
k_table_mul(const uint32_t* __restrict__ tbl, const uint32_t* __restrict__ scalars, uint32_t n, int allow_zero,
            uint32_t* __restrict__ out_xy, uint32_t* __restrict__ out_inf, unsigned int* err) {
  using G = typename Cv::G;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  typename G::Acc acc = G::identity();
  const bool ok = i < n && table_mul_body<Cv>(i, tbl, scalars, allow_zero, acc, err);
  const typename G::Field iz = warp_batch_inverse(G::inv_target(acc));  // whole warp, also the idle lanes
  if (!ok) return;
  uint32_t xy[G::IN_WORDS];
  uint32_t inf;
  G::to_affine_canonical_with_inv(acc, iz, xy, &inf);
  store_words<G::IN_WORDS>(out_xy + (size_t)i * G::IN_WORDS, xy);
  out_inf[i] = inf;
}

// out[i] = scalars[i] * pts[i].  The to-affine step is the reference's normalizeZ (curve.ts:311-326: one inversion for
// a whole batch by Montgomery's trick, FpInvertBatch modular.ts:734-760): here ONE inversion per warp shared through
// prefix / suffix products over the lanes (warp_batch_inverse), instead of a ~770-step binary xgcd in every thread.
// QUAD: one item per quad of lanes (ec.cuh Par4) — a batch of a few thousand multiplications is a pure latency chain of
// ~130 doublings + ~70 additions per item, and the lane-parallel formulas cut each link from 9 / 14 dependent field
// multiplications to 3 / 4 levels.  The engine picks it while the batch leaves multiply-pipe slots idle (engine.cuh).
template <class Cv, bool QUAD>
__global__ void __launch_bounds__(128)
k_mul_batch(const uint32_t* __restrict__ pts, const uint32_t* __restrict__ scalars, uint32_t n,
            int allow_zero, uint32_t* __restrict__ out_xy, uint32_t* __restrict__ out_inf,
            unsigned int* err) {
  using G = typename Cv::G;
  const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t i = QUAD ? gt >> 2 : gt;
  typename G::Acc acc = G::identity();
  bool ok;
  if (QUAD) ok = i < n && mul_acc_body<Cv, QuadOps<G>>(i, pts, scalars, allow_zero, acc, err);  // whole quads leave together
  else ok = i < n && mul_acc_body<Cv>(i, pts, scalars, allow_zero, acc, err);
  const typename G::Field iz = warp_batch_inverse(G::inv_target(acc));  // whole warp, also the idle lanes
  if (!ok || (QUAD && (gt & 3u))) return;
  uint32_t xy[G::IN_WORDS];
  uint32_t inf;
  G::to_affine_canonical_with_inv(acc, iz, xy, &inf);
  store_words<G::IN_WORDS>(out_xy + (size_t)i * G::IN_WORDS, xy);
  out_inf[i] = inf;
}

// Batch normalisation of raw accumulators to canonical affine: the device form of normalizeZ (curve.ts:311-326) — one
// field inversion per warp shared through prefix / suffix products (FpInvertBatch, modular.ts:734-760), identities pass
// through as (0,0) / (0,1) with the infinity flag like toAffine(ZERO).
template <class Cv>
__global__ void __launch_bounds__(128)
k_normalize_batch(const uint32_t* __restrict__ accs, uint32_t n, uint32_t* __restrict__ out_xy, uint32_t* __restrict__ out_inf) {
  using G = typename Cv::G;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  typename G::Acc acc = G::identity();
  if (i < n) acc = load_acc<G>(accs + (size_t)i * G::ACC_WORDS);
  const typename G::Field iz = warp_batch_inverse(G::inv_target(acc));  // whole warp, also the idle lanes
  if (i >= n) return;
  uint32_t xy[G::IN_WORDS];
  uint32_t inf;
  G::to_affine_canonical_with_inv(acc, iz, xy, &inf);
  store_words<G::IN_WORDS>(out_xy + (size_t)i * G::IN_WORDS, xy);
  out_inf[i] = inf;
}

// n * P == O per point (nmsm_points_torsion_free)
template <class Cv>
__global__ void __launch_bounds__(128)
k_torsion(const uint32_t* __restrict__ pts, uint32_t n, uint8_t* __restrict__ out_ok, unsigned int* err) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) torsion_body<Cv>(i, pts, out_ok, err);
}

// Profiling only: how many of the sorted entries START an accumulator (a copy, no field multiplications) instead of
// being added to one — one per non-empty bucket plus one per accumulate segment that begins inside a bucket — and how
// many same-bucket PAIRS the segments hold (added in affine first).  The roofline accounting counts the executed
// field multiplications of k_accumulate from them:  10 * (entries - starts) - 4 * pairs + 12 * threads.
static __global__ void k_count_starts(const uint32_t* __restrict__ offsets, MsmPlan plan, unsigned long long* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned int c = 0, pairs = 0;
  if (i < (uint32_t)plan.G && offsets[i + 1] > offsets[i]) c++;
  const uint64_t nseg = (uint64_t)plan.W * plan.TPW;
  if (i < nseg) {  // segment (w, t): does it begin strictly inside a bucket?  how many same-bucket pairs does it hold?
    const uint32_t w = i / plan.TPW, t = i % plan.TPW;
    const uint32_t base = offsets[w * (uint32_t)plan.B], T = offsets[(w + 1) * (uint32_t)plan.B];
    const uint64_t seg = (uint64_t)base + (uint64_t)t * (uint32_t)plan.L;
    if (seg < T) {
      uint32_t g = bucket_of_entry(offsets, plan, w, (uint32_t)seg);
      if (t > 0 && offsets[g] < seg) c++;
      // pairs (b0 + 2j, b0 + 2j + 1) of every bucket run inside [seg, end): the rule of accumulate_pairs_pass1/2
      const uint32_t end = (T - (uint32_t)seg > (uint32_t)plan.L) ? (uint32_t)seg + plan.L : T;
      for (uint32_t pos = (uint32_t)seg; pos < end;) {
        while (offsets[g + 1] <= pos) g++;
        const uint32_t b0 = offsets[g], b1 = offsets[g + 1];
        const uint32_t re = b1 < end ? b1 : end;
        const uint32_t first = pos + ((pos - b0) & 1u);  // first even offset >= pos
        if (re > first) pairs += (re - first) / 2;
        pos = re;
      }
    }
  }
  c = __reduce_add_sync(0xffffffffu, c);
  pairs = __reduce_add_sync(0xffffffffu, pairs);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
  if ((threadIdx.x & 31) == 0 && pairs) atomicAdd(out + 1, (unsigned long long)pairs);
}

// curve-equation check per point (nmsm_points_on_curve)
template <class Cv>
__global__ void __launch_bounds__(128)
k_on_curve(const uint32_t* __restrict__ pts, uint32_t n, uint8_t* __restrict__ out_ok) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out_ok[i] = (uint8_t)point_on_curve<Cv>(pts + (size_t)i * Cv::G::IN_WORDS);
}

}  // namespace nmsm
