// Per-thread bodies of the MSM / scalar-multiplication kernels.
//
// Each function is what ONE CUDA thread of the corresponding kernel in msm.cuh executes.  They are
// written against plain pointers and a thread index so that tests/hostemu can drive exactly the same
// code on the CPU (loops over the thread index, emulated PTX carry flag) — test infrastructure that
// lets the limb arithmetic and the bucket bookkeeping be verified without a GPU.  The product
// library only ever runs them inside the CUDA kernels.
//
// Pipeline (replaces /root/reference/src/abstract/curve.ts:863-905 `pippenger`):
//   prepare -> count digits -> scan -> scatter -> accumulate -> stitch -> reduce1 -> reduce2/3 -> final
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "ec.cuh"

#if defined(__CUDACC__)
#define NMSM_NL __host__ __device__ __noinline__
#else
#define NMSM_NL inline
#endif

namespace nmsm {

static constexpr int MAX_WINDOW_BITS = 16;
static constexpr int MAX_TABLE_BITS = 22;  // fixed-base tables: one bucket set of 2^(c-1) buckets
static constexpr int SCALAR_WORDS = 8;

struct MsmPlan {
  int c;       // window bits
  int W;       // bucket windows (1 when the point set carries precomputed 2^(c*j) multiples)
  int B;       // buckets per window = 2^(c-1)
  int G;       // W*B
  int L;       // sorted entries per accumulate thread
  int K;       // buckets per reduce chunk
  int chunks;  // B / K
  int D;       // signed digits per (half-)scalar; == W unless stride != 0
  uint32_t stride;  // 0: digit w goes to bucket window w.  != 0 (fixed-base tables): every digit goes to the
                    // single bucket window and selects the point  index + w * stride  = 2^(offset_w) * P_index
  int wb, r;        // digit w is  wb + (w < r)  bits wide and starts at bit  w * wb + min(w, r).  Ordinary plans:
                    // wb = c, r = 0.  Table plans spread the bits+1 scalar bits evenly over the D digits so that no
                    // digit is much narrower than the others (a narrow digit piles its terms onto few buckets)
  uint32_t TPW;     // accumulate segments (= threads) reserved per bucket window, a multiple of SEG_ALIGN.  Segment
                    // (w, t) owns the sorted entries [offsets[w*B] + t*L, + L) of window w, so no segment straddles
                    // two windows and the windows can be accumulated and reduced as independent launches
};
// Blocks of 128 threads per SM that k_accumulate is built for: its __launch_bounds__ (so 65536 / (128 * blocks)
// registers per thread) and the wave that plan_seg_len sizes the segments for.  By accumulator size:
//   128 B  XYZZ over a 256-bit field, ed25519 extended coordinates   4 blocks, <= 128 registers
//   192 B  XYZZ over the 381-bit BLS12-381 field                      3 blocks, <= 168 registers: the mixed addition
//          with inline products (ec.cuh madd<true>) fits without local memory; under 128 registers it spills
//   256 B  bn254 G2 (XYZZ over Fp2, 254 bits)                         4 blocks
//   384 B  BLS12-381 G2 (XYZZ over Fp2, 381 bits)                     2 blocks: the accumulator alone is 96 registers
template <class G>
NMSM_HD constexpr int acc_blocks_per_sm() {
  return sizeof(typename G::Acc) == 192 ? 3 : (sizeof(typename G::Acc) > 256 ? 2 : 4);
}
// Inline products in k_accumulate's mixed addition where that budget holds them without spills.  Under 128 registers
// (the 256-bit curves) the inline form spills more than the calls to the shared out-of-line body do.
template <class G>
NMSM_HD constexpr bool acc_inline_products() {
  return acc_blocks_per_sm<G>() == 3;
}
// Entries per accumulate thread: whole waves of the grid (acc_blocks_per_sm blocks of 128 threads per SM) with at most
// 64 entries per thread.  Longer segments mean fewer bucket partials for k_reduce1 to stitch, and sizing them to fill
// the last wave keeps k_accumulate's tail short.
NMSM_HD int plan_seg_len(double entries, int sm_count, int blocks_per_sm) {
  const double wave = (double)sm_count * blocks_per_sm * 128.0;  // threads of one full wave
  const double waves = ceil(entries / (64.0 * wave));
  int L = (int)ceil(entries / ((waves < 1.0 ? 1.0 : waves) * wave));
  return L < 4 ? 4 : (L > 64 ? 64 : L);
}
static constexpr uint32_t SEG_ALIGN = 1024;  // two stitch-tile levels of fan 32 never straddle a window
// entries a single window can receive at most: one per term and digit routed to it
NMSM_HD uint32_t plan_tpw(uint64_t max_window_entries, int L) {
  const uint64_t t = (max_window_entries + (uint32_t)L - 1) / (uint32_t)L;
  return (uint32_t)((t + SEG_ALIGN - 1) / SEG_ALIGN * SEG_ALIGN);
}
NMSM_HD int digit_width(const MsmPlan& p, int w) { return p.wb + (w < p.r ? 1 : 0); }
NMSM_HD int digit_offset(const MsmPlan& p, int w) { return w * p.wb + (w < p.r ? w : p.r); }

template <class Cv>
constexpr int glv_bits() {
  if constexpr (Cv::GLV) return Cv::Glv::BITS;
  else return Cv::Fn::BITS;
}
// sub-terms per input term: k*P = sum_j k_j * E_j(P) with short k_j; sub-term j of term i lives at index j*n + i
template <class Cv>
constexpr int split_of() { return Cv::GLV_KIND == 3 ? 4 : (Cv::GLV ? 2 : 1); }

// ---------------------------------------------------------------------------------------------
// plan selection: pick the window size c that minimises a TIME model of the pipeline.  The constants are for
// BLS12-381 G1, scaled by field size / formula cost for the others; only their ratios steer the choice of c:
//   accumulate   entries * 0.352 ns            (k_accumulate at ~88 % of the multiply-pipe bound)
//   reduce1      max( buckets * (1 + parts) adds at 0.93 ns each  [throughput],
//                     K * (1 + parts_top) dependent adds at ~30 us each  [one thread's chain] )
//                where parts = accumulate segments a bucket straddles; the TOP window matters most: if it
//                holds only a few scalar bits its buckets are huge and every reduce1 thread stitches
//                parts_top partials per bucket
//   reduce2/3    ~0.75 ms latency,  final  ~6.2 us per Horner doubling
// ---------------------------------------------------------------------------------------------
// n: term count the window size is chosen for (the GLOBAL count of a sharded MSM, so that every GPU uses the same
// windows and buckets); n_local (0 = n): terms this GPU accumulates, which sizes the accumulate segments.
template <class Cv>
inline MsmPlan make_plan(uint64_t n, int forced_c, int sm_count, uint64_t n_local = 0, int min_c = 2) {
  using G = typename Cv::G;
  using F = typename G::Field;
  // with GLV every scalar becomes two signed halves of at most 127 bits, each attached to its own point
  const int bits = glv_bits<Cv>();
  const double terms = (double)n * split_of<Cv>();
  const double limb_ratio = (double)(F::LIMBS / F::BASE_MULS == 12 ? 1.0 : (8.0 * 8.0) / (12.0 * 12.0));
  const double fscale = limb_ratio * F::BASE_MULS;                       // field multiplication cost vs 381-bit Fp
  const double t_madd = 0.352e-6 * fscale * G::COST_MADD / 10.0;         // ms
  const double t_add_tp = 0.93e-6 * fscale * G::COST_ADD / 14.0;         // ms, throughput
  const double t_add_lat = 0.030 * fscale * G::COST_ADD / 14.0;          // ms, dependent chain (2 warps / sub-partition)
  const double t_dbl_par = 0.0062 * fscale;                              // ms per Horner doubling (lane-parallel)
  const int K = 8;
  auto seg_len = [&](double entries) { return plan_seg_len(entries, sm_count, acc_blocks_per_sm<G>()); };
  int best_c = min_c;
  double best = 1e300;
  for (int c = min_c; c <= MAX_WINDOW_BITS; c++) {  // min_c: sharded MSMs run one launch group per window, keep W small
    const int W = (bits + 1 + c - 1) / c;
    const double B = (double)(1u << (c - 1));
    const double entries = terms * W;
    const int L = seg_len(entries);
    const double parts_avg = 1.0 + (terms / B) / L;
    const int top_bits = bits + 1 - (W - 1) * c;                          // scalar bits left for the top window
    const double per_bucket_top = terms / (double)(1u << (top_bits > 1 ? top_bits - 1 : 0));
    double parts_top = 1.0 + per_bucket_top / L;
    if (parts_top > 100.0) parts_top = 100.0 + per_bucket_top / L / 32.0;  // tile sums take over (k_stitch_tiles)
    const double kk = B < K ? B : K;
    const double t_acc = entries * t_madd;
    const double t_r1a = W * B * (1.0 + parts_avg) * t_add_tp, t_r1b = kk * (1.0 + parts_top) * t_add_lat;
    const double cost = t_acc + (t_r1a > t_r1b ? t_r1a : t_r1b) + 0.75 * fscale + (double)(W - 1) * c * t_dbl_par;
    if (cost < best) {
      best = cost;
      best_c = c;
    }
  }
  int c = (forced_c >= 1 && forced_c <= MAX_WINDOW_BITS) ? forced_c : best_c;
  if (c < min_c) c = min_c;
  MsmPlan p;
  p.c = c;
  p.W = (bits + 1 + c - 1) / c;
  p.B = 1 << (c - 1);
  p.G = p.W * p.B;
  const double terms_local = n_local ? (double)n_local * split_of<Cv>() : terms;
  p.L = seg_len(terms_local * p.W);
  // reduce chunk: the first reduction level is a latency chain of 2K additions per chunk, and wants ~2 warps per SM
  // sub-partition (~1000 warps on 132 SMs).  8 buckets per thread does that for the 262144 buckets of a c = 16, 8-window
  // plan; plans with fewer buckets take 4, and at <= 65536 buckets 2 with one chunk per QUAD of lanes (reduce1_quad_form).
  // At 262144 buckets and more, the shorter chunks lose (too few additions per thread to hide the chain).
  const uint64_t nbuckets = (uint64_t)p.W * (uint64_t)p.B;
  int Kc = nbuckets <= 65536u ? 2 : (nbuckets <= 131072u ? 4 : K);
#if !defined(__CUDA_ARCH__)
  if (const char* e = getenv("NMSM_L")) { int v = atoi(e); if (v >= 1 && v <= 1024) p.L = v; }      // tuning experiments
  if (const char* e = getenv("NMSM_K")) { int v = atoi(e); if (v >= 1 && (v & (v - 1)) == 0) Kc = v; }
#endif
  p.K = p.B < Kc ? p.B : Kc;
  p.chunks = p.B / p.K;
  p.D = p.W;
  p.stride = 0;
  p.wb = p.c;
  p.r = 0;
  p.TPW = plan_tpw((uint64_t)terms_local, p.L);
  return p;
}

// first reduction level in the lane-parallel form (k_reduce1<QUAD>)?  see make_plan's reduce chunk
NMSM_HD bool reduce1_quad_form(const MsmPlan& p) { return p.stride == 0 && (uint64_t)p.W * (uint64_t)p.B <= 65536u; }

// Sharded MSM run as one accumulate launch per window (engine.cuh): size the segments so that ONE window is one wave of
// short blocks.  The windows then finish one after the other (instead of all together at the end of two long waves) and
// the bucket exchange / owner reduction of window w overlaps the accumulation of windows w-1..0.
template <class Cv>
inline void plan_one_wave_per_window(MsmPlan& p, uint64_t n_local, int sm_count) {
  const double terms_local = (double)(n_local ? n_local : 1) * split_of<Cv>();
  int L1 = (int)ceil(terms_local / ((double)sm_count * acc_blocks_per_sm<typename Cv::G>() * 128.0));
  p.L = L1 < 4 ? 4 : (L1 > 64 ? 64 : L1);
  p.TPW = plan_tpw((uint64_t)terms_local, p.L);
}

// Fixed-base tables (nmsm_points_precompute): level j of the table holds 2^(offset_j) * P_i for every point of the
// set, so all D digits of a scalar land in ONE bucket window: 1/W of the bucket reduction, no Horner doublings,
// and c can grow past 16 because the reduce cost no longer multiplies by W.  Same time model as make_plan.
// A table is identified by its window bits c; D = ceil((bits+1)/c) digits of width floor/ceil((bits+1)/D).
template <class Cv>
inline int table_digits(int c) { return (glv_bits<Cv>() + 1 + c - 1) / c; }
// the (c, D) pair with D = ceil(T/c) and c = ceil(T/D) reached from a requested upper bound on the digit width
template <class Cv>
inline int canonical_table_bits(int c_req) {
  const int T = glv_bits<Cv>() + 1;
  int c = c_req;
  for (int it = 0; it < 8; it++) {
    const int D = (T + c - 1) / c;
    const int c2 = (T + D - 1) / D;
    if (c2 == c) break;
    c = c2;
  }
  return c;
}

static constexpr int TABLE_REDUCE_CHUNK = 8;  // buckets per k_reduce1 thread in table mode

template <class Cv>
inline int choose_table_bits(uint64_t n_points, int sm_count, double mem_budget_bytes) {
  using G = typename Cv::G;
  using F = typename G::Field;
  const int T = glv_bits<Cv>() + 1;
  const double terms = (double)n_points * split_of<Cv>();
  const double limb_ratio = (double)(F::LIMBS / F::BASE_MULS == 12 ? 1.0 : (8.0 * 8.0) / (12.0 * 12.0));
  const double fscale = limb_ratio * F::BASE_MULS;
  const double t_madd = 0.352e-6 * fscale * G::COST_MADD / 10.0;
  const double t_add_tp = 0.93e-6 * fscale * G::COST_ADD / 14.0;
  const double t_add_lat = 0.006 * fscale * G::COST_ADD / 14.0;  // one dependent addition of a sparse k_reduce1 grid
  const double t_level = 0.2 * fscale;                            // one more k_reduce2 pass (latency)
  int best_c = 4;
  double best = 1e300;
  for (int c0 = 4; c0 <= MAX_TABLE_BITS; c0++) {
    const int c = canonical_table_bits<Cv>(c0);
    if (c != c0) continue;
    const int D = table_digits<Cv>(c);
    if ((double)D * terms * G::AFF_WORDS * 4.0 > mem_budget_bytes && c > 4) continue;
    const int wb = T / D, r = T % D;
    const double B = (double)(1u << (c - 1));
    const double entries = terms * D;
    const int L = plan_seg_len(entries, sm_count, acc_blocks_per_sm<G>());
    // r digits are c bits wide, D - r only c - 1: the lower half of the buckets receives all D digits
    const double load_low = r ? terms * ((double)(D - r) / (double)(1u << (wb - 1)) + (double)r / (double)(1u << wb))
                              : entries / B;
    const double parts_top = 1.0 + load_low / L;
    const double kk = B < TABLE_REDUCE_CHUNK ? B : TABLE_REDUCE_CHUNK;
    const double t_r1a = (entries / L + 2.0 * B) * t_add_tp, t_r1b = kk * (1.0 + parts_top) * t_add_lat;
    const double chunks = B / kk;
    const int levels = chunks <= 4096.0 ? 1 : (chunks <= 524288.0 ? 2 : 3);
    const double cost = entries * t_madd + (t_r1a > t_r1b ? t_r1a : t_r1b) + levels * t_level;
    if (cost < best) {
      best = cost;
      best_c = c;
    }
  }
  return best_c;
}

// `c` must be canonical (canonical_table_bits)
template <class Cv>
inline MsmPlan make_table_plan(uint64_t n_points, int c, int sm_count) {
  MsmPlan p;
  const int T = glv_bits<Cv>() + 1;
  const double terms = (double)n_points * split_of<Cv>();
  p.D = table_digits<Cv>(c);
  p.wb = T / p.D;
  p.r = T % p.D;
  p.c = p.wb + (p.r ? 1 : 0);
  p.W = 1;
  p.B = 1 << (p.c - 1);
  p.G = p.B;
  p.stride = (uint32_t)(n_points * split_of<Cv>());
  p.L = plan_seg_len(terms * p.D, sm_count, acc_blocks_per_sm<typename Cv::G>());
  int Kc = TABLE_REDUCE_CHUNK;
#if !defined(__CUDA_ARCH__)
  if (const char* e = getenv("NMSM_TK")) { int v = atoi(e); if (v >= 1 && (v & (v - 1)) == 0) Kc = v; }  // tuning experiments
#endif
  p.K = p.B < Kc ? p.B : Kc;
  p.chunks = p.B / p.K;
  p.TPW = plan_tpw((uint64_t)terms * p.D, p.L);
  return p;
}

template <class Cv>
inline uint64_t plan_modmuls(const MsmPlan& p, uint64_t entries) {
  using G = typename Cv::G;
  using F = typename G::Field;
  // field-mul equivalents in the base field (Fp2 mul = 3, SURVEY §8d)
  uint64_t per = F::BASE_MULS;
  uint64_t m = entries * G::COST_MADD + (uint64_t)p.W * 2ull * p.B * G::COST_ADD +
               (uint64_t)(p.W - 1) * p.c * G::COST_DBL;
  return m * per;
}

// ---------------------------------------------------------------------------------------------
// memory helpers: rows are multiples of 16 bytes -> 128-bit vector loads/stores on the device
// ---------------------------------------------------------------------------------------------
template <int WORDS>
NMSM_HD void load_words(uint32_t* dst, const uint32_t* src) {
  static_assert(WORDS % 4 == 0, "rows are 16-byte multiples");
#if defined(__CUDA_ARCH__)
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
#pragma unroll
  for (int k = 0; k < WORDS / 4; k++) {
    uint4 v = __ldg(s4 + k);
    dst[4 * k + 0] = v.x;
    dst[4 * k + 1] = v.y;
    dst[4 * k + 2] = v.z;
    dst[4 * k + 3] = v.w;
  }
#else
  for (int k = 0; k < WORDS; k++) dst[k] = src[k];
#endif
}
// same, for buffers written earlier by the same grid sequence (no read-only cache path)
template <int WORDS>
NMSM_HD void load_words_rw(uint32_t* dst, const uint32_t* src) {
#if defined(__CUDA_ARCH__)
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
#pragma unroll
  for (int k = 0; k < WORDS / 4; k++) {
    uint4 v = s4[k];
    dst[4 * k + 0] = v.x;
    dst[4 * k + 1] = v.y;
    dst[4 * k + 2] = v.z;
    dst[4 * k + 3] = v.w;
  }
#else
  for (int k = 0; k < WORDS; k++) dst[k] = src[k];
#endif
}
#if defined(__CUDA_ARCH__)
// Asynchronous copy of WORDS words (16-byte pieces) from global memory to dst[piece][threadIdx.x] in shared memory, as
// one cp.async group: consecutive threads write consecutive 16 bytes, so the stores are free of bank conflicts.
template <int WORDS>
__device__ __forceinline__ void load_words_async(uint4 (*dst)[128], const uint32_t* src) {
  static_assert(WORDS % 4 == 0, "rows are 16-byte multiples");
#pragma unroll
  for (int k = 0; k < WORDS / 4; k++) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(&dst[k][threadIdx.x]);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src + 4 * k) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}
#endif
template <int WORDS>
NMSM_HD void store_words(uint32_t* dst, const uint32_t* src) {
#if defined(__CUDA_ARCH__)
  uint4* d4 = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int k = 0; k < WORDS / 4; k++) d4[k] = make_uint4(src[4 * k], src[4 * k + 1], src[4 * k + 2], src[4 * k + 3]);
#else
  for (int k = 0; k < WORDS; k++) dst[k] = src[k];
#endif
}
NMSM_HD uint32_t atomic_add_u32(unsigned int* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
  return atomicAdd(p, v);
#else
  uint32_t o = *p;
  *p += v;
  return o;
#endif
}
NMSM_HD void atomic_min_u32(unsigned int* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
  atomicMin(p, v);
#else
  if (v < *p) *p = v;
#endif
}

template <class G>
NMSM_HD typename G::Acc load_acc(const uint32_t* src) {
  typename G::Acc a;
  load_words_rw<G::ACC_WORDS>(reinterpret_cast<uint32_t*>(&a), src);
  return a;
}
template <class G>
NMSM_HD void save_acc(uint32_t* dst, const typename G::Acc& a) {
  store_words<G::ACC_WORDS>(dst, reinterpret_cast<const uint32_t*>(&a));
}
template <class G>
NMSM_HD typename G::Affine load_aff(const uint32_t* src) {
  typename G::Affine a;
  load_words<G::AFF_WORDS>(reinterpret_cast<uint32_t*>(&a), src);
  return a;
}

// Out-of-line group operations for the cold kernels (everything except accumulate): one copy of
// each formula per curve keeps code size and ptxas time bounded; the call overhead (accumulators
// passed through local memory) is ~2% of a 14-multiplication addition.
template <class G>
NMSM_NL void nl_add(typename G::Acc& p, const typename G::Acc& q) { G::add(p, q); }
template <class G>
NMSM_NL void nl_dbl(typename G::Acc& p) { G::dbl(p); }
template <class G>
NMSM_NL void nl_madd(typename G::Acc& p, const typename G::Affine& a) { G::madd(p, a); }
template <class G>
NMSM_NL void nl_to_affine(const typename G::Acc& p, uint32_t* xy, uint32_t* inf) {
  G::to_affine_canonical(p, xy, inf);
}

// Group-operation policy of reduce1_body: one logical thread per lane, out-of-line serial formulas (a quad-per-thread
// policy was measured slower there: msm.cuh k_reduce1).
template <class G>
struct SerialOps {
  NMSM_HD static void add(typename G::Acc& p, const typename G::Acc& q) { nl_add<G>(p, q); }
  NMSM_HD static void dbl(typename G::Acc& p) { nl_dbl<G>(p); }
  NMSM_HD static void madd(typename G::Acc& p, const typename G::Affine& q) { nl_madd<G>(p, q); }
};
// same, formulas inlined at the call site (bucket_finalize_body explains why the dense kernels avoid nl_add)
template <class G>
struct InlineOps {
  NMSM_HD static void add(typename G::Acc& p, const typename G::Acc& q) { G::add(p, q); }
  NMSM_HD static void dbl(typename G::Acc& p) { G::dbl(p); }
};

// c bits of a 256-bit little-endian scalar starting at bit `off`
NMSM_HD uint32_t scalar_bits(const uint32_t* s, int off, int c, int nwords = SCALAR_WORDS) {
  int w = off >> 5, sh = off & 31;
  if (w >= nwords) return 0;
  uint64_t lo = s[w];
  uint64_t hi = (w + 1 < nwords) ? s[w + 1] : 0;
  uint64_t v = (lo | (hi << 32)) >> sh;
  return (uint32_t)v & ((1u << c) - 1u);
}

// words of a scalar below the order of Fn: 8 for every curve id of the MSM (SCALAR_WORDS, its input layout), 12 for
// P-384, whose ECDSA bodies pass 12-word scalars to table_mul_body and scalar_mul_acc
template <class Fn>
NMSM_HD constexpr int scalar_words() { return (Fn::BITS + 31) / 32; }

template <class Fn>
NMSM_HD bool scalar_in_range(const uint32_t* s) {
  uint32_t t = sub_cc(s[0], Fn::ORDER(0));
#pragma unroll
  for (int k = 1; k < scalar_words<Fn>(); k++) t = subc_cc(s[k], Fn::ORDER(k));
  (void)t;
  return subc(0, 0) != 0;
}

// ---------------------------------------------------------------------------------------------
// GLV split for curves with r = lambda^2 + lambda + 1 (BLS12-381 G1):
//   k = v1 + v2*lambda (mod r),  |v1|, |v2| <= lambda/2 + 1 < 2^127
// q = floor(k / lambda) by a Barrett step with MU = floor(2^256 / lambda) (at most one correction),
// then both halves are centred using lambda^2 + lambda = -1 (mod r).
// ---------------------------------------------------------------------------------------------
NMSM_HD bool gt4(const uint32_t* a, const uint32_t* b) {  // a > b, 4 limbs
  for (int k = 3; k >= 0; k--) {
    if (a[k] != b[k]) return a[k] > b[k];
  }
  return false;
}
NMSM_HD void sub4(uint32_t* r, const uint32_t* a, const uint32_t* b) {  // r = a - b (a >= b)
  uint64_t br = 0;
  for (int k = 0; k < 4; k++) {
    uint64_t t = (uint64_t)a[k] - b[k] - br;
    r[k] = (uint32_t)t;
    br = (t >> 63) & 1;
  }
}
NMSM_HD void inc4(uint32_t* a) {
  for (int k = 0; k < 4; k++)
    if (++a[k] != 0) break;
}
NMSM_HD void dec4(uint32_t* a) {
  for (int k = 0; k < 4; k++)
    if (a[k]-- != 0) break;
}
template <class GC>
NMSM_HD void glv_split(const uint32_t* k, uint32_t* m1, bool& neg1, uint32_t* m2, bool& neg2) {
  uint32_t lam[4], half[4], lp1[4];
  for (int i = 0; i < 4; i++) lam[i] = GC::LAMBDA(i);
  for (int i = 0; i < 4; i++) half[i] = (lam[i] >> 1) | (i < 3 ? lam[i + 1] << 31 : 0);
  for (int i = 0; i < 4; i++) lp1[i] = lam[i];
  inc4(lp1);
  // q = (k * MU) >> 256
  uint32_t prod[13];
  for (int i = 0; i < 13; i++) prod[i] = 0;
  for (int i = 0; i < 8; i++) {
    uint64_t carry = 0;
    for (int j = 0; j < 5; j++) {
      uint64_t t = (uint64_t)k[i] * GC::MU(j) + prod[i + j] + carry;
      prod[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
    prod[i + 5] = (uint32_t)carry;
  }
  uint32_t q[5];
  for (int i = 0; i < 5; i++) q[i] = prod[8 + i];
  // r = k - q*lambda, low 5 limbs (0 <= r < 2*lambda)
  uint32_t t[5] = {0, 0, 0, 0, 0};
  for (int i = 0; i < 5; i++) {
    uint64_t carry = 0;
    for (int j = 0; j < 4 && i + j < 5; j++) {
      uint64_t x = (uint64_t)q[i] * lam[j] + t[i + j] + carry;
      t[i + j] = (uint32_t)x;
      carry = x >> 32;
    }
    if (i == 0) t[4] += (uint32_t)carry;  // only row 0 ends below limb 5; t[4] is still zero here
  }
  uint32_t r[5];
  {
    uint64_t br = 0;
    for (int i = 0; i < 5; i++) {
      uint64_t x = (uint64_t)k[i] - t[i] - br;
      r[i] = (uint32_t)x;
      br = (x >> 63) & 1;
    }
  }
  if (r[4] != 0 || !gt4(lam, r)) {  // r >= lambda
    uint64_t br = 0;
    for (int i = 0; i < 4; i++) {
      uint64_t x = (uint64_t)r[i] - lam[i] - br;
      r[i] = (uint32_t)x;
      br = (x >> 63) & 1;
    }
    inc4(q);
  }
  for (int i = 0; i < 4; i++) {
    m1[i] = r[i];
    m2[i] = q[i];
  }
  neg1 = false;
  neg2 = false;
  if (gt4(m1, half)) {  // v1 = k1 - lambda, borrow one lambda from v2
    sub4(m1, lam, m1);
    neg1 = true;
    inc4(m2);
  }
  if (gt4(m2, half)) {  // v2 = k2 - (lambda + 1); (lambda + 1)*lambda = -1  =>  v1 -= 1
    if (gt4(lp1, m2)) {
      sub4(m2, lp1, m2);
      neg2 = true;
    } else {
      sub4(m2, m2, lp1);
    }
    if (neg1) {
      inc4(m1);
    } else if ((m1[0] | m1[1] | m1[2] | m1[3]) == 0) {
      m1[0] = 1;
      neg1 = true;
    } else {
      dec4(m1);
    }
  }
}

// Lattice GLV split (secp256k1, bn254 G1), the device form of weierstrass.ts:121-148 `_splitEndoScalar`:
//   c1 = round(b2*k/n) = (k*G1 + 2^383) >> 384,  c2 = round(-b1*k/n) = (k*G2 + 2^383) >> 384
//   k1 = k - c1*a1 - c2*a2,   k2 = -c1*b1 - c2*b2 = c1*|b1| - c2*b2      (a1, a2, b2 > 0 > b1)
// evaluated in 320-bit two's complement; outputs are 5-limb magnitudes (< 2^BITS) and signs.
template <class GC>
NMSM_HD void glv_split_lattice(const uint32_t* k, uint32_t* m1, bool& neg1, uint32_t* m2, bool& neg2) {
  auto mul_shift = [&](auto g, uint32_t* c) {  // c[5] = (k * g + 2^383) >> 384
    uint32_t prod[17];
    for (int i = 0; i < 17; i++) prod[i] = 0;
    for (int i = 0; i < 8; i++) {
      uint64_t carry = 0;
      for (int j = 0; j < 9; j++) {
        uint64_t t = (uint64_t)k[i] * g(j) + prod[i + j] + carry;
        prod[i + j] = (uint32_t)t;
        carry = t >> 32;
      }
      prod[i + 9] = (uint32_t)carry;
    }
    uint64_t carry = 0x80000000ull;  // + 2^383: bit 31 of limb 11
    for (int i = 11; i < 17; i++) {
      uint64_t t = (uint64_t)prod[i] + carry;
      prod[i] = (uint32_t)t;
      carry = t >> 32;
    }
    for (int i = 0; i < 5; i++) c[i] = prod[12 + i];
  };
  auto mul5 = [](const uint32_t* a, auto b, uint32_t* r) {  // r[10] = a[5] * b[5]
    for (int i = 0; i < 10; i++) r[i] = 0;
    for (int i = 0; i < 5; i++) {
      uint64_t carry = 0;
      for (int j = 0; j < 5; j++) {
        uint64_t t = (uint64_t)a[i] * b(j) + r[i + j] + carry;
        r[i + j] = (uint32_t)t;
        carry = t >> 32;
      }
      r[i + 5] = (uint32_t)carry;
    }
  };
  auto sub10 = [](uint32_t* x, const uint32_t* y) {  // x -= y mod 2^320
    uint64_t br = 0;
    for (int i = 0; i < 10; i++) {
      uint64_t t = (uint64_t)x[i] - y[i] - br;
      x[i] = (uint32_t)t;
      br = (t >> 63) & 1;
    }
  };
  auto abs10 = [](uint32_t* x, bool& neg) {  // two's complement -> magnitude
    neg = (x[9] >> 31) != 0;
    if (neg) {
      uint64_t carry = 1;
      for (int i = 0; i < 10; i++) {
        uint64_t t = (uint64_t)(~x[i]) + carry;
        x[i] = (uint32_t)t;
        carry = t >> 32;
      }
    }
  };
  uint32_t c1[5], c2[5], t[10], v1[10], v2[10];
  mul_shift([](int j) { return GC::G1(j); }, c1);
  mul_shift([](int j) { return GC::G2(j); }, c2);
  for (int i = 0; i < 10; i++) v1[i] = i < 8 ? k[i] : 0;
  mul5(c1, [](int j) { return GC::A1(j); }, t);
  sub10(v1, t);
  mul5(c2, [](int j) { return GC::A2(j); }, t);
  sub10(v1, t);
  mul5(c1, [](int j) { return GC::B1ABS(j); }, v2);
  mul5(c2, [](int j) { return GC::B2(j); }, t);
  sub10(v2, t);
  abs10(v1, neg1);
  abs10(v2, neg2);
  for (int i = 0; i < 5; i++) {
    m1[i] = v1[i];
    m2[i] = v2[i];
  }
}

// ---------------------------------------------------------------------------------------------
// psi-GLS split (BLS12-381 G2, GLV_KIND 3): balanced digits of k in base z = |x| (the 64-bit curve parameter),
//   k = k0 + k1 z + k2 z^2 + k3 z^3 (mod r),  |k_i| <= z/2 + 1 < 2^63,
// attached to P, -psi(P), psi^2(P), -psi^3(P) (psi(P) = [x]P = -[z]P on the prime-order subgroup, bls12-381.ts:600).
// Three schoolbook divisions by the normalised two-word z (Knuth D with a one-word quotient estimate), then the digits
// are centred; a carry out of the top digit is folded back with z^4 = z^2 - 1 (mod r = z^4 - z^2 + 1).
// ---------------------------------------------------------------------------------------------
// u (nw words, little-endian) := floor(u / z); returns u mod z.  z = z1 * 2^32 + z0 with bit 31 of z1 set.
NMSM_HD uint64_t divmod_2w(uint32_t* u, int nw, uint32_t z1, uint32_t z0) {
  uint64_t rem = 0;  // < z
  for (int i = nw - 1; i >= 0; i--) {
    // cur = rem * 2^32 + u[i] (96 bits, held as hi = bits 32.., lo = bits 0..31); the quotient word is < 2^32
    const uint64_t cur_hi = rem;
    const uint32_t cur_lo = u[i];
    uint64_t q = cur_hi / z1;
    if (q > 0xffffffffull) q = 0xffffffffull;
    uint64_t p0 = q * z0, p1 = q * z1;
    uint64_t prod_hi = p1 + (p0 >> 32);
    uint32_t prod_lo = (uint32_t)p0;
    // the estimate exceeds the true quotient word by at most 2
    for (int it = 0; it < 3 && (prod_hi > cur_hi || (prod_hi == cur_hi && prod_lo > cur_lo)); it++) {
      q--;
      const uint32_t br = prod_lo < z0 ? 1u : 0u;
      prod_lo -= z0;
      prod_hi -= (uint64_t)z1 + br;
    }
    const uint32_t br = cur_lo < prod_lo ? 1u : 0u;
    const uint32_t d_lo = cur_lo - prod_lo;
    const uint64_t d_hi = cur_hi - prod_hi - br;  // < 2^32
    rem = (d_hi << 32) | d_lo;
    u[i] = (uint32_t)q;
  }
  return rem;
}
// (mag, neg) += delta for delta = +-1
NMSM_HD void signed_adjust(uint64_t& mag, bool& neg, int delta) {
  const bool dneg = delta < 0;
  if (mag == 0) {
    mag = 1;
    neg = dneg;
  } else if (neg == dneg) {
    mag += 1;
  } else {
    mag -= 1;
    if (mag == 0) neg = false;
  }
}
template <class Gls>
NMSM_HD void gls_split(const uint32_t* s, uint64_t* mag, bool* neg) {
  const uint32_t z0 = Gls::Z(0), z1 = Gls::Z(1);
  const uint64_t z = ((uint64_t)z1 << 32) | z0, half = ((uint64_t)Gls::HALF(1) << 32) | Gls::HALF(0);
  uint32_t q[SCALAR_WORDS];
  for (int k = 0; k < SCALAR_WORDS; k++) q[k] = s[k];
  uint64_t d[4];
  d[0] = divmod_2w(q, 8, z1, z0);
  d[1] = divmod_2w(q, 6, z1, z0);
  d[2] = divmod_2w(q, 4, z1, z0);
  d[3] = ((uint64_t)q[1] << 32) | q[0];  // k < r < z^4
  uint32_t carry = 0;
  for (int i = 0; i < 4; i++) {
    const uint64_t u = d[i] + carry;  // <= z
    if (u > half) {
      mag[i] = z - u;
      neg[i] = true;
      carry = 1;
    } else {
      mag[i] = u;
      neg[i] = false;
      carry = 0;
    }
  }
  if (carry) {  // + z^4 = z^2 - 1
    signed_adjust(mag[2], neg[2], +1);
    signed_adjust(mag[0], neg[0], -1);
  }
}

// ---------------------------------------------------------------------------------------------
// bodies
// ---------------------------------------------------------------------------------------------
// err[0] = min index of an out-of-range point coordinate, err[1] = min index of an invalid scalar
template <class Cv>
NMSM_HD void prepare_body(uint32_t i, uint32_t n, const uint32_t* pts, uint32_t* aff, unsigned int* err) {
  using G = typename Cv::G;
  uint32_t in[G::IN_WORDS];
  load_words<G::IN_WORDS>(in, pts + (size_t)i * G::IN_WORDS);
  if (!G::input_in_range(in)) {
    atomic_min_u32(&err[0], i);
    return;
  }
  typename G::Affine a = G::prepare(in);
  store_words<G::AFF_WORDS>(aff + (size_t)i * G::AFF_WORDS, reinterpret_cast<const uint32_t*>(&a));
  if constexpr (Cv::GLV_KIND == 3) {  // psi^j(P) at index j*n + i, j = 1..3; (0,0) stays the identity
    using F2 = typename G::Field;
    using B = typename F2::Base;
    using Gls = typename Cv::Glv;
    F2 px, py, p3x, p3y;
    B p2x;
    for (int k = 0; k < B::LIMBS; k++) {
      px.c0.v[k] = Gls::PSI_X_C0_MONT(k);
      px.c1.v[k] = Gls::PSI_X_C1_MONT(k);
      py.c0.v[k] = Gls::PSI_Y_C0_MONT(k);
      py.c1.v[k] = Gls::PSI_Y_C1_MONT(k);
      p3x.c0.v[k] = Gls::PSI3_X_C0_MONT(k);
      p3x.c1.v[k] = Gls::PSI3_X_C1_MONT(k);
      p3y.c0.v[k] = Gls::PSI3_Y_C0_MONT(k);
      p3y.c1.v[k] = Gls::PSI3_Y_C1_MONT(k);
      p2x.v[k] = Gls::PSI2_X_MONT(k);
    }
    const F2 cx{a.x.c0, -a.x.c1}, cy{a.y.c0, -a.y.c1};  // Frobenius = conjugation
    typename G::Affine t;
    t.x = cx * px;
    t.y = cy * py;
    store_words<G::AFF_WORDS>(aff + (size_t)(n + i) * G::AFF_WORDS, reinterpret_cast<const uint32_t*>(&t));
    t.x = F2{a.x.c0 * p2x, a.x.c1 * p2x};
    t.y = -a.y;
    store_words<G::AFF_WORDS>(aff + (size_t)(2 * (size_t)n + i) * G::AFF_WORDS, reinterpret_cast<const uint32_t*>(&t));
    t.x = cx * p3x;
    t.y = cy * p3y;
    store_words<G::AFF_WORDS>(aff + (size_t)(3 * (size_t)n + i) * G::AFF_WORDS, reinterpret_cast<const uint32_t*>(&t));
  } else if constexpr (Cv::GLV) {  // phi(P) = (beta * x, y) at index n + i; (0,0) stays the identity
    typename G::Field beta;
    for (int k = 0; k < G::Field::LIMBS; k++) beta.v[k] = Cv::Glv::BETA_MONT(k);
    a.x = a.x * beta;
    store_words<G::AFF_WORDS>(aff + (size_t)(n + i) * G::AFF_WORDS, reinterpret_cast<const uint32_t*>(&a));
  }
}

// One level of a fixed-base table: next[i] = 2^c * prev[i], back in the prepared affine layout (one xgcd
// inversion per point; a one-off cost paid by nmsm_points_precompute).
template <class Cv>
NMSM_HD void table_level_body(uint32_t i, const uint32_t* prev, uint32_t* next, int c) {
  using G = typename Cv::G;
  typename G::Affine a = load_aff<G>(prev + (size_t)i * G::AFF_WORDS);
  typename G::Acc acc = G::from_affine(a);
  for (int j = 0; j < c; j++) nl_dbl<G>(acc);
  a = G::to_affine_prepared(acc);
  store_words<G::AFF_WORDS>(next + (size_t)i * G::AFF_WORDS, reinterpret_cast<const uint32_t*>(&a));
}

// ---- fixed-point multiplication tables (nmsm_point_table_*) -------------------------------------------
// The device-resident form of Point.precompute(W) + the cached signed-window walk (curve.ts:532-577 table,
// :588-606 walk): tbl[j][d-1] = d * 2^(16 j) * P for d in [1, 2^15], j < levels, prepared affine layout.  One
// multiplication is then `levels` mixed additions and NO doublings; the table (36-107 MB) lives in L2/HBM.
static constexpr int PT_BITS = 16;
static constexpr uint32_t PT_HALF = 1u << (PT_BITS - 1);
// BITS is a template parameter only so that tests/hostemu can run the same bodies with small tables
template <class Cv, int BITS = PT_BITS>
NMSM_HD constexpr int point_table_levels() { return (Cv::Fn::BITS + 1 + BITS - 1) / BITS; }

// level 0 entry i: (i + 1) * P by BITS double-and-add steps
template <class Cv, int BITS = PT_BITS>
NMSM_HD void table_base_body(uint32_t i, const uint32_t* p_aff, uint32_t* level0) {
  using G = typename Cv::G;
  const typename G::Affine P = load_aff<G>(p_aff);
  typename G::Acc acc = G::identity();
  const uint32_t k = i + 1;
  for (int b = BITS - 1; b >= 0; b--) {
    nl_dbl<G>(acc);
    if ((k >> b) & 1u) nl_madd<G>(acc, P);
  }
  typename G::Affine a = G::to_affine_prepared(acc);
  store_words<G::AFF_WORDS>(level0 + (size_t)i * G::AFF_WORDS, reinterpret_cast<const uint32_t*>(&a));
}

// acc += s * P by the signed BITS-bit digit walk: level w of the table holds d * 2^(BITS w) * P for d in [1, 2^(BITS-1)]
// at tbl + (w * STRIDE + d - 1) * AFF_WORDS; s has scalar_words<Fn>() words.  One gathered mixed addition per non-zero
// digit and no doublings.  A nmsm_point_table_* table holds one point (STRIDE = 2^(BITS-1)); the EIP-4844 setup table
// (kzg.cuh) interleaves its points within each level.
template <class Cv, int BITS, size_t STRIDE>
NMSM_HD void table_walk_acc(const uint32_t* tbl, const uint32_t* s, typename Cv::G::Acc& acc) {
  using G = typename Cv::G;
  constexpr uint32_t HALF = 1u << (BITS - 1);
  constexpr int SW = scalar_words<typename Cv::Fn>();
  uint32_t carry = 0;
  constexpr int LEVELS = point_table_levels<Cv, BITS>();
  for (int w = 0; w < LEVELS; w++) {
    uint32_t v = scalar_bits(s, w * BITS, BITS, SW) + carry;
    carry = 0;
    bool neg = false;
    if (v > HALF) {
      v = (1u << BITS) - v;
      neg = true;
      carry = 1;
    }
    if (v != 0) {
      typename G::Affine a = load_aff<G>(tbl + ((size_t)w * STRIDE + (v - 1)) * G::AFF_WORDS);
      a = G::cneg(a, neg);
      nl_madd<G>(acc, a);
    }
  }
}

// k * P from the table as an un-normalised accumulator; scalars are scalar_words<Fn>() words each.  Returns false (and records the index) for a scalar
// outside Point.multiply's range 1 <= k < n (allow_zero: multiplyUnsafe's 0 <= k < n).
template <class Cv, int BITS = PT_BITS>
NMSM_HD bool table_mul_body(uint32_t i, const uint32_t* tbl, const uint32_t* scalars, int allow_zero,
                            typename Cv::G::Acc& acc, unsigned int* err) {
  using G = typename Cv::G;
  constexpr uint32_t HALF = 1u << (BITS - 1);
  constexpr int SW = scalar_words<typename Cv::Fn>();
  uint32_t s[SW];
  load_words<SW>(s, scalars + (size_t)i * SW);
  uint32_t nz = 0;
  for (int k = 0; k < SW; k++) nz |= s[k];
  acc = G::identity();
  if (!scalar_in_range<typename Cv::Fn>(s) || (!allow_zero && nz == 0)) {
    atomic_min_u32(&err[1], i);
    return false;
  }
  table_walk_acc<Cv, BITS, HALF>(tbl, s, acc);
  return true;
}

// Signed-digit recoding of one magnitude shared by the count and scatter passes: digit d_w in
// [-(2^(c-1)-1), 2^(c-1)], sum d_w 2^(cw) = m (the fixed-window analogue of curve.ts:454-472
// signedWindowDigits).  Bucket id g = w*B + |d| - 1, weight |d|; the sign rides in bit 31 of the entry.
template <bool SCATTER>
NMSM_HD void emit_digits(const uint32_t* m, int nwords, uint32_t index, uint32_t flip, const MsmPlan& plan,
                         unsigned int* counts_or_cursor, uint32_t* sorted) {
  uint32_t carry = 0;
  for (int w = 0; w < plan.D; w++) {
    const int width = digit_width(plan, w);
    const uint32_t half = 1u << (width - 1);
    uint32_t v = scalar_bits(m, digit_offset(plan, w), width, nwords) + carry;
    carry = 0;
    uint32_t neg = flip;
    if (v > half) {
      v = (1u << width) - v;
      neg ^= 1u;
      carry = 1;
    }
    if (v != 0) {
      const uint32_t g = (plan.stride ? 0u : (uint32_t)w * (uint32_t)plan.B) + (v - 1);
      if (SCATTER) {
        uint32_t pos = atomic_add_u32(&counts_or_cursor[g], 1u);
        sorted[pos] = (index + (uint32_t)w * plan.stride) | (neg << 31);
      } else {
        atomic_add_u32(&counts_or_cursor[g], 1u);
      }
    }
  }
}

template <class Cv, bool SCATTER>
NMSM_HD void digits_body(uint32_t i, uint32_t n, const uint32_t* scalars, const MsmPlan& plan,
                         unsigned int* counts_or_cursor, uint32_t* sorted, unsigned int* err) {
  uint32_t s[SCALAR_WORDS];
  load_words<SCALAR_WORDS>(s, scalars + (size_t)i * SCALAR_WORDS);
  if (!scalar_in_range<typename Cv::Fn>(s)) {  // same decision in both passes keeps count == scatter
    if (!SCATTER) atomic_min_u32(&err[1], i);
    return;
  }
  if constexpr (Cv::GLV_KIND == 1) {
    uint32_t m1[4], m2[4];
    bool neg1, neg2;
    glv_split<typename Cv::Glv>(s, m1, neg1, m2, neg2);
    emit_digits<SCATTER>(m1, 4, i, neg1 ? 1u : 0u, plan, counts_or_cursor, sorted);
    emit_digits<SCATTER>(m2, 4, n + i, neg2 ? 1u : 0u, plan, counts_or_cursor, sorted);
  } else if constexpr (Cv::GLV_KIND == 2) {
    uint32_t m1[5], m2[5];
    bool neg1, neg2;
    glv_split_lattice<typename Cv::Glv>(s, m1, neg1, m2, neg2);
    emit_digits<SCATTER>(m1, 5, i, neg1 ? 1u : 0u, plan, counts_or_cursor, sorted);
    emit_digits<SCATTER>(m2, 5, n + i, neg2 ? 1u : 0u, plan, counts_or_cursor, sorted);
  } else if constexpr (Cv::GLV_KIND == 3) {
    uint64_t mag[4];
    bool neg[4];
    gls_split<typename Cv::Glv>(s, mag, neg);
    for (int j = 0; j < 4; j++) {  // k_j against (-1)^j psi^j(P)
      const uint32_t m[2] = {(uint32_t)mag[j], (uint32_t)(mag[j] >> 32)};
      emit_digits<SCATTER>(m, 2, (uint32_t)j * n + i, (neg[j] ? 1u : 0u) ^ (uint32_t)(j & 1), plan, counts_or_cursor, sorted);
    }
  } else {
    emit_digits<SCATTER>(s, SCALAR_WORDS, i, 0u, plan, counts_or_cursor, sorted);
  }
}

// Balanced bucket accumulation: segment (w, t) owns L consecutive sorted entries of window w (see MsmPlan::TPW).
// Constant work per thread whatever the bucket sizes; a bucket that is wholly inside the segment is written straight
// to `buckets`, a bucket cut by the segment start goes to heads[sid], one cut by the end to tails[sid], with
// sid = w * TPW + t the global segment id.
template <class Cv>
NMSM_HD void accumulate_body(uint32_t w, uint32_t t, const uint32_t* aff, const uint32_t* sorted, const uint32_t* offsets,
                             const MsmPlan& plan, uint32_t* buckets, uint32_t* heads, uint32_t* tails) {
  using G = typename Cv::G;
  const uint32_t g_lo = w * (uint32_t)plan.B, g_hi = g_lo + (uint32_t)plan.B;
  const uint32_t base = offsets[g_lo], T = offsets[g_hi];  // this window's slice of the sorted array
  const uint64_t seg64 = (uint64_t)base + (uint64_t)t * (uint32_t)plan.L;
  if (seg64 >= T) return;
  const uint32_t seg = (uint32_t)seg64;
  const uint32_t end = (T - seg > (uint32_t)plan.L) ? seg + plan.L : T;
  const size_t sid = (size_t)w * plan.TPW + t;
  // bucket containing `seg`: the last g of this window with offsets[g] <= seg
  uint32_t lo = g_lo, hi = g_hi;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (offsets[mid] <= seg) lo = mid; else hi = mid;
  }
  uint32_t g = lo;
  uint32_t bstart = offsets[g], bend = offsets[g + 1];
  typename G::Acc acc = G::identity();
  // bucket g is finished inside this segment at entry pos: flush it, move on to the bucket of pos
  auto next_bucket = [&](uint32_t pos) {
    if (bstart >= seg) save_acc<G>(buckets + (size_t)g * G::ACC_WORDS, acc);
    else save_acc<G>(heads + sid * G::ACC_WORDS, acc);
    acc = G::identity();
    do { g++; } while (offsets[g + 1] <= pos);
    bstart = offsets[g];
    bend = offsets[g + 1];
  };
#if defined(__CUDA_ARCH__)
  if constexpr (acc_inline_products<G>()) {
    // The point of entry pos + 1 is requested before the addition of entry pos (cp.async into a per-thread double buffer
    // in shared memory, 2 x AFF_WORDS words per thread, no registers), and the sorted index two entries ahead: the
    // gathers' latency hides behind one mixed addition.  At 3 blocks per SM too few warps are resident to hide it.
    // k_accumulate runs 128-thread blocks.
    constexpr int Q = G::AFF_WORDS / 4;
    __shared__ uint4 next_pts[2][Q][128];
    uint32_t e = sorted[seg], e_next = seg + 1 < end ? sorted[seg + 1] : 0u;
    load_words_async<G::AFF_WORDS>(next_pts[0], aff + (size_t)(e & 0x7fffffffu) * G::AFF_WORDS);
    for (uint32_t pos = seg, slot = 0; pos < end; pos++, slot ^= 1u) {
      if (pos == bend) next_bucket(pos);
      const uint32_t e_after = pos + 2 < end ? sorted[pos + 2] : 0u;
      if (pos + 1 < end) load_words_async<G::AFF_WORDS>(next_pts[slot ^ 1u], aff + (size_t)(e_next & 0x7fffffffu) * G::AFF_WORDS);
      else asm volatile("cp.async.commit_group;" ::: "memory");  // empty group: the wait below then means "entry pos"
      asm volatile("cp.async.wait_group 1;" ::: "memory");          // all groups but the newest are complete
      typename G::Affine a;
      uint32_t* aw = reinterpret_cast<uint32_t*>(&a);
#pragma unroll
      for (int k = 0; k < Q; k++) {
        const uint4 v = next_pts[slot][k][threadIdx.x];
        aw[4 * k] = v.x;
        aw[4 * k + 1] = v.y;
        aw[4 * k + 2] = v.z;
        aw[4 * k + 3] = v.w;
      }
      a = G::cneg(a, (e >> 31) != 0);
      G::template madd<true>(acc, a);
      e = e_next;
      e_next = e_after;
    }
  } else
#endif
  {
    for (uint32_t pos = seg; pos < end; pos++) {
      if (pos == bend) next_bucket(pos);
      uint32_t e = sorted[pos];
      typename G::Affine a = load_aff<G>(aff + (size_t)(e & 0x7fffffffu) * G::AFF_WORDS);
      a = G::cneg(a, (e >> 31) != 0);
      if constexpr (acc_inline_products<G>()) G::template madd<true>(acc, a);
      else G::madd(acc, a);
    }
  }
  const bool head_open = bstart < seg;
  const bool tail_open = bend > end;
  if (!head_open && !tail_open) save_acc<G>(buckets + (size_t)g * G::ACC_WORDS, acc);
  else if (head_open) save_acc<G>(heads + sid * G::ACC_WORDS, acc);
  else save_acc<G>(tails + sid * G::ACC_WORDS, acc);
}

// ---- paired accumulation (short Weierstrass) ---------------------------------------------------------------------
// Two neighbours of the same bucket are first added in AFFINE coordinates, lambda = (y2 - y1) / (x2 - x1), and only the
// sum goes through the mixed addition into the XYZZ accumulator.  The division costs one inversion per WARP and segment:
// every thread multiplies up the denominators of its pairs (pass 1), the 32 running products are inverted together
// (k_accumulate: warp_batch_inverse — Montgomery's trick, the reference's FpInvertBatch modular.ts:734-760), and pass 2
// peels the individual inverses off again.  Per pair: 3 multiplications for the shared inversion + 3 for the affine
// addition (2M + 1S) + 10 for the mixed addition = 16 instead of 20 for two mixed additions.
// Pairs are fixed by parity relative to the bucket start, (b0 + 2j, b0 + 2j + 1), as far as both entries lie inside the
// thread's segment; a pair whose x coordinates coincide (P = +-Q: doubling or cancellation) or contain a zero (the
// affine identity has x = 0) is left to the complete mixed addition, one entry at a time.  Both passes take that
// decision from the same data, so they agree.
static constexpr int MAX_PAIRS = 32;  // L <= 64 entries per segment

template <class F>
NMSM_HD bool pair_usable(const F& x1, const F& x2) {
  return !x1.is_zero() && !x2.is_zero() && x1 != x2;
}

// Pass 1, backwards over the segment's pairs: suf[j] = product of the denominators of the pairs AFTER pair (M-1-j) in
// forward order, i.e. suf is filled in the order the pairs are met walking down.  Returns the product of all of them
// (one() if the thread has no pair) and the pair count in `npairs`.
template <class Cv>
NMSM_HD typename Cv::G::Field accumulate_pairs_pass1(uint32_t w, uint32_t t, const uint32_t* aff, const uint32_t* sorted,
                                                     const uint32_t* offsets, const MsmPlan& plan,
                                                     typename Cv::G::Field* suf, int& npairs) {
  using G = typename Cv::G;
  using F = typename G::Field;
  npairs = 0;
  F run = F::one();
  const uint32_t g_lo = w * (uint32_t)plan.B, g_hi = g_lo + (uint32_t)plan.B;
  const uint32_t base = offsets[g_lo], T = offsets[g_hi];
  const uint64_t seg64 = (uint64_t)base + (uint64_t)t * (uint32_t)plan.L;
  if (seg64 >= T) return run;
  const uint32_t seg = (uint32_t)seg64;
  const uint32_t end = (T - seg > (uint32_t)plan.L) ? seg + plan.L : T;
  // bucket containing the LAST entry of the segment
  uint32_t lo = g_lo, hi = g_hi;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (offsets[mid] <= end - 1) lo = mid; else hi = mid;
  }
  uint32_t g = lo;
  uint32_t pos = end;  // walk down: [.., pos) still to do
  while (pos > seg) {
    while (offsets[g] >= pos) g--;  // bucket of entry pos - 1 (skips empty buckets)
    const uint32_t b0 = offsets[g];
    const uint32_t rs = b0 > seg ? b0 : seg;  // run [rs, pos) of bucket g inside the segment
    // pair starts p = b0 (mod 2) with rs <= p and p + 1 < pos, from the last one down (signed: p may step below 0)
    if (pos - rs >= 2) {
      long long p = (long long)pos - 2;
      if ((((uint32_t)p - b0) & 1u) != 0) p--;
      for (; p >= (long long)rs; p -= 2) {
        const uint32_t e1 = sorted[p], e2 = sorted[p + 1];
        F x1, x2;
        load_words<F::LIMBS>(reinterpret_cast<uint32_t*>(&x1), aff + (size_t)(e1 & 0x7fffffffu) * G::AFF_WORDS);
        load_words<F::LIMBS>(reinterpret_cast<uint32_t*>(&x2), aff + (size_t)(e2 & 0x7fffffffu) * G::AFF_WORDS);
        if (pair_usable(x1, x2)) {
          suf[npairs++] = run;
          run = run * (x2 - x1);
        }
      }
    }
    pos = rs;
  }
  return run;
}

// Pass 2, forwards: the accumulate loop of accumulate_body with usable pairs replaced by their affine sum.
// `inv_all` = 1 / (product returned by pass 1).
template <class Cv>
NMSM_HD void accumulate_pairs_pass2(uint32_t w, uint32_t t, const uint32_t* aff, const uint32_t* sorted, const uint32_t* offsets,
                                    const MsmPlan& plan, const typename Cv::G::Field* suf, int npairs,
                                    typename Cv::G::Field inv_all, uint32_t* buckets, uint32_t* heads, uint32_t* tails) {
  using G = typename Cv::G;
  using F = typename G::Field;
  const uint32_t g_lo = w * (uint32_t)plan.B, g_hi = g_lo + (uint32_t)plan.B;
  const uint32_t base = offsets[g_lo], T = offsets[g_hi];
  const uint64_t seg64 = (uint64_t)base + (uint64_t)t * (uint32_t)plan.L;
  if (seg64 >= T) return;
  const uint32_t seg = (uint32_t)seg64;
  const uint32_t end = (T - seg > (uint32_t)plan.L) ? seg + plan.L : T;
  const size_t sid = (size_t)w * plan.TPW + t;
  uint32_t lo = g_lo, hi = g_hi;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (offsets[mid] <= seg) lo = mid; else hi = mid;
  }
  uint32_t g = lo;
  uint32_t bstart = offsets[g], bend = offsets[g + 1];
  typename G::Acc acc = G::identity();
  int k = 0;  // usable pairs consumed so far (forward order); pass 1 stored pair k at suf[npairs - 1 - k]
  for (uint32_t pos = seg; pos < end;) {
    if (pos == bend) {
      if (bstart >= seg) save_acc<G>(buckets + (size_t)g * G::ACC_WORDS, acc);
      else save_acc<G>(heads + sid * G::ACC_WORDS, acc);
      acc = G::identity();
      do { g++; } while (offsets[g + 1] <= pos);
      bstart = offsets[g];
      bend = offsets[g + 1];
    }
    const uint32_t e1 = sorted[pos];
    const uint32_t* p1 = aff + (size_t)(e1 & 0x7fffffffu) * G::AFF_WORDS;
    const uint32_t rs = bstart > seg ? bstart : seg;
    const uint32_t re = bend < end ? bend : end;
    // a pair start: even offset from the bucket start, partner inside the same run (pass 1 enumerated exactly these:
    // pairs (p, p+1) with p = bstart (mod 2), rs <= p, p + 1 < re)
    // ONE mixed addition per iteration, of either the affine sum of a usable pair or the single entry at `pos` (an
    // unusable pair — P = +-Q, or a zero x: the affine identity — is simply taken as two single entries): a single call
    // site keeps the accumulator in registers; everything live across an out-of-line multiplication is spilled, so the
    // coordinates are loaded as late and dropped as early as possible.
    typename G::Affine r;
    bool paired = false;
    if (((pos - bstart) & 1u) == 0 && pos >= rs && pos + 1 < re) {
      const uint32_t e2 = sorted[pos + 1];
      const uint32_t* p2 = aff + (size_t)(e2 & 0x7fffffffu) * G::AFF_WORDS;
      F x1, x2;
      load_words<F::LIMBS>(reinterpret_cast<uint32_t*>(&x1), p1);
      load_words<F::LIMBS>(reinterpret_cast<uint32_t*>(&x2), p2);
      if (pair_usable(x1, x2)) {
        paired = true;
        const F d = x2 - x1;
        const F sx = x1 + x2;
        const F dinv = inv_all * suf[npairs - 1 - k];
        inv_all = inv_all * d;
        k++;
        F y1, y2;
        load_words<F::LIMBS>(reinterpret_cast<uint32_t*>(&y1), p1 + F::LIMBS);
        load_words<F::LIMBS>(reinterpret_cast<uint32_t*>(&y2), p2 + F::LIMBS);
        if ((e1 >> 31) != 0) y1 = -y1;
        if ((e2 >> 31) != 0) y2 = -y2;
        const F lam = (y2 - y1) * dinv;
        r.x = sqr(lam) - sx;
        r.y = lam * (x1 - r.x) - y1;
      }
    }
    if (!paired) {
      r = load_aff<G>(p1);
      r = G::cneg(r, (e1 >> 31) != 0);
    }
    G::madd(acc, r);
    pos += paired ? 2u : 1u;
  }
  const bool head_open = bstart < seg;
  const bool tail_open = bend > end;
  if (!head_open && !tail_open) save_acc<G>(buckets + (size_t)g * G::ACC_WORDS, acc);
  else if (head_open) save_acc<G>(heads + sid * G::ACC_WORDS, acc);
  else save_acc<G>(tails + sid * G::ACC_WORDS, acc);
}

// Adds the value of bucket g into `sum`.  A bucket wholly inside one accumulate segment was written
// to `buckets`; one that straddles segments is the sum of tails[ts] and heads[ts+1..te]; an empty
// bucket contributes nothing.  (This stitching used to be a separate pass; fusing it here costs no
// extra additions and removes a launch plus one write+read of every bucket.)
// ---- stitching of buckets that straddle accumulate segments -------------------------------------
// Segment (= accumulate thread) t holds in heads[t] the partial of the bucket that was already open
// when the segment started.  A bucket spanning segments ts..te is tails[ts] + heads[ts+1..te].  For
// ordinary inputs that is 1-3 partials, but a bucket can span thousands of segments (all scalars
// equal, benchmark/msm_timings.ts:45-63; a narrow top window).  Two levels of tile sums keep the
// serial walk short: tile1[j] = sum heads[32j .. 32j+31], tile2[j] = sum heads[1024j .. 1024j+1023],
// each defined only when all of its segments lie inside ONE bucket's (ts, te] range.
static constexpr uint32_t STITCH_FAN = 32;

// bucket of window w containing sorted entry e: the last g in [w*B, (w+1)*B) with offsets[g] <= e
NMSM_HD uint32_t bucket_of_entry(const uint32_t* offsets, const MsmPlan& plan, uint32_t w, uint32_t e) {
  uint32_t lo = w * (uint32_t)plan.B, hi = lo + (uint32_t)plan.B;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (offsets[mid] <= e) lo = mid; else hi = mid;
  }
  return lo;
}
// Do the segments with global ids [t0, t0 + span) all hold a head partial of one and the same bucket?  (t0 is a
// multiple of span and span divides SEG_ALIGN, so the run lies inside one window.)
NMSM_HD bool tile_is_uniform(const uint32_t* offsets, const MsmPlan& plan, uint64_t t0, uint32_t span) {
  const uint32_t w = (uint32_t)(t0 / plan.TPW), tl = (uint32_t)(t0 % plan.TPW);
  if (w >= (uint32_t)plan.W) return false;
  const uint32_t base = offsets[w * (uint32_t)plan.B], T = offsets[(w + 1) * (uint32_t)plan.B];
  const uint64_t e0 = (uint64_t)base + (uint64_t)tl * (uint32_t)plan.L, e_last = e0 + (uint64_t)(span - 1) * (uint32_t)plan.L;
  if (e_last >= T) return false;
  const uint32_t g = bucket_of_entry(offsets, plan, w, (uint32_t)e0);
  return offsets[g] < e0 && offsets[g + 1] > e_last;
}
// serial statement of one tile sum (the kernel uses a warp-shuffle tree over the 32 inputs)
template <class Cv>
NMSM_HD void stitch_tile_serial(uint32_t j, uint32_t span, const uint32_t* offsets, const MsmPlan& plan,
                                const uint32_t* in, uint32_t* out) {
  using G = typename Cv::G;
  if (!tile_is_uniform(offsets, plan, (uint64_t)j * span, span)) return;
  typename G::Acc acc = G::identity();
  for (uint32_t k = 0; k < STITCH_FAN; k++) nl_add<G>(acc, load_acc<G>(in + ((size_t)j * STITCH_FAN + k) * G::ACC_WORDS));
  save_acc<G>(out + (size_t)j * G::ACC_WORDS, acc);
}

// The value of bucket g: a bucket wholly inside one accumulate segment was written to `buckets`; one that
// straddles segments ts..te is tails[ts] + heads[ts+1..te], with aligned runs of 32 / 1024 heads replaced by
// their tile sums; an empty bucket contributes nothing.
// Thread (w, k): chunk of K buckets of window w ->
//   sums[id]  = sum_{b in chunk} B_b
//   wsums[id] = sum_{b in chunk} (b - kK + 1) * B_b          (running-sum trick, curve.ts:897-900)
// so that  sum_b (b+1) B_b = sum_k wsums_k + K * sum_k k * sums_k  (second level: reduce2).
//
// The walk is written as ONE loop with ONE addition per iteration — either `sum += next partial of the current
// bucket` or, when the bucket is exhausted, `wsum += sum` — selected by pointers.  A point addition occupies the
// multiply pipe for the whole warp whatever the number of active lanes, so the lanes of a warp must reach the same
// call site in the same iteration: with one call site the warp executes max-over-lanes of (partials + K)
// additions instead of one per distinct branch taken by any lane.
template <class Cv, class Ops>
NMSM_HD void reduce1_body(uint32_t id, const uint32_t* offsets, const uint32_t* buckets, const uint32_t* heads,
                          const uint32_t* tails, const uint32_t* tile1, const uint32_t* tile2, const MsmPlan& plan,
                          uint32_t* sums, uint32_t* wsums) {
  using G = typename Cv::G;
  using Acc = typename G::Acc;
  const uint32_t w = id / plan.chunks, k = id % plan.chunks;
  const uint32_t g0 = w * plan.B + k * plan.K;
  const uint32_t wbase = offsets[w * (uint32_t)plan.B];  // first sorted entry of this window
  const uint32_t sid0 = w * plan.TPW;                    // its first segment id
  constexpr uint32_t F1 = STITCH_FAN, F2 = STITCH_FAN * STITCH_FAN;
  Acc acc[2] = {G::identity(), G::identity()};  // [0] = sum, [1] = wsum
  Acc part;
  int b = plan.K - 1;
  bool open = false;
  uint32_t g = 0, t = 1, ts = 0, te = 0;  // t > te: no partial left in the current bucket
  for (;;) {
    if (!open) {
      if (b < 0) break;
      g = g0 + (uint32_t)b;
      const uint32_t b0 = offsets[g], b1 = offsets[g + 1];
      ts = 0;
      te = 0;
      t = 1;
      if (b0 != b1) {
        ts = sid0 + (b0 - wbase) / plan.L;
        te = sid0 + (b1 - 1 - wbase) / plan.L;
        t = ts;
      }
      open = true;
    }
    const bool fold = t > te;  // bucket exhausted (or empty): wsum += sum and move to the next bucket
    if (!fold) {
      const uint32_t* src;
      uint32_t step = 1;
      if (t == ts) {
        src = (ts == te) ? buckets + (size_t)g * G::ACC_WORDS : tails + (size_t)ts * G::ACC_WORDS;
      } else if ((t % F2) == 0 && te - t >= F2 - 1) {
        src = tile2 + (size_t)(t / F2) * G::ACC_WORDS;
        step = F2;
      } else if ((t % F1) == 0 && te - t >= F1 - 1) {
        src = tile1 + (size_t)(t / F1) * G::ACC_WORDS;
        step = F1;
      } else {
        src = heads + (size_t)t * G::ACC_WORDS;
      }
      part = load_acc<G>(src);
      t += step;
    }
    Ops::add(acc[fold ? 1 : 0], fold ? acc[0] : part);
    if (fold) {
      open = false;
      b--;
    }
  }
  save_acc<G>(sums + (size_t)id * G::ACC_WORDS, acc[0]);
  save_acc<G>(wsums + (size_t)id * G::ACC_WORDS, acc[1]);
}

// ---- dense buckets (multi-GPU bucket exchange, SURVEY §8e) ---------------------------------------------------
// bucket_finalize_body: after it, buckets[g] holds the complete value of bucket g for every g of the window range —
// straddling buckets are stitched from tails / heads / tile sums, empty buckets become the identity — so a window's
// B accumulators form one contiguous array that can be sent to the GPU that owns the window.
template <class Cv>
NMSM_HD void bucket_finalize_body(uint32_t g, const uint32_t* offsets, uint32_t* buckets, const uint32_t* heads,
                                  const uint32_t* tails, const uint32_t* tile1, const uint32_t* tile2, const MsmPlan& plan) {
  using G = typename Cv::G;
  using Acc = typename G::Acc;
  constexpr uint32_t F1 = STITCH_FAN, F2 = STITCH_FAN * STITCH_FAN;
  const uint32_t w = g / (uint32_t)plan.B;
  const uint32_t wbase = offsets[w * (uint32_t)plan.B], sid0 = w * plan.TPW;
  const uint32_t b0 = offsets[g], b1 = offsets[g + 1];
  if (b0 == b1) {
    save_acc<G>(buckets + (size_t)g * G::ACC_WORDS, G::identity());
    return;
  }
  const uint32_t ts = sid0 + (b0 - wbase) / plan.L, te = sid0 + (b1 - 1 - wbase) / plan.L;
  if (ts == te) return;  // wholly inside one segment: k_accumulate wrote it
  Acc acc = load_acc<G>(tails + (size_t)ts * G::ACC_WORDS);
  for (uint32_t t = ts + 1; t <= te;) {
    const uint32_t* src;
    uint32_t step = 1;
    if ((t % F2) == 0 && te - t >= F2 - 1) {
      src = tile2 + (size_t)(t / F2) * G::ACC_WORDS;
      step = F2;
    } else if ((t % F1) == 0 && te - t >= F1 - 1) {
      src = tile1 + (size_t)(t / F1) * G::ACC_WORDS;
      step = F1;
    } else {
      src = heads + (size_t)t * G::ACC_WORDS;
    }
    // G::add inline, not nl_add: ptxas 12.9 clones the out-of-line nl_add into this kernel with its operand
    // addresses in uniform registers and reads one of them uninitialised (compute-sanitizer: invalid __local__ read)
    const Acc part = load_acc<G>(src);
    G::add(acc, part);
    t += step;
  }
  save_acc<G>(buckets + (size_t)g * G::ACC_WORDS, acc);
}

// bucket b of an owned window: own partial += the partials received from the `npeers` other GPUs (peer arrays are
// `stride_words` apart).  The EC fold of the "allreduce of bucket accumulators": point addition is not an NCCL
// reduction operator, so the exchange is send/recv + this kernel.
template <class Cv, class Ops = InlineOps<typename Cv::G>>
NMSM_HD void bucket_fold_body(uint32_t b, uint32_t* own, const uint32_t* recv, int npeers, size_t stride_words) {
  using G = typename Cv::G;
  typename G::Acc acc = load_acc<G>(own + (size_t)b * G::ACC_WORDS);
  for (int r = 0; r < npeers; r++) {
    const typename G::Acc part = load_acc<G>(recv + (size_t)r * stride_words + (size_t)b * G::ACC_WORDS);
    Ops::add(acc, part);
  }
  save_acc<G>(own + (size_t)b * G::ACC_WORDS, acc);
}
// Same with the peers' partials read in place from THEIR memory (pointers into the peers' bucket arrays, mapped over
// NVLink): the exchange is the loads of the fold itself, no copy is made.  peers[r] = window base in rank r's array.
template <class Cv, class Ops = InlineOps<typename Cv::G>>
NMSM_HD void bucket_fold_peers_body(uint32_t b, uint32_t* own, const uint32_t* const* peers, int world, int rank) {
  using G = typename Cv::G;
  typename G::Acc acc = load_acc<G>(own + (size_t)b * G::ACC_WORDS);
  for (int r = 0; r < world; r++) {
    if (r == rank) continue;
    const typename G::Acc part = load_acc<G>(peers[r] + (size_t)b * G::ACC_WORDS);
    Ops::add(acc, part);
  }
  save_acc<G>(own + (size_t)b * G::ACC_WORDS, acc);
}

// reduce1 over dense buckets: chunk running sums without any stitching (curve.ts:897-900)
template <class Cv, class Ops = InlineOps<typename Cv::G>>
NMSM_HD void reduce1_dense_body(uint32_t id, const uint32_t* buckets, const MsmPlan& plan, uint32_t* sums, uint32_t* wsums) {
  using G = typename Cv::G;
  const uint32_t w = id / plan.chunks, k = id % plan.chunks;
  const uint32_t g0 = w * plan.B + k * plan.K;
  typename G::Acc sum = G::identity(), wsum = G::identity();
  for (int b = plan.K - 1; b >= 0; b--) {
    const typename G::Acc part = load_acc<G>(buckets + (size_t)(g0 + (uint32_t)b) * G::ACC_WORDS);
    Ops::add(sum, part);
    Ops::add(wsum, sum);
  }
  save_acc<G>(sums + (size_t)id * G::ACC_WORDS, sum);
  save_acc<G>(wsums + (size_t)id * G::ACC_WORDS, wsum);
}

// Serial statement of the second level for one window (what k_reduce2 computes cooperatively):
//   window_out[w] = sum_k wsums_k + K * sum_k k * sums_k
template <class Cv>
NMSM_HD void reduce2_serial(uint32_t w, const uint32_t* sums, const uint32_t* wsums, const MsmPlan& plan,
                            uint32_t* window_out) {
  using G = typename Cv::G;
  typename G::Acc run = G::identity(), ksum = G::identity(), wtot = G::identity();
  for (int k = plan.chunks - 1; k >= 0; k--) {
    const size_t id = (size_t)w * plan.chunks + k;
    nl_add<G>(wtot, load_acc<G>(wsums + id * G::ACC_WORDS));
    if (k >= 1) {
      nl_add<G>(run, load_acc<G>(sums + id * G::ACC_WORDS));
      nl_add<G>(ksum, run);  // after the loop: sum_k k * sums_k
    }
  }
  for (int j = 1; j < plan.K; j <<= 1) nl_dbl<G>(ksum);  // * K (power of two)
  nl_add<G>(wtot, ksum);
  save_acc<G>(window_out + (size_t)w * G::ACC_WORDS, wtot);
}

// Horner over the window sums (curve.ts:901-902).  AFFINE_OUT: canonical affine + infinity flag,
// else the raw accumulator (multi-GPU partial, folded later by fold_body).
template <class Cv, bool AFFINE_OUT>
NMSM_HD void final_body(const uint32_t* window_out, const MsmPlan& plan, uint32_t* out, uint32_t* out_inf) {
  using G = typename Cv::G;
  typename G::Acc acc = G::identity();
  for (int w = plan.W - 1; w >= 0; w--) {
    if (w != plan.W - 1)
      for (int j = 0; j < plan.c; j++) nl_dbl<G>(acc);
    nl_add<G>(acc, load_acc<G>(window_out + (size_t)w * G::ACC_WORDS));
  }
  if (AFFINE_OUT) {
    uint32_t xy[G::IN_WORDS];
    uint32_t inf;
    nl_to_affine<G>(acc, xy, &inf);
    for (int k = 0; k < G::IN_WORDS; k++) out[k] = xy[k];
    *out_inf = inf;
  } else {
    save_acc<G>(out, acc);
  }
}

// One step of the Horner evaluation over window groups (curve.ts:901-902 walks the windows MSB -> LSB the same way):
//   hacc = first ? sum_{w in [w_lo, w_hi)} 2^(c (w - w_lo)) S_w : 2^(c (w_hi - w_lo)) * hacc + (that sum)
// Groups arrive top windows first, so the doubling chains of the upper windows run while the lower windows are still
// being accumulated and reduced (engine.cuh submit_msm); after the last group hacc is the MSM result.
// shift != 0 (multi-GPU window owners): afterwards hacc *= 2^(c * w_lo), the group's absolute weight.
template <class Cv>
NMSM_HD void horner_step_body(const uint32_t* window_out, const MsmPlan& plan, int w_lo, int w_hi, bool first, bool shift,
                              uint32_t* hacc) {
  using G = typename Cv::G;
  typename G::Acc acc = first ? G::identity() : load_acc<G>(hacc);
  for (int w = w_hi - 1; w >= w_lo; w--) {
    if (!(first && w == w_hi - 1))
      for (int j = 0; j < plan.c; j++) nl_dbl<G>(acc);
    nl_add<G>(acc, load_acc<G>(window_out + (size_t)w * G::ACC_WORDS));
  }
  if (shift)
    for (int j = 0; j < plan.c * w_lo; j++) nl_dbl<G>(acc);
  save_acc<G>(hacc, acc);
}

// Fold `count` raw accumulators (e.g. one per GPU) and emit canonical affine.
template <class Cv>
NMSM_HD void fold_body(const uint32_t* accs, int count, uint32_t* out, uint32_t* out_inf) {
  using G = typename Cv::G;
  typename G::Acc acc = G::identity();
  for (int i = 0; i < count; i++) nl_add<G>(acc, load_acc<G>(accs + (size_t)i * G::ACC_WORDS));
  uint32_t xy[G::IN_WORDS];
  uint32_t inf;
  nl_to_affine<G>(acc, xy, &inf);
  for (int k = 0; k < G::IN_WORDS; k++) out[k] = xy[k];
  *out_inf = inf;
}

// k_i * P_i (Point.multiply / multiplyUnsafe, weierstrass.ts:900-928, edwards.ts:555-577): fixed 4-bit signed
// windows over a per-thread table {1..8} * P (the shape of the reference's uncached constant-time kernel,
// curve.ts:707-729, without its blinding), canonical affine out.  Public-input / variable-time like multiplyUnsafe;
// the value equals multiply()'s.  Why windows and not NAF: a point addition costs the whole warp its multiply-pipe
// time whenever ANY lane needs it, so sparse per-lane digit patterns buy nothing under SIMT, while a window does one
// table addition per 4 doublings for every lane at once.  On the cofactor-1 GLV curves (secp256k1, bn254 G1;
// weierstrass.ts:843-861 is the reference's use of the same endomorphism for secp256k1) k = k1 + k2 * lambda halves
// the doublings: the second table is phi of the first, (beta * X, Y, ZZ, ZZZ).  BLS12-381 G1 takes the plain route:
// multiply() is what subgroup checks and cofactor clearing run on points OUTSIDE the prime-order subgroup, where
// phi(P) != lambda * P.
static constexpr int MUL_WBITS = 4;
static constexpr int MUL_TABLE = 1 << (MUL_WBITS - 1);  // |digit| <= 8

// digit w of the signed MUL_WBITS-bit recoding of m (nwords 32-bit words); `carry` threads through ascending w
NMSM_HD int mul_window_digit(const uint32_t* m, int nwords, int w, uint32_t& carry) {
  uint32_t v = scalar_bits(m, w * MUL_WBITS, MUL_WBITS, nwords) + carry;
  carry = 0;
  if (v > (uint32_t)MUL_TABLE) {
    carry = 1;
    return (int)v - (1 << MUL_WBITS);
  }
  return (int)v;
}

// s * P as an un-normalised accumulator (the core of mul_body / torsion_body); s < n, scalar_words<Fn>() words
// Ops: SerialOps (one thread per item) or msm.cuh QuadOps (one item per quad of lanes, k_mul_batch for small batches).
template <class Cv, class Ops = SerialOps<typename Cv::G>>
NMSM_HD typename Cv::G::Acc scalar_mul_acc(const typename Cv::G::Affine& P, const uint32_t* s) {
  using G = typename Cv::G;
  using Acc = typename G::Acc;
  // table[d - 1] = d * P, d = 1..8
  Acc table[MUL_TABLE];
  table[0] = G::from_affine(P);
  table[1] = table[0];
  Ops::dbl(table[1]);
  for (int d = 2; d < MUL_TABLE; d++) {
    table[d] = table[d - 1];
    Ops::madd(table[d], P);
  }
  Acc acc = G::identity();
  if constexpr (Cv::GLV && Cv::COFACTOR_ONE) {  // multiply() must be right for every on-curve point (subgroup checks, cofactor clearing)
    constexpr int MW = Cv::GLV_KIND == 1 ? 4 : 5;       // words of a half-scalar magnitude
    constexpr int HB = Cv::Glv::BITS;                    // |k1|, |k2| < 2^HB
    constexpr int NW = (HB + 1 + MUL_WBITS - 1) / MUL_WBITS;
    uint32_t m1[MW], m2[MW];
    bool neg1, neg2;
    if constexpr (Cv::GLV_KIND == 1) glv_split<typename Cv::Glv>(s, m1, neg1, m2, neg2);
    else glv_split_lattice<typename Cv::Glv>(s, m1, neg1, m2, neg2);
    typename G::Field beta;
    for (int k = 0; k < G::Field::LIMBS; k++) beta.v[k] = Cv::Glv::BETA_MONT(k);
    // digits, least significant first (the carries run upwards), consumed from the top
    signed char d1[NW], d2[NW];
    uint32_t c1 = 0, c2 = 0;
    for (int w = 0; w < NW; w++) {
      d1[w] = (signed char)mul_window_digit(m1, MW, w, c1);
      d2[w] = (signed char)mul_window_digit(m2, MW, w, c2);
    }
    for (int w = NW - 1; w >= 0; w--) {
      if (w != NW - 1)
        for (int j = 0; j < MUL_WBITS; j++) Ops::dbl(acc);
      if (d1[w] != 0) {
        const int a = d1[w] < 0 ? -d1[w] : d1[w];
        Acc t = table[a - 1];
        if ((d1[w] < 0) != neg1) t = G::neg(t);
        Ops::add(acc, t);
      }
      if (d2[w] != 0) {
        const int a = d2[w] < 0 ? -d2[w] : d2[w];
        Acc t = table[a - 1];
        t.X = t.X * beta;  // phi on XYZZ coordinates: x = X / ZZ
        if ((d2[w] < 0) != neg2) t = G::neg(t);
        Ops::add(acc, t);
      }
    }
  } else {
    constexpr int NW = (Cv::Fn::BITS + 1 + MUL_WBITS - 1) / MUL_WBITS;
    signed char dg[NW];
    uint32_t c = 0;
    for (int w = 0; w < NW; w++) dg[w] = (signed char)mul_window_digit(s, scalar_words<typename Cv::Fn>(), w, c);
    for (int w = NW - 1; w >= 0; w--) {
      if (w != NW - 1)
        for (int j = 0; j < MUL_WBITS; j++) Ops::dbl(acc);
      if (dg[w] != 0) {
        const int a = dg[w] < 0 ? -dg[w] : dg[w];
        Acc t = table[a - 1];
        if (dg[w] < 0) t = G::neg(t);
        Ops::add(acc, t);
      }
    }
  }
  return acc;
}

// Validation + scalar multiplication of item i; false (and the index recorded) when the point or scalar is rejected.
template <class Cv, class Ops = SerialOps<typename Cv::G>>
NMSM_HD bool mul_acc_body(uint32_t i, const uint32_t* pts, const uint32_t* scalars, int allow_zero,
                          typename Cv::G::Acc& acc, unsigned int* err) {
  using G = typename Cv::G;
  uint32_t in[G::IN_WORDS];
  load_words<G::IN_WORDS>(in, pts + (size_t)i * G::IN_WORDS);
  uint32_t s[SCALAR_WORDS];
  load_words<SCALAR_WORDS>(s, scalars + (size_t)i * SCALAR_WORDS);
  bool bad_pt = !G::input_in_range(in);
  bool bad_sc = !scalar_in_range<typename Cv::Fn>(s);
  uint32_t nz = 0;
  for (int k = 0; k < SCALAR_WORDS; k++) nz |= s[k];
  if (!allow_zero && nz == 0) bad_sc = true;
  if (bad_pt) atomic_min_u32(&err[0], i);
  if (bad_sc) atomic_min_u32(&err[1], i);
  acc = G::identity();
  if (bad_pt || bad_sc) return false;
  acc = scalar_mul_acc<Cv, Ops>(G::prepare(in), s);
  return true;
}

// serial statement (tests/hostemu): one inversion per item; the kernel shares ONE inversion per warp (msm.cuh k_mul_batch)
template <class Cv>
NMSM_HD void mul_body(uint32_t i, const uint32_t* pts, const uint32_t* scalars, int allow_zero, uint32_t* out_xy,
                      uint32_t* out_inf, unsigned int* err) {
  using G = typename Cv::G;
  typename G::Acc acc;
  if (!mul_acc_body<Cv>(i, pts, scalars, allow_zero, acc, err)) return;
  uint32_t xy[G::IN_WORDS];
  uint32_t inf;
  nl_to_affine<G>(acc, xy, &inf);
  store_words<G::IN_WORDS>(out_xy + (size_t)i * G::IN_WORDS, xy);
  out_inf[i] = inf;
}

// isTorsionFree (weierstrass.ts:971-975, edwards.ts:584-586; the curve files' endomorphism shortcuts
// bls12-381.ts:567-577,599-601 and bn254.ts:241 decide the same predicate): n * P == O, evaluated as
// (n - 1) * P + P.  Every lane walks the same digits of n - 1, so the warp never diverges.
template <class Cv>
NMSM_HD void torsion_body(uint32_t i, const uint32_t* pts, uint8_t* out_ok, unsigned int* err) {
  using G = typename Cv::G;
  uint32_t in[G::IN_WORDS];
  load_words<G::IN_WORDS>(in, pts + (size_t)i * G::IN_WORDS);
  if (!G::input_in_range(in)) {
    atomic_min_u32(&err[0], i);
    return;
  }
  uint32_t s[SCALAR_WORDS];
  for (int k = 0; k < SCALAR_WORDS; k++) s[k] = Cv::Fn::ORDER(k);
  s[0] -= 1u;  // the group orders are odd
  const typename G::Affine P = G::prepare(in);
  typename G::Acc acc = scalar_mul_acc<Cv>(P, s);
  nl_madd<G>(acc, P);
  out_ok[i] = G::is_identity(acc) ? 1 : 0;
}

}  // namespace nmsm
