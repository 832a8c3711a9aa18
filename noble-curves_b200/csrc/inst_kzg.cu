// EIP-4844 KZG proof verification (SURVEY §8 row f15, kzg.cuh): the kernels and the two C-ABI implementations.
//   k_kzg_roots      (once per context) one thread per root: the bit-reversed domain into Context::kzg_roots
//   k_kzg_setup      (every call) one thread: decode and subgroup-check [tau] G2
//   k_kzg_challenge  (blobs only) one thread per blob: z = compute_challenge(blob, C)
//   k_kzg_eval       (blobs only) one block per blob: y = f(z), and whether every element is < r
//   k_kzg_prepare    one thread per check: validation and the pairs (Q, -G2), (pi, [tau] G2)
//   k_bls_miller, k_bls_final  the BLS pairing checks of inst_bls381_pairing.cu, two pairs per check
// Blobs go up and are evaluated KZG_CHUNK at a time (128 MiB); only z, y and the verdict of each (65 bytes) outlive
// their chunk, so device memory stays bounded at any n.  The proof stage then runs once over all n.
// The prover (SURVEY §8 row f16), the same chunking:
//   k_kzg_setup_points, k_prepare, k_kzg_table_base, k_table_level  (setup_create) the setup table of a KzgSetup
//   k_kzg_commit_check    (blob proofs) one thread per item: validate_kzg_g1 of the commitment
//   k_kzg_quotient        (proofs) one block per blob, after k_kzg_eval: the quotient in place of the blob
//   k_kzg_lincomb, k_kzg_lincomb_finish  the comb over the setup table: the commitment or the proof
#include "kzg.cuh"
#include "pairing_driver.cuh"

namespace nmsm {

__global__ void __launch_bounds__(128) k_kzg_roots(uint32_t* __restrict__ roots) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= KZG_N) return;
  store_words<8>(roots + 8 * (size_t)i, kzg_root(i).v);
}

__global__ void k_kzg_setup(const uint8_t* __restrict__ g2_96, uint32_t* __restrict__ xy, uint32_t* __restrict__ ok) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *ok = kzg_setup_body(g2_96, xy) ? 1u : 0u;
}

// Blocks of 32 threads spread the latency-bound hashes over as many SMs as there are warps.
__global__ void __launch_bounds__(32)
k_kzg_challenge(uint32_t n, const uint8_t* __restrict__ blobs, const uint8_t* __restrict__ commitments48,
                uint8_t* __restrict__ zs32) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) kzg_challenge_body(i, blobs, commitments48, zs32);
}

// block b = blob b: each lane sums its 16 fractions (kzg_eval_lane), a shuffle tree and the 8 warp partials in shared
// memory give the blob's sum, and thread 0 does the one inversion.  __syncthreads_or is the range vote.
__global__ void __launch_bounds__(KZG_EVAL_THREADS)
k_kzg_eval(const uint8_t* __restrict__ blobs, const uint8_t* __restrict__ zs32, const uint32_t* __restrict__ roots,
           uint8_t* __restrict__ ys32, uint8_t* __restrict__ item_ok) {
  __shared__ KzgFrac part[KZG_EVAL_THREADS / 32];
  __shared__ int s_hit;
  const uint32_t b = blockIdx.x, t = threadIdx.x, lane = t & 31;
  const uint8_t* blob = blobs + (size_t)b * KZG_BLOB_BYTES;
  if (t == 0) s_hit = -1;
  __syncthreads();
  uint32_t zw[8];
  kzg_load_fr(zw, zs32 + (size_t)b * 32);
  const KzgFr z = KzgFr::from_canonical(zw);
  bool bad = false;
  int hit = -1;
  KzgFrac s = kzg_eval_lane(t, blob, z, roots, bad, hit);
  if (hit >= 0) s_hit = hit;  // the roots are distinct: at most one lane writes
  for (uint32_t d = 16; d; d >>= 1) {
    const int src = lane + d < 32 ? lane + d : lane;
    s = kzg_frac_add(s, KzgFrac{shfl_field(s.num, src), shfl_field(s.den, src)});
  }
  if (lane == 0) part[t >> 5] = s;
  bad = __syncthreads_or(bad);
  if (t == 0) {
    for (int w = 1; w < KZG_EVAL_THREADS / 32; w++) s = kzg_frac_add(s, part[w]);
    kzg_eval_finish(blob, z, s, s_hit, bad, ys32 + (size_t)b * 32, item_ok + b);
  }
}

// Lanes past n and rejected checks feed 1 to the warp-shared inversion, so one bad item cannot touch its neighbours.
__global__ void __launch_bounds__(PAIRING_BLOCK)
k_kzg_prepare(uint32_t n, const uint8_t* __restrict__ commitments48, const uint8_t* __restrict__ zs32,
              const uint8_t* __restrict__ ys32, const uint8_t* __restrict__ proofs48, const uint8_t* __restrict__ vhs32,
              const uint8_t* __restrict__ item_ok, const uint32_t* __restrict__ setup_xy, uint32_t* __restrict__ g1,
              uint32_t* __restrict__ g2, uint8_t* __restrict__ pre_ok) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  KzgG::Acc q = KzgG::identity();
  uint32_t pi[24];
  const bool ok = i < n && kzg_prepare_body(i, commitments48, zs32, ys32, proofs48, vhs32, item_ok, q, pi);
  const BlsF zi = warp_batch_inverse(ok ? KzgG::inv_target(q) : BlsF::one());
  if (i < n) kzg_store_pairs(i, ok, q, zi, pi, setup_xy, g1, g2, pre_ok);
}

// ---- the prover -------------------------------------------------------------------------------------------------------
// one thread per setup point: decode and G1 check into bit-reversed position; err[0] = the smallest bad index
__global__ void __launch_bounds__(128)
k_kzg_setup_points(const uint8_t* __restrict__ g1_48, uint32_t* __restrict__ xy, unsigned int* __restrict__ err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < KZG_N && !kzg_setup_point_body(i, g1_48, xy)) atomic_min_u32(&err[0], i);
}

// level 0 of the setup table, one thread per (point, d); the higher levels are k_table_level's
__global__ void __launch_bounds__(128) k_kzg_table_base(const uint32_t* __restrict__ aff, uint32_t* __restrict__ tbl) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < KZG_N << (KZG_COMB_BITS - 1)) kzg_table_base_body(t, aff, tbl);
}

// validate_kzg_g1 of each commitment of compute_blob_kzg_proof
__global__ void __launch_bounds__(128)
k_kzg_commit_check(uint32_t n, const uint8_t* __restrict__ commitments48, uint8_t* __restrict__ ok) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t xy[24];
  if (i < n) ok[i] = kzg_decode_g1(commitments48 + 48 * (size_t)i, xy) != 0;
}

// block b = blob b, after k_kzg_eval (y and the range vote): the quotient in place of the blob.  Each lane's Montgomery
// chain (kzg_quotient_fwd) ends in one warp-shared inversion; when z is on the domain (a lane hit w_m), the lanes'
// sums of q_i w_i meet in a shuffle tree and shared memory and thread 0 writes q_m.  A blob that failed its range vote
// or whose z is >= r is left alone with item_ok 0.
__global__ void __launch_bounds__(KZG_EVAL_THREADS)
k_kzg_quotient(uint8_t* __restrict__ blobs, const uint8_t* __restrict__ zs32, const uint8_t* __restrict__ ys32,
               const uint32_t* __restrict__ roots, uint8_t* __restrict__ item_ok) {
  __shared__ KzgFr part[KZG_EVAL_THREADS / 32];
  __shared__ int s_hit;
  const uint32_t b = blockIdx.x, t = threadIdx.x, lane = t & 31;
  uint8_t* blob = blobs + (size_t)b * KZG_BLOB_BYTES;
  KzgFr z, y;
  if (!kzg_quotient_start(b, zs32, ys32, item_ok, z, y)) {  // the same verdict in every thread
    __syncthreads();  // every thread has read item_ok[b]
    if (t == 0) item_ok[b] = 0;
    return;
  }
  if (t == 0) s_hit = -1;
  __syncthreads();
  int hit = -1;
  const KzgFr pre = kzg_quotient_fwd(t, blob, z, y, roots, hit);
  if (hit >= 0) s_hit = hit;  // the roots are distinct: at most one lane writes
  const KzgFr ri = warp_batch_inverse(pre);
  __syncthreads();
  const int m = s_hit;
  KzgFr s = kzg_quotient_back(t, blob, z, roots, ri, m >= 0);
  if (m < 0) return;  // the same in every thread
  for (uint32_t d = 16; d; d >>= 1) s = s + shfl_field(s, lane + d < 32 ? lane + d : lane);
  if (lane == 0) part[t >> 5] = s;
  __syncthreads();
  if (t == 0) {
    for (int w = 1; w < KZG_EVAL_THREADS / 32; w++) s = s + part[w];
    kzg_quotient_in_domain(blob, m, z, s);
  }
}

// S lanes per blob (a power of two), 128-thread blocks: lane t of blob b = g / S sums s_p P_p over its points
// (kzg_lincomb_lane).  The lanes' accumulators are added by a shuffle tree within the warp and, for S >= 64, across
// the block's warps in shared memory; one partial per blob and block goes to parts[b * P + t / 128], P = max(1, S / 128).
// A scalar >= r clears item_ok[b].
__global__ void __launch_bounds__(128)
k_kzg_lincomb(uint32_t cnt, uint32_t S, const uint8_t* __restrict__ scalars_be, const uint32_t* __restrict__ tbl,
              uint32_t* __restrict__ parts, uint8_t* __restrict__ item_ok) {
  __shared__ KzgG::Acc wsum[4];
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x, b = g / S, t = g % S, lane = threadIdx.x & 31,
                 warp = threadIdx.x >> 5;
  KzgG::Acc acc = KzgG::identity();
  bool bad = false;
  if (b < cnt) kzg_lincomb_lane(t, S, scalars_be + (size_t)b * KZG_BLOB_BYTES, tbl, acc, bad);
  if (bad) item_ok[b] = 0;
  const uint32_t W = S < 32 ? S : 32;
  for (uint32_t d = W / 2; d; d >>= 1) {  // lane k of a group of W takes lane k + d's sum, k < d
    const KzgG::Acc o = shfl_field(acc, lane + d < 32 ? lane + d : lane);
    if ((lane & (W - 1)) < d) nl_add<KzgG>(acc, o);
  }
  if (S >= 64) {  // uniform
    const uint32_t wpb = (S < 128 ? S : 128) / 32;  // warps per blob in this block
    if (lane == 0) wsum[warp] = acc;
    __syncthreads();
    if (lane != 0 || warp % wpb != 0) return;
    for (uint32_t w = 1; w < wpb; w++) nl_add<KzgG>(acc, wsum[warp + w]);
  } else if (lane % W != 0) {
    return;
  }
  if (b < cnt) save_acc<KzgG>(parts + ((size_t)b * (S > 128 ? S / 128 : 1) + t / 128) * KzgG::ACC_WORDS, acc);
}

// one thread per blob: the sum of its P partials, one warp-shared inversion, the compressed point
__global__ void __launch_bounds__(128)
k_kzg_lincomb_finish(uint32_t cnt, uint32_t P, const uint32_t* __restrict__ parts, uint8_t* __restrict__ out48) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  const KzgG::Acc acc = b < cnt ? kzg_sum_parts(parts + (size_t)b * P * KzgG::ACC_WORDS, P) : KzgG::identity();
  const KzgG::Field zi = warp_batch_inverse(KzgG::inv_target(acc));  // whole warp, also the idle lanes
  if (b < cnt) kzg_store_g1(acc, zi, out48 + 48 * (size_t)b);
}

namespace {
constexpr uint64_t KZG_CHUNK = 1024;  // blobs per upload and evaluation (128 MiB)

// the bit-reversed domain in Montgomery form (4096 x 32 B), built by the first blob call after nmsm_init
int ensure_kzg_roots(Context& X, cudaStream_t st) {
  if (X.kzg_roots) return NMSM_OK;
  CK(cudaMalloc((void**)&X.kzg_roots, 32 * KZG_N));
  k_kzg_roots<<<KZG_N / 128, 128, 0, st>>>(X.kzg_roots);
  CK(cudaGetLastError());
  return NMSM_OK;
}

// Both entry points after the argument checks of capi.cu (0 < n < 2^30, pointers non-null).  blobs == nullptr: the
// proof call, z and y from the caller (vhs32 optional); else the blob call, z and y from the blobs.
int kzg_verify_impl(const uint8_t* blobs, const uint8_t* commitments48, const uint8_t* zs32, const uint8_t* ys32,
                    const uint8_t* proofs48, const uint8_t* vhs32, uint64_t n, const uint8_t* setup_g2_96,
                    uint8_t* out_ok) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  cudaStream_t st = C.stream;
  if (X.profiling) memset(X.last_ms, 0, sizeof(X.last_ms));
  const int s0 = blobs ? 2 : 0;  // timing slot of k_kzg_prepare
  const uint64_t nb = blobs ? std::min(n, KZG_CHUNK) : 0;
  const uint64_t o_set = 0, o_sxy = 256, o_err = o_sxy + 256, o_c = o_err + 256, o_pi = o_c + al256(48 * n),
                 o_z = o_pi + al256(48 * n), o_y = o_z + al256(32 * n), o_vh = o_y + al256(32 * n),
                 o_iok = o_vh + (vhs32 ? al256(32 * n) : 0), o_g1 = o_iok + (blobs ? al256(n) : 0),
                 o_g2 = o_g1 + al256(192 * n), o_pre = o_g2 + al256(384 * n), o_ok = o_pre + al256(n),
                 o_w = o_ok + al256(n), o_blob = o_w + al256(pairing_workspace_bytes<BlsPairing>()),
                 bytes = o_blob + nb * KZG_BLOB_BYTES;
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  uint32_t* d_sxy = (uint32_t*)(base + o_sxy);
  unsigned int* d_err = (unsigned int*)(base + o_err);  // [0]: the setup verdict, [2..3]: k_bls_miller's errors
  uint8_t *d_c = base + o_c, *d_z = base + o_z, *d_y = base + o_y, *d_iok = blobs ? base + o_iok : nullptr;
  if (int r = h2d_any(base + o_set, setup_g2_96, 96, st)) return r;
  CK(cudaMemsetAsync(d_err, 0xff, 16, st));
  if (int r = pairing_launch(X, C, s0, [&] { k_kzg_setup<<<1, 32, 0, st>>>(base + o_set, d_sxy, d_err); })) return r;
  unsigned int setup_ok = 0;
  CK(cudaMemcpyAsync(&setup_ok, d_err, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (!setup_ok)
    return fail(NMSM_ERR_ARG, "setup_g2_96 does not decode to a point of G2 other than the identity");
  if (int r = h2d_any(d_c, commitments48, 48 * n, st)) return r;
  if (int r = h2d_any(base + o_pi, proofs48, 48 * n, st)) return r;
  if (vhs32)
    if (int r = h2d_any(base + o_vh, vhs32, 32 * n, st)) return r;
  if (blobs) {
    if (int r = ensure_kzg_roots(X, st)) return r;
    uint8_t* d_blob = base + o_blob;
    for (uint64_t c0 = 0; c0 < n; c0 += KZG_CHUNK) {
      const uint32_t cnt = (uint32_t)std::min(KZG_CHUNK, n - c0);
      // a large pageable upload is staged on other streams (h2d_any) that do not wait for this one: the previous
      // chunk's kernels must be done with the buffer first
      if (c0) CK(cudaStreamSynchronize(st));
      if (int r = h2d_any(d_blob, blobs + c0 * KZG_BLOB_BYTES, cnt * KZG_BLOB_BYTES, st)) return r;
      if (int r = pairing_launch(X, C, 0, [&] {
            k_kzg_challenge<<<cdiv(cnt, 32), 32, 0, st>>>(cnt, d_blob, d_c + 48 * c0, d_z + 32 * c0);
          }))
        return r;
      if (int r = pairing_launch(X, C, 1, [&] {
            k_kzg_eval<<<cnt, KZG_EVAL_THREADS, 0, st>>>(d_blob, d_z + 32 * c0, X.kzg_roots, d_y + 32 * c0,
                                                         d_iok + c0);
          }))
        return r;
    }
  } else {
    if (int r = h2d_any(d_z, zs32, 32 * n, st)) return r;
    if (int r = h2d_any(d_y, ys32, 32 * n, st)) return r;
  }
  uint32_t *d_g1 = (uint32_t*)(base + o_g1), *d_g2 = (uint32_t*)(base + o_g2);
  uint8_t *d_pre = base + o_pre, *d_ok = base + o_ok;
  if (int r = pairing_launch(X, C, s0, [&] {
        k_kzg_prepare<<<cdiv(n, PAIRING_BLOCK), PAIRING_BLOCK, 0, st>>>(
            (uint32_t)n, d_c, d_z, d_y, base + o_pi, vhs32 ? base + o_vh : nullptr, d_iok, d_sxy, d_g1, d_g2, d_pre);
      }))
    return r;
  if (int r = pairing_checks_run<BlsPairing>(X, C, BLS_KERNELS, n, nullptr, nullptr, d_g1, d_g2, d_pre,
                                              (uint32_t*)(base + o_w), d_ok, d_err + 2, s0 + 1))
    return r;
  unsigned int err[2];
  CK(cudaMemcpyAsync(err, d_err + 2, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (err[0] != 0xffffffffu || err[1] != 0xffffffffu)  // prepare only emits valid or identity pairs
    return fail(NMSM_ERR_CUDA, "internal error: a prepared KZG pair failed validation");
  CK(cudaMemcpy(out_ok, d_ok, n, cudaMemcpyDeviceToHost));
  return NMSM_OK;
}

// ---- the prover -------------------------------------------------------------------------------------------------------
struct KzgSetup {
  uint32_t* d_tbl;  // nullptr once nmsm_shutdown has released it
};
std::vector<KzgSetup*> g_kzg_setups;  // live handles

constexpr uint32_t KZG_TABLE_LEVELS = point_table_levels<KzgCv, KZG_COMB_BITS>();
constexpr uint64_t KZG_LEVEL_ENTRIES = (uint64_t)KZG_N << (KZG_COMB_BITS - 1);

// Lanes per blob of k_kzg_lincomb: halved from 4096 (one point per lane) while the chunk still has about 512 lanes per
// SM, the residency of its 128-thread blocks, so a few blobs spread over every SM and a full chunk walks 32 points per
// lane with a negligible reduction.
uint32_t kzg_lincomb_lanes(const Context& X, uint64_t cnt) {
  uint32_t S = KZG_N;
  while (S > 1 && cnt * (S / 2) >= 512ull * X.sm_count) S /= 2;
  return S;
}
uint64_t kzg_lincomb_parts(const Context& X, uint64_t cnt) {
  const uint32_t S = kzg_lincomb_lanes(X, cnt);
  return cnt * (S > 128 ? S / 128 : 1);
}

int kzg_find_setup(uint64_t handle, KzgSetup** out) {
  for (KzgSetup* s : g_kzg_setups)
    if ((uint64_t)(uintptr_t)s == handle) {
      if (!s->d_tbl) return fail(NMSM_ERR_ARG, "the KZG setup was released by nmsm_shutdown");
      *out = s;
      return NMSM_OK;
    }
  return fail(NMSM_ERR_ARG, "unknown KZG setup handle");
}

// the table of a setup whose points are on the device (bit-reversed prepared affine): level 0 by k_kzg_table_base,
// level j = 2^b level j-1 by k_table_level
int kzg_build_table(Context& X, Slot& C, const uint32_t* d_aff, uint32_t* tbl) {
  cudaStream_t st = C.stream;
  constexpr uint64_t LW = KZG_LEVEL_ENTRIES * KzgG::AFF_WORDS;
  if (int r = pairing_launch(X, C, 1, [&] {
        k_kzg_table_base<<<cdiv(KZG_LEVEL_ENTRIES, 128), 128, 0, st>>>(d_aff, tbl);
        for (uint32_t j = 1; j < KZG_TABLE_LEVELS; j++)
          k_table_level<KzgCv><<<cdiv(KZG_LEVEL_ENTRIES, 128), 128, 0, st>>>(tbl + (j - 1) * LW, tbl + j * LW,
                                                                            (uint32_t)KZG_LEVEL_ENTRIES, KZG_COMB_BITS);
      }))
    return r;
  CK(cudaStreamSynchronize(st));
  return NMSM_OK;
}

// The three provers after the argument checks of capi.cu (0 < n < 2^30, pointers non-null).  zs32: compute_kzg_proof
// (z from the caller, y out); commitments48: compute_blob_kzg_proof (z from the challenge); neither: the commitments.
// Each chunk of blobs is uploaded once and, for a proof, evaluated and replaced by its quotient in place.
int kzg_prove_impl(uint64_t handle, const uint8_t* blobs, const uint8_t* zs32, const uint8_t* commitments48, uint64_t n,
                   uint8_t* out48, uint8_t* out_ys32, uint8_t* out_ok) {
  KzgSetup* S = nullptr;
  if (int r = kzg_find_setup(handle, &S)) return r;
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  cudaStream_t st = C.stream;
  if (X.profiling) memset(X.last_ms, 0, sizeof(X.last_ms));
  const bool prove = zs32 || commitments48;
  const int s_eval = commitments48 ? 1 : 0, s_comb = prove ? s_eval + 2 : 0;  // timing slots
  const uint64_t nb = std::min(n, KZG_CHUNK), last = n - (n - 1) / KZG_CHUNK * KZG_CHUNK;
  const uint64_t parts = std::max(kzg_lincomb_parts(X, nb), kzg_lincomb_parts(X, last));
  const uint64_t o_c = 0, o_cok = o_c + (commitments48 ? al256(48 * n) : 0),
                 o_z = o_cok + (commitments48 ? al256(n) : 0), o_y = o_z + (prove ? al256(32 * n) : 0),
                 o_iok = o_y + (prove ? al256(32 * n) : 0), o_out = o_iok + al256(n), o_parts = o_out + al256(48 * n),
                 o_blob = o_parts + al256(parts * KzgG::ACC_WORDS * 4), bytes = o_blob + nb * KZG_BLOB_BYTES;
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  uint8_t *d_c = base + o_c, *d_cok = base + o_cok, *d_z = base + o_z, *d_y = base + o_y, *d_iok = base + o_iok,
          *d_out = base + o_out, *d_blob = base + o_blob;
  uint32_t* d_parts = (uint32_t*)(base + o_parts);
  if (commitments48) {
    if (int r = h2d_any(d_c, commitments48, 48 * n, st)) return r;
    if (int r = pairing_launch(X, C, 0,
                               [&] { k_kzg_commit_check<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, d_c, d_cok); }))
      return r;
  }
  if (zs32)
    if (int r = h2d_any(d_z, zs32, 32 * n, st)) return r;
  if (prove)
    if (int r = ensure_kzg_roots(X, st)) return r;
  for (uint64_t c0 = 0; c0 < n; c0 += KZG_CHUNK) {
    const uint32_t cnt = (uint32_t)std::min(KZG_CHUNK, n - c0);
    if (c0) CK(cudaStreamSynchronize(st));  // h2d_any may stage on other streams (kzg_verify_impl)
    if (int r = h2d_any(d_blob, blobs + c0 * KZG_BLOB_BYTES, cnt * KZG_BLOB_BYTES, st)) return r;
    if (commitments48)
      if (int r = pairing_launch(X, C, 0, [&] {
            k_kzg_challenge<<<cdiv(cnt, 32), 32, 0, st>>>(cnt, d_blob, d_c + 48 * c0, d_z + 32 * c0);
          }))
        return r;
    if (prove) {
      if (int r = pairing_launch(X, C, s_eval, [&] {
            k_kzg_eval<<<cnt, KZG_EVAL_THREADS, 0, st>>>(d_blob, d_z + 32 * c0, X.kzg_roots, d_y + 32 * c0,
                                                         d_iok + c0);
          }))
        return r;
      if (int r = pairing_launch(X, C, s_eval + 1, [&] {
            k_kzg_quotient<<<cnt, KZG_EVAL_THREADS, 0, st>>>(d_blob, d_z + 32 * c0, d_y + 32 * c0, X.kzg_roots,
                                                             d_iok + c0);
          }))
        return r;
    } else {
      CK(cudaMemsetAsync(d_iok + c0, 1, cnt, st));
    }
    const uint32_t lanes = kzg_lincomb_lanes(X, cnt);
    if (int r = pairing_launch(X, C, s_comb, [&] {
          k_kzg_lincomb<<<cdiv((uint64_t)cnt * lanes, 128), 128, 0, st>>>(cnt, lanes, d_blob, S->d_tbl, d_parts,
                                                                          d_iok + c0);
          k_kzg_lincomb_finish<<<cdiv(cnt, 128), 128, 0, st>>>(cnt, lanes > 128 ? lanes / 128 : 1, d_parts,
                                                               d_out + 48 * c0);
        }))
      return r;
  }
  CK(cudaMemcpyAsync(out48, d_out, 48 * n, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(out_ok, d_iok, n, cudaMemcpyDeviceToHost, st));
  if (out_ys32) CK(cudaMemcpyAsync(out_ys32, d_y, 32 * n, cudaMemcpyDeviceToHost, st));
  std::vector<uint8_t> cok(commitments48 ? n : 0);
  if (commitments48) CK(cudaMemcpyAsync(cok.data(), d_cok, n, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (uint64_t i = 0; i < n; i++) {  // where the spec raises: ok = 0 and zero output bytes
    out_ok[i] = out_ok[i] && (!commitments48 || cok[i]);
    if (out_ok[i]) continue;
    memset(out48 + 48 * i, 0, 48);
    if (out_ys32) memset(out_ys32 + 32 * i, 0, 32);
  }
  return NMSM_OK;
}
}  // namespace

int bls12_381_kzg_setup_create_impl(const uint8_t* g1_lagrange48, uint64_t* out_handle) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  cudaStream_t st = C.stream;
  if (X.profiling) memset(X.last_ms, 0, sizeof(X.last_ms));
  const uint64_t o_err = 0, o_enc = 256, o_xy = o_enc + al256(48 * KZG_N), o_aff = o_xy + 96ull * KZG_N,
                 bytes = o_aff + (uint64_t)KZG_N * KzgG::AFF_WORDS * 4;
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  unsigned int* d_err = (unsigned int*)(base + o_err);  // [0]: the smallest bad point, [1..2]: k_prepare's (unused)
  uint32_t *d_xy = (uint32_t*)(base + o_xy), *d_aff = (uint32_t*)(base + o_aff);
  if (int r = h2d_any(base + o_enc, g1_lagrange48, 48 * KZG_N, st)) return r;
  CK(cudaMemsetAsync(d_err, 0xff, 12, st));
  if (int r = pairing_launch(X, C, 0, [&] {
        k_kzg_setup_points<<<KZG_N / 128, 128, 0, st>>>(base + o_enc, d_xy, d_err);
        k_prepare<KzgCv><<<KZG_N / 128, 128, 0, st>>>(d_xy, KZG_N, d_aff, d_err + 1);
      }))
    return r;
  unsigned int bad = 0;
  CK(cudaMemcpyAsync(&bad, d_err, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (bad != 0xffffffffu)
    return fail(NMSM_ERR_POINT,
                "KZG setup point " + std::to_string(bad) + " does not decode to a point of G1 other than the identity",
                (long long)bad);
  uint32_t* tbl = nullptr;
  CK(cudaMalloc((void**)&tbl, kzg_table_bytes(KZG_N)));
  if (int r = kzg_build_table(X, C, d_aff, tbl)) {
    cudaFree(tbl);
    return r;
  }
  KzgSetup* s = new KzgSetup{tbl};
  g_kzg_setups.push_back(s);
  *out_handle = (uint64_t)(uintptr_t)s;
  return NMSM_OK;
}

int bls12_381_kzg_setup_free_impl(uint64_t handle) {
  for (size_t k = 0; k < g_kzg_setups.size(); k++)
    if ((uint64_t)(uintptr_t)g_kzg_setups[k] == handle) {
      cudaFree(g_kzg_setups[k]->d_tbl);
      delete g_kzg_setups[k];
      g_kzg_setups.erase(g_kzg_setups.begin() + k);
      return NMSM_OK;
    }
  return fail(NMSM_ERR_ARG, "unknown KZG setup handle");
}

void kzg_release_setups() {
  for (KzgSetup* s : g_kzg_setups) {
    cudaFree(s->d_tbl);
    s->d_tbl = nullptr;
  }
}

int bls12_381_kzg_commit_batch_impl(uint64_t setup, const uint8_t* blobs, uint64_t n, uint8_t* out_commitments48,
                                    uint8_t* out_ok) {
  return kzg_prove_impl(setup, blobs, nullptr, nullptr, n, out_commitments48, nullptr, out_ok);
}

int bls12_381_kzg_compute_proof_batch_impl(uint64_t setup, const uint8_t* blobs, const uint8_t* zs32, uint64_t n,
                                           uint8_t* out_proofs48, uint8_t* out_ys32, uint8_t* out_ok) {
  return kzg_prove_impl(setup, blobs, zs32, nullptr, n, out_proofs48, out_ys32, out_ok);
}

int bls12_381_kzg_compute_blob_proof_batch_impl(uint64_t setup, const uint8_t* blobs, const uint8_t* commitments48,
                                                uint64_t n, uint8_t* out_proofs48, uint8_t* out_ok) {
  return kzg_prove_impl(setup, blobs, nullptr, commitments48, n, out_proofs48, nullptr, out_ok);
}

int bls12_381_kzg_verify_proof_batch_impl(const uint8_t* commitments48, const uint8_t* zs32, const uint8_t* ys32,
                                          const uint8_t* proofs48, const uint8_t* versioned_hashes32, uint64_t n,
                                          const uint8_t* setup_g2_96, uint8_t* out_ok) {
  return kzg_verify_impl(nullptr, commitments48, zs32, ys32, proofs48, versioned_hashes32, n, setup_g2_96, out_ok);
}

int bls12_381_kzg_verify_blob_batch_impl(const uint8_t* blobs, const uint8_t* commitments48, const uint8_t* proofs48,
                                         uint64_t n, const uint8_t* setup_g2_96, uint8_t* out_ok) {
  return kzg_verify_impl(blobs, commitments48, nullptr, nullptr, proofs48, nullptr, n, setup_g2_96, out_ok);
}

}  // namespace nmsm
