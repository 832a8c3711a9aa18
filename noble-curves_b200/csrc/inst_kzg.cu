// EIP-4844 KZG proof verification (SURVEY §8 row f15, kzg.cuh): the kernels and the two C-ABI implementations.
//   k_kzg_roots      (once per context) one thread per root: the bit-reversed domain into Context::kzg_roots
//   k_kzg_setup      (every call) one thread: decode and subgroup-check [tau] G2
//   k_kzg_challenge  (blobs only) one thread per blob: z = compute_challenge(blob, C)
//   k_kzg_eval       (blobs only) one block per blob: y = f(z), and whether every element is < r
//   k_kzg_prepare    one thread per check: validation and the pairs (Q, -G2), (pi, [tau] G2)
//   k_bls_miller, k_bls_final  the BLS pairing checks of inst_bls381_pairing.cu, two pairs per check
// Blobs go up and are evaluated KZG_CHUNK at a time (128 MiB); only z, y and the verdict of each (65 bytes) outlive
// their chunk, so device memory stays bounded at any n.  The proof stage then runs once over all n.
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
}  // namespace

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
