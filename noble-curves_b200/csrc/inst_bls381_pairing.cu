// BLS12-381 pairing checks and BLS signature verification (SURVEY §8 row f7, pairing.cuh): the kernels and the two
// C-ABI implementations.  The chunked check driver is pairing_driver.cuh's (shared with bn254):
//   k_bls_verify_prepare  (verify only) one thread per signature: decode, subgroup checks, the two pairs
//   k_bls_miller          one thread per pair: validation and f_i = f_{|x|,Q_i}(P_i) into the workspace
//   k_bls_final           one thread per check: the product of its f_i, the final exponentiation, the verdict
// The Miller values of at most PAIRING_CHUNK pairs are alive at once (PAIRING_CHUNK x 576 B = 37.7 MB).
#include "pairing.cuh"
#include "pairing_driver.cuh"

namespace nmsm {

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bls_miller(uint64_t q0, uint32_t cnt, const uint32_t* __restrict__ g1, const uint32_t* __restrict__ g2,
             uint32_t* __restrict__ W, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) pairing_miller_body<BlsPairing>(q0 + i, g1, g2, W + (size_t)i * BLS_F12_WORDS, err);
}

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bls_final(uint64_t j0, uint32_t cnt, const uint64_t* __restrict__ off, uint64_t q0, uint64_t q1,
            const uint32_t* __restrict__ W, const uint32_t* carry_in, uint32_t* carry_out,
            const uint8_t* __restrict__ pre_ok, uint8_t* __restrict__ out_ok) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) pairing_final_body<BlsPairing>(j0 + i, off, q0, q1, W, carry_in, carry_out, pre_ok, out_ok);
}

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bls_verify_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                     const uint32_t* __restrict__ msg_pts, uint32_t* __restrict__ g1, uint32_t* __restrict__ g2,
                     uint8_t* __restrict__ pre_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) bls_verify_prepare_body(i, sigs, pks, msg_pts, g1, g2, pre_ok, err);
}

namespace {
const PairingKernels BLS_KERNELS{k_bls_miller, k_bls_final};
}  // namespace

int bls12_381_pairing_check_batch_impl(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                       uint64_t n_checks, uint8_t* out_ok) {
  return pairing_check_batch_impl<BlsPairing>(BLS_KERNELS, g1_xy, g2_xy, pair_off, n_checks, out_ok);
}

int bls12_381_verify_batch_impl(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msg_pts, uint64_t n,
                                uint8_t* out_ok) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");
  if (X.profiling) memset(X.last_ms, 0, sizeof(X.last_ms));
  const uint64_t o_sig = 0, o_pk = o_sig + al256(96 * n), o_h = o_pk + al256(48 * n), o_g1 = o_h + al256(192 * n),
                 o_g2 = o_g1 + al256(192 * n), o_pre = o_g2 + al256(384 * n),
                 o_w = o_pre + al256(n), o_ok = o_w + al256(pairing_workspace_bytes<BlsPairing>()),
                 o_misc = o_ok + al256(n), bytes = o_misc + 256;
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  if (int r = h2d_any(base + o_sig, sigs96, 96 * n, st)) return r;
  if (int r = h2d_any(base + o_pk, pks48, 48 * n, st)) return r;
  if (int r = h2d_any(base + o_h, msg_pts, 192 * n, st)) return r;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  uint32_t *d_g1 = (uint32_t*)(base + o_g1), *d_g2 = (uint32_t*)(base + o_g2);
  uint8_t *d_pre = base + o_pre, *d_ok = base + o_ok;
  CK(cudaMemsetAsync(d_err, 0xff, 16, st));
  if (int r = pairing_launch(X, C, 0, [&] {
        k_bls_verify_prepare<<<cdiv(n, PAIRING_BLOCK), PAIRING_BLOCK, 0, st>>>(
            (uint32_t)n, base + o_sig, base + o_pk, (const uint32_t*)(base + o_h), d_g1, d_g2, d_pre, d_err);
      }))
    return r;
  if (int r = pairing_checks_run<BlsPairing>(X, C, BLS_KERNELS, n, nullptr, nullptr, d_g1, d_g2, d_pre,
                                              (uint32_t*)(base + o_w), d_ok, d_err + 2, 1))
    return r;
  unsigned int err[4];
  CK(cudaMemcpyAsync(err, d_err, 16, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (err[0] != 0xffffffffu)
    return fail(NMSM_ERR_POINT,
                "message point " + std::to_string(err[0]) + " is out of range or not on the twist", err[0]);
  if (err[2] != 0xffffffffu || err[3] != 0xffffffffu)  // prepare only emits valid or identity pairs
    return fail(NMSM_ERR_CUDA, "internal error: a prepared pair failed validation");
  CK(cudaMemcpy(out_ok, d_ok, n, cudaMemcpyDeviceToHost));
  return NMSM_OK;
}

}  // namespace nmsm
