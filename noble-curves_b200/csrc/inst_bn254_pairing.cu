// bn254 pairing checks (SURVEY §8 row f8, pairing_bn254.cuh): the kernels and the C-ABI implementation.  The chunked
// check driver is pairing_driver.cuh's (shared with BLS12-381):
//   k_bn254_miller  one thread per pair: validation and f_i = f_{6u+2,Q_i}(P_i) (with the two Frobenius steps)
//   k_bn254_final   one thread per check: the product of its f_i, the final exponentiation, the verdict
// The Miller values of at most PAIRING_CHUNK pairs are alive at once (PAIRING_CHUNK x 384 B = 25.2 MB).
#include "pairing_bn254.cuh"
#include "pairing_driver.cuh"

namespace nmsm {

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bn254_miller(uint64_t q0, uint32_t cnt, const uint32_t* __restrict__ g1, const uint32_t* __restrict__ g2,
               uint32_t* __restrict__ W, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) pairing_miller_body<Bn254Pairing>(q0 + i, g1, g2, W + (size_t)i * BN_F12_WORDS, err);
}

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bn254_final(uint64_t j0, uint32_t cnt, const uint64_t* __restrict__ off, uint64_t q0, uint64_t q1,
              const uint32_t* __restrict__ W, const uint32_t* carry_in, uint32_t* carry_out,
              const uint8_t* __restrict__ pre_ok, uint8_t* __restrict__ out_ok) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) pairing_final_body<Bn254Pairing>(j0 + i, off, q0, q1, W, carry_in, carry_out, pre_ok, out_ok);
}

int bn254_pairing_check_batch_impl(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                   uint64_t n_checks, uint8_t* out_ok) {
  return pairing_check_batch_impl<Bn254Pairing>(PairingKernels{k_bn254_miller, k_bn254_final}, g1_xy, g2_xy,
                                                pair_off, n_checks, out_ok);
}

}  // namespace nmsm
