// P-256 (secp256r1) ECDSA batch verification (ecdsa_verify.cuh on CurveP256): the same two kernels as secp256k1's
// k_ecdsa_prepare / k_ecdsa_check, over the a = -3 group law.  P-256 is not an MSM curve id: this unit instantiates
// only the verification kernels, the host driver of ecdsa_driver.cuh and, through
// Engine<CurveP256>::build_point_table, the three kernels that build the fixed-point table of G (k_prepare,
// k_table_base, k_table_level).
#include "ecdsa_driver.cuh"

namespace nmsm {

// decode + SHA-256 + range checks, then u1 = h/s, u2 = r/s with one inversion per warp.  Every lane of a warp reaches
// warp_batch_inverse: lanes past n and invalid signatures feed 1, so one bad signature cannot touch its neighbours.
__global__ void __launch_bounds__(128)
k_p256_ecdsa_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                     const uint64_t* __restrict__ pk_off, const uint8_t* __restrict__ msgs,
                     const uint64_t* __restrict__ msg_off, int flags, uint32_t* __restrict__ qs,
                     uint32_t* __restrict__ u1s, uint32_t* __restrict__ u2s, uint32_t* __restrict__ rs,
                     uint8_t* __restrict__ ok_out) {
  using S = EcdsaS<CurveP256>;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t q[16], r[8], s[8], h[8];
  const bool ok = i < n && ecdsa_prepare_body<CurveP256>(i, sigs, pks, pk_off, msgs, msg_off, flags, q, r, s, h);
  const S w = warp_batch_inverse(ok ? S::from_canonical(s) : S::one());
  if (i < n) ecdsa_store<CurveP256>(i, ok, q, r, h, w, qs, u1s, u2s, rs, ok_out);
}

// R = u1 G (fixed-point table of G) + u2 Q (4-bit windows), complete addition, and the x comparison.  Bounds of 4 blocks
// per SM: with (128) alone ptxas picks 96 registers and spills 32 B around the out-of-line group operations; at 127
// registers nothing spills.
__global__ void __launch_bounds__(128, 4)
k_p256_ecdsa_check(uint32_t n, const uint32_t* __restrict__ g_tbl, const uint32_t* __restrict__ qs,
                   const uint32_t* __restrict__ u1s, const uint32_t* __restrict__ u2s, const uint32_t* __restrict__ rs,
                   uint8_t* __restrict__ out_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ecdsa_check_body<PT_BITS, CurveP256>(i, g_tbl, qs, u1s, u2s, rs, out_ok, err);
}

// The fixed-point table of G: 17 levels of 2^15 points (36 MB) in Context::p256_g_table.
int p256_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                           const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok) {
  return ecdsa_verify_batch<CurveP256, P256Consts>(k_p256_ecdsa_prepare, k_p256_ecdsa_check, &g_ctx.p256_g_table, sigs,
                                                   pks, pk_off, msgs, msg_off, n, flags, out_ok);
}

}  // namespace nmsm
