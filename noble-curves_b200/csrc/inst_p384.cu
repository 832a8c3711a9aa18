// P-384 (secp384r1) ECDSA batch verification (ecdsa_verify.cuh on CurveP384): P-256's two kernels at 12 limbs, with
// SHA-384 as the prehash.  P-384 is not an MSM curve id: this unit instantiates only the verification kernels, the
// host driver of ecdsa_nist.cuh and, through Engine<CurveP384>::build_point_table, the three kernels that build the
// fixed-point table of G (k_prepare, k_table_base, k_table_level).
#include "ecdsa_nist.cuh"

namespace nmsm {

// decode + SHA-384 + range checks, then u1 = h/s, u2 = r/s with one inversion per warp, as k_p256_ecdsa_prepare: lanes
// past n and invalid signatures feed 1 to warp_batch_inverse.
__global__ void __launch_bounds__(128)
k_p384_ecdsa_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                     const uint64_t* __restrict__ pk_off, const uint8_t* __restrict__ msgs,
                     const uint64_t* __restrict__ msg_off, int flags, uint32_t* __restrict__ qs,
                     uint32_t* __restrict__ u1s, uint32_t* __restrict__ u2s, uint32_t* __restrict__ rs,
                     uint8_t* __restrict__ ok_out) {
  using S = EcdsaS<CurveP384>;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t q[24], r[12], s[12], h[12];
  const bool ok = i < n && ecdsa_prepare_body<CurveP384>(i, sigs, pks, pk_off, msgs, msg_off, flags, q, r, s, h);
  const S w = warp_batch_inverse(ok ? S::from_canonical(s) : S::one());
  if (i < n) ecdsa_store<CurveP384>(i, ok, q, r, h, w, qs, u1s, u2s, rs, ok_out);
}

// R = u1 G (fixed-point table of G, 25 levels) + u2 Q (97 plain 4-bit windows), complete addition, and the x
// comparison.  The 8-entry XYZZ window table is 1.5 KB of stack per thread.  Bounds of 4 blocks per SM: 128 registers
// with 56 B of spill stores, against 164 registers and no spills (3 blocks per SM) under (128) alone; at 2^20
// signatures on an H100 the kernel took 214 ms with these bounds and 235 ms without.
__global__ void __launch_bounds__(128, 4)
k_p384_ecdsa_check(uint32_t n, const uint32_t* __restrict__ g_tbl, const uint32_t* __restrict__ qs,
                   const uint32_t* __restrict__ u1s, const uint32_t* __restrict__ u2s, const uint32_t* __restrict__ rs,
                   uint8_t* __restrict__ out_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ecdsa_check_body<PT_BITS, CurveP384>(i, g_tbl, qs, u1s, u2s, rs, out_ok, err);
}

// The fixed-point table of G: 25 levels of 2^15 points of 96 B (79 MB) in Context::p384_g_table.
int p384_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                           const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok) {
  return nist_ecdsa_verify_batch<CurveP384, P384Consts>(k_p384_ecdsa_prepare, k_p384_ecdsa_check, &g_ctx.p384_g_table,
                                                        sigs, pks, pk_off, msgs, msg_off, n, flags, out_ok);
}

}  // namespace nmsm
