// P-256 (secp256r1) ECDSA batch verification (ecdsa_verify.cuh on CurveP256): the same two kernels as secp256k1's
// k_ecdsa_prepare / k_ecdsa_check, over the a = -3 group law.  P-256 is not an MSM curve id: this unit instantiates
// only the verification kernels and, through Engine<CurveP256>::build_point_table, the three kernels that build the
// fixed-point table of G (k_prepare, k_table_base, k_table_level).
#include "engine.cuh"
#include "ecdsa_verify.cuh"

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

// The fixed-point table of G: d * 2^(16 j) * G, 17 levels of 2^15 points (36 MB).  Built by the first verify after
// nmsm_init, freed by nmsm_shutdown.
static int ensure_p256_g_table(Context& X) {
  if (X.p256_g_table) return NMSM_OK;
  uint32_t g_xy[16];
  for (int k = 0; k < 8; k++) {
    g_xy[k] = P256Consts::GX(k);
    g_xy[8 + k] = P256Consts::GY(k);
  }
  int levels = 0;
  return Engine<CurveP256>::build_point_table((const uint8_t*)g_xy, &X.p256_g_table, &levels);
}

int p256_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                           const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  if (int r = check_offsets(pk_off, "pk_off", n)) return r;
  if (int r = check_offsets(msg_off, "msg_off", n)) return r;
  if (int r = ensure_p256_g_table(X)) return r;
  const uint64_t pk_bytes = pk_off[n], msg_bytes = msg_off[n];
  auto al = [](uint64_t x) { return (x + 255) & ~255ull; };
  const uint64_t o_sig = 0, o_pk = o_sig + al(64 * n), o_pko = o_pk + al(pk_bytes + 16), o_msg = o_pko + al(8 * (n + 1)),
                 o_mo = o_msg + al(msg_bytes + 16), o_q = o_mo + al(8 * (n + 1)), o_u1 = o_q + al(64 * n),
                 o_u2 = o_u1 + al(32 * n), o_r = o_u2 + al(32 * n), o_ok = o_r + al(32 * n), o_misc = o_ok + al(n),
                 total = o_misc + 256;
  CK(X.ed_scratch.ensure(total));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  if (int r = h2d_any(base + o_sig, sigs, 64 * n, st)) return r;
  if (pk_bytes)
    if (int r = h2d_any(base + o_pk, pks, pk_bytes, st)) return r;
  if (int r = h2d_any(base + o_pko, pk_off, 8 * (n + 1), st)) return r;
  if (msg_bytes)
    if (int r = h2d_any(base + o_msg, msgs, msg_bytes, st)) return r;
  if (int r = h2d_any(base + o_mo, msg_off, 8 * (n + 1), st)) return r;
  uint32_t *d_q = (uint32_t*)(base + o_q), *d_u1 = (uint32_t*)(base + o_u1), *d_u2 = (uint32_t*)(base + o_u2),
           *d_r = (uint32_t*)(base + o_r);
  uint8_t* d_ok = base + o_ok;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  CK(cudaMemsetAsync(d_err, 0xff, 8, st));
  EV(0);
  k_p256_ecdsa_prepare<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, base + o_sig, base + o_pk,
                                                     (const uint64_t*)(base + o_pko), base + o_msg,
                                                     (const uint64_t*)(base + o_mo), flags, d_q, d_u1, d_u2, d_r, d_ok);
  EV(1);
  k_p256_ecdsa_check<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, X.p256_g_table, d_q, d_u1, d_u2, d_r, d_ok, d_err);
  EV(2);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out_ok, d_ok, n, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  record_verify_timing(X, C);
  return NMSM_OK;
}

}  // namespace nmsm
