// Instantiation of the MSM / scalar-multiplication engine for secp256k1, plus ECDSA batch verification
// (SURVEY §8 f5, ecdsa_verify.cuh), BIP340 Schnorr batch verification (f6, schnorr_verify.cuh) and ECDSA public-key
// recovery / Ethereum ecrecover (f9, recover.cuh).
#include "engine.cuh"
#include "ecdsa_driver.cuh"
#include "recover.cuh"
#include "schnorr_verify.cuh"

namespace nmsm {
NMSM_DEFINE_ENGINE(engine_secp256k1, CurveSecp256k1)

// decode + SHA-256 + range checks, then u1 = h/s, u2 = r/s with one inversion per warp.  Every lane of a warp reaches
// warp_batch_inverse: lanes past n and invalid signatures feed 1, so one bad signature cannot touch its neighbours.
__global__ void __launch_bounds__(128)
k_ecdsa_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                const uint64_t* __restrict__ pk_off, const uint8_t* __restrict__ msgs,
                const uint64_t* __restrict__ msg_off, int flags, uint32_t* __restrict__ qs, uint32_t* __restrict__ u1s,
                uint32_t* __restrict__ u2s, uint32_t* __restrict__ rs, uint8_t* __restrict__ ok_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t q[16], r[8], s[8], h[8];
  const bool ok = i < n && ecdsa_prepare_body(i, sigs, pks, pk_off, msgs, msg_off, flags, q, r, s, h);
  const EcS w = warp_batch_inverse(ok ? EcS::from_canonical(s) : EcS::one());
  if (i < n) ecdsa_store(i, ok, q, r, h, w, qs, u1s, u2s, rs, ok_out);
}

// R = u1 G + u2 Q and the x comparison
__global__ void __launch_bounds__(128)
k_ecdsa_check(uint32_t n, const uint32_t* __restrict__ g_tbl, const uint32_t* __restrict__ qs,
              const uint32_t* __restrict__ u1s, const uint32_t* __restrict__ u2s, const uint32_t* __restrict__ rs,
              uint8_t* __restrict__ out_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ecdsa_check_body(i, g_tbl, qs, u1s, u2s, rs, out_ok, err);
}

// BIP340: range checks, lift_x, the tagged challenge hash, u = n - e
__global__ void __launch_bounds__(128)
k_schnorr_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                  const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ msg_off, uint32_t* __restrict__ ps,
                  uint32_t* __restrict__ ss, uint32_t* __restrict__ us, uint32_t* __restrict__ rs,
                  uint8_t* __restrict__ ok_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t p[16], r[8], s[8], u[8];
  const bool ok = schnorr_prepare_body(i, sigs, pks, msgs, msg_off, p, r, s, u);
  schnorr_store(i, ok, p, r, s, u, ps, ss, us, rs, ok_out);
}

// R = s G + u P, the x comparison, and y(R) through one inversion per warp.  Every lane of a warp reaches
// warp_batch_inverse: lanes past n, signatures rejected before or by the x comparison, and R = O feed 1.
__global__ void __launch_bounds__(128)
k_schnorr_check(uint32_t n, const uint32_t* __restrict__ g_tbl, const uint32_t* __restrict__ ps,
                const uint32_t* __restrict__ ss, const uint32_t* __restrict__ us, const uint32_t* __restrict__ rs,
                uint8_t* __restrict__ out_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  SchF y = SchF::zero(), z = SchF::one();
  const bool x_ok = i < n && schnorr_check_lane(i, g_tbl, ps, ss, us, rs, out_ok, y, z, err);
  const SchF zi = warp_batch_inverse(z);
  if (i < n) schnorr_finish(i, x_ok, y, zi, out_ok);
}

// Recovery: parse + range checks + lift R + h, then u1 = -h/r, u2 = s/r with one inversion per warp.  Lanes past n
// and failed items feed 1 to warp_batch_inverse.
template <int LAYOUT>
__global__ void __launch_bounds__(128)
k_recover_prepare(uint32_t n, const uint8_t* __restrict__ in, const uint8_t* __restrict__ msgs,
                  const uint64_t* __restrict__ msg_off, int flags, uint32_t* __restrict__ rpts,
                  uint32_t* __restrict__ u1s, uint32_t* __restrict__ u2s, uint8_t* __restrict__ ok_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t rxy[16], r[8], s[8], h[8];
  const bool ok = i < n && recover_prepare_body<LAYOUT>(i, in, msgs, msg_off, flags, rxy, r, s, h);
  const EcS w = warp_batch_inverse(ok ? EcS::from_canonical(r) : EcS::one());
  if (i < n) recover_store(i, ok, rxy, s, h, w, rpts, u1s, u2s, ok_out);
}

// Q = u1 G + u2 R and its affine form (or address word) through one inversion of ZZZ per warp.  Lanes past n, items
// rejected by prepare and Q = O feed 1 to warp_batch_inverse.
template <int LAYOUT>
__global__ void __launch_bounds__(128)
k_recover_check(uint32_t n, const uint32_t* __restrict__ g_tbl, const uint32_t* __restrict__ rpts,
                const uint32_t* __restrict__ u1s, const uint32_t* __restrict__ u2s, uint8_t* __restrict__ ok,
                uint32_t* __restrict__ out, unsigned int* err) {
  using G = CurveSecp256k1::G;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  G::Acc acc = G::identity();
  const bool q_ok = i < n && recover_check_lane(i, g_tbl, rpts, u1s, u2s, ok, acc, err);
  const G::Field zi = warp_batch_inverse(G::inv_target(acc));
  if (i < n) recover_finish<LAYOUT>(i, q_ok, acc, zi, out, ok);
}

// ECDSA, Schnorr verification and recovery share the fixed-point table of G in Context::secp256k1_g_table
int secp256k1_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                                const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok) {
  return ecdsa_verify_batch<CurveSecp256k1, Secp256k1Consts>(k_ecdsa_prepare, k_ecdsa_check, &g_ctx.secp256k1_g_table,
                                                             sigs, pks, pk_off, msgs, msg_off, n, flags, out_ok);
}

int secp256k1_schnorr_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs,
                                        const uint64_t* msg_off, uint64_t n, uint8_t* out_ok) {
  Context& X = g_ctx;
  if (int r = check_offsets(msg_off, "msg_off", n)) return r;
  if (int r = ensure_g_table<CurveSecp256k1, Secp256k1Consts>(&X.secp256k1_g_table)) return r;
  const uint64_t msg_bytes = msg_off[n];
  const uint64_t o_sig = 0, o_pk = o_sig + al256(64 * n), o_msg = o_pk + al256(32 * n),
                 o_mo = o_msg + al256(msg_bytes + 16), o_p = o_mo + al256(8 * (n + 1)), o_s = o_p + al256(64 * n),
                 o_u = o_s + al256(32 * n), o_r = o_u + al256(32 * n), o_ok = o_r + al256(32 * n),
                 o_misc = o_ok + al256(n), total = o_misc + 256;
  CK(X.ed_scratch.ensure(total));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = X.slot[0].stream;
  if (int r = h2d_any(base + o_sig, sigs, 64 * n, st)) return r;
  if (int r = h2d_any(base + o_pk, pks, 32 * n, st)) return r;
  if (int r = h2d_any(base + o_msg, msgs, msg_bytes, st)) return r;
  if (int r = h2d_any(base + o_mo, msg_off, 8 * (n + 1), st)) return r;
  uint32_t *d_p = (uint32_t*)(base + o_p), *d_s = (uint32_t*)(base + o_s), *d_u = (uint32_t*)(base + o_u),
           *d_r = (uint32_t*)(base + o_r);
  uint8_t* d_ok = base + o_ok;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  return verify_launch(
      d_err,
      [&] {
        k_schnorr_prepare<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, base + o_sig, base + o_pk, base + o_msg,
                                                        (const uint64_t*)(base + o_mo), d_p, d_s, d_u, d_r, d_ok);
      },
      [&] {
        k_schnorr_check<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, X.secp256k1_g_table, d_p, d_s, d_u, d_r, d_ok,
                                                      d_err);
      },
      d_ok, out_ok, n);
}

// The host side of both recovery entry points: in = n x 65 B (RECOVER_SIG65, with msgs / msg_off) or n x 128 B
// (RECOVER_ECREC); out = n x 64 B keys or n x 32 B address words.
template <int LAYOUT>
static int recover_batch_impl(const uint8_t* in, const uint8_t* msgs, const uint64_t* msg_off, uint64_t n, int flags,
                              uint8_t* out, uint8_t* out_ok) {
  constexpr bool SIG65 = LAYOUT == RECOVER_SIG65;
  constexpr uint64_t IN_BYTES = SIG65 ? 65 : 128, OUT_WORDS = SIG65 ? 16 : 8;
  Context& X = g_ctx;
  if (SIG65)
    if (int r = check_offsets(msg_off, "msg_off", n)) return r;
  if (int r = ensure_g_table<CurveSecp256k1, Secp256k1Consts>(&X.secp256k1_g_table)) return r;
  const uint64_t msg_bytes = SIG65 ? msg_off[n] : 0;
  const uint64_t o_in = 0, o_msg = o_in + al256(IN_BYTES * n), o_mo = o_msg + al256(msg_bytes + 16),
                 o_r = o_mo + al256(SIG65 ? 8 * (n + 1) : 0), o_u1 = o_r + al256(64 * n), o_u2 = o_u1 + al256(32 * n),
                 o_out = o_u2 + al256(32 * n), o_ok = o_out + al256(4 * OUT_WORDS * n), o_misc = o_ok + al256(n),
                 total = o_misc + 256;
  CK(X.ed_scratch.ensure(total));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = X.slot[0].stream;
  if (int r = h2d_any(base + o_in, in, IN_BYTES * n, st)) return r;
  if (int r = h2d_any(base + o_msg, msgs, msg_bytes, st)) return r;
  if (SIG65)
    if (int r = h2d_any(base + o_mo, msg_off, 8 * (n + 1), st)) return r;
  uint32_t *d_r = (uint32_t*)(base + o_r), *d_u1 = (uint32_t*)(base + o_u1), *d_u2 = (uint32_t*)(base + o_u2),
           *d_out = (uint32_t*)(base + o_out);
  uint8_t* d_ok = base + o_ok;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  return verify_launch(
      d_err,
      [&] {
        k_recover_prepare<LAYOUT><<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, base + o_in, base + o_msg,
                                                                (const uint64_t*)(base + o_mo), flags, d_r, d_u1, d_u2,
                                                                d_ok);
      },
      [&] {
        k_recover_check<LAYOUT><<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, X.secp256k1_g_table, d_r, d_u1, d_u2, d_ok,
                                                              d_out, d_err);
      },
      d_ok, out_ok, n, d_out, out, 4 * OUT_WORDS * n);
}

int secp256k1_recover_batch_impl(const uint8_t* sigs65, const uint8_t* msgs, const uint64_t* msg_off, uint64_t n,
                                 int flags, uint8_t* out_xy, uint8_t* out_ok) {
  return recover_batch_impl<RECOVER_SIG65>(sigs65, msgs, msg_off, n, flags, out_xy, out_ok);
}

int secp256k1_ecrecover_batch_impl(const uint8_t* inputs128, uint64_t n, uint8_t* out32, uint8_t* out_ok) {
  return recover_batch_impl<RECOVER_ECREC>(inputs128, nullptr, nullptr, n, 0, out32, out_ok);
}

}  // namespace nmsm
