// secp256k1 BIP340 Schnorr batch verification (SURVEY §8 row f6): one independent verdict per signature.
//
// The reference verifies one signature at a time: secp256k1.ts `schnorr.verify(signature, message, publicKey)`
// (noble-curves v2), i.e. BIP340 verification.  sig = r || s (64 B, big-endian), pk = x (32 B); inside the reference's
// try (any failure = false):
//   P = lift_x(x): x < p and x^3 + 7 a square, y the even root;  1 <= r < p;  1 <= s < n;
//   e = int(SHA256(T || T || r || pk || m)) mod n, T = SHA256("BIP0340/challenge"), r hashed as the 32 bytes given;
//   R = s G - e P;  accept iff R != O, y(R) even and x(R) == r (an integer comparison in Fp).
// As for ECDSA (ecdsa_verify.cuh) the batch is data-parallel, split into two kernels (inst_secp256k1.cu):
//   schnorr_prepare_body  range checks, lift_x (sec1_decode_secp256k1 with the even prefix 0x02), the tagged hash from
//                         the constant midstate of T || T, u = n - e
//   schnorr_check_lane    R = s G (fixed-point table of G) + u P (GLV scalar_mul_acc), complete addition, x(R) == r
//                         in XYZZ coordinates (X == r ZZ) without an inversion
//   (kernel)              ZZZ^-1 through one warp-shared inversion per 32 signatures (msm.cuh warp_batch_inverse)
//   schnorr_finish        y(R) = Y ZZZ^-1, canonical, even
// Bodies are host/device so tests/hostemu can run them; the *_serial statements invert once per signature.
#pragma once
#include "ecdsa_verify.cuh"

namespace nmsm {

using SchF = Fp<FpSecp256k1>;

// SHA-256 state after the one block T || T, T = SHA256("BIP0340/challenge") (BIP340 tagged hash)
NMSM_HD uint32_t bip340_challenge_midstate(int k) {
  constexpr uint32_t M[8] = {0x9cecba11u, 0x23925381u, 0x11679112u, 0xd1627e0fu,
                             0x97c87550u, 0x003cc765u, 0x90f61164u, 0x33e9b66au};
  return M[k];
}

// SHA256(T || T || r32 || pk32 || m[0..mlen)) -> out[32]
NMSM_HD void bip340_challenge(const uint8_t* r32, const uint8_t* pk32, const uint8_t* m, uint64_t mlen, uint8_t* out) {
  uint32_t st[8];
  for (int k = 0; k < 8; k++) st[k] = bip340_challenge_midstate(k);
  auto byte_at = [&](uint64_t j) -> uint32_t { return j < 32 ? r32[j] : j < 64 ? pk32[j - 32] : m[j - 64]; };
  sha256_finish(st, 64, 64 + mlen, byte_at, out);
}

// Signature i: P = lift_x(pk) (canonical affine words), r, s and u = (n - e) mod n.  False = the reference's verify
// returns false before any scalar multiplication; the outputs are then unspecified.
NMSM_HD bool schnorr_prepare_body(uint32_t i, const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs,
                                  const uint64_t* msg_off, uint32_t* p_xy, uint32_t* r, uint32_t* s, uint32_t* u) {
  const uint8_t* sig = sigs + (size_t)i * 64;
  const uint8_t* pk = pks + (size_t)i * 32;
  words_from_be_bytes<32>(r, sig);
  words_from_be_bytes<32>(s, sig + 32);
  if (!words8_nonzero(r) || !SchF::canonical_in_range(r) || !words8_nonzero(s) || !EcS::canonical_in_range(s))
    return false;
  uint8_t enc[33];  // lift_x(x) is the SEC1 decode of 02 || x
  enc[0] = 0x02;
  for (int k = 0; k < 32; k++) enc[1 + k] = pk[k];
  if (sec1_decode_secp256k1(enc, p_xy) != 1) return false;
  uint8_t digest[32];
  bip340_challenge(sig, pk, msgs + msg_off[i], msg_off[i + 1] - msg_off[i], digest);
  uint32_t e[8];
  words_from_be_bytes<32>(e, digest);
  if (!EcS::canonical_in_range(e)) {  // e < 2^256 < 2n: one subtraction reduces it
    e[0] = sub_cc(e[0], FnSecp256k1Mod::P(0));
    for (int k = 1; k < 8; k++) e[k] = subc_cc(e[k], FnSecp256k1Mod::P(k));
  }
  const bool e_zero = !words8_nonzero(e);
  u[0] = sub_cc(FnSecp256k1Mod::P(0), e[0]);
  for (int k = 1; k < 8; k++) u[k] = subc_cc(FnSecp256k1Mod::P(k), e[k]);
  if (e_zero)
    for (int k = 0; k < 8; k++) u[k] = 0;
  return true;
}

// the per-signature state k_schnorr_check reads; ok_out[i] carries the prepare verdict to the check
NMSM_HD void schnorr_store(uint32_t i, bool ok, const uint32_t* p_xy, const uint32_t* r, const uint32_t* s,
                           const uint32_t* u, uint32_t* ps, uint32_t* ss, uint32_t* us, uint32_t* rs, uint8_t* ok_out) {
  ok_out[i] = ok ? 1 : 0;
  if (!ok) return;
  store_words<16>(ps + (size_t)i * 16, p_xy);
  store_words<8>(ss + (size_t)i * 8, s);
  store_words<8>(us + (size_t)i * 8, u);
  store_words<8>(rs + (size_t)i * 8, r);
}

NMSM_HD void schnorr_prepare_serial(uint32_t n, const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs,
                                    const uint64_t* msg_off, uint32_t* ps, uint32_t* ss, uint32_t* us, uint32_t* rs,
                                    uint8_t* ok_out) {
  for (uint32_t i = 0; i < n; i++) {
    uint32_t p[16], r[8], s[8], u[8];
    const bool ok = schnorr_prepare_body(i, sigs, pks, msgs, msg_off, p, r, s, u);
    schnorr_store(i, ok, p, r, s, u, ps, ss, us, rs, ok_out);
  }
}

// The per-lane part of the check for signature i after schnorr_store: R = s G + u P.  Returns true iff prepare
// accepted, R != O and x(R) == r (X == r ZZ); then y_num = Y and zzz = ZZZ (y(R) = Y / ZZZ).  Otherwise zzz = 1, so
// that the lane can feed the warp-shared inversion without touching its neighbours.  tbl: the fixed-point table of G
// (table_mul_body layout, BITS-bit digits; BITS is a parameter only so that tests/hostemu can use a small table).
template <int BITS = PT_BITS>
NMSM_HD bool schnorr_check_lane(uint32_t i, const uint32_t* tbl, const uint32_t* ps, const uint32_t* ss,
                                const uint32_t* us, const uint32_t* rs, const uint8_t* ok_in, SchF& y_num, SchF& zzz,
                                unsigned int* err) {
  using Cv = CurveSecp256k1;
  using G = Cv::G;
  zzz = SchF::one();
  if (!ok_in[i]) return false;
  G::Acc acc;
  table_mul_body<Cv, BITS>(i, tbl, ss, 1, acc, err);  // 1 <= s < n
  uint32_t p[16], u[8], r[8];
  load_words<16>(p, ps + (size_t)i * 16);
  load_words<8>(u, us + (size_t)i * 8);
  load_words<8>(r, rs + (size_t)i * 8);
  nl_add<G>(acc, scalar_mul_acc<Cv>(G::prepare(p), u));  // complete: u = 0 adds O, s G == u P doubles
  if (G::is_identity(acc) || !(acc.X == SchF::from_canonical(r) * acc.ZZ)) return false;  // r < p
  y_num = acc.Y;
  zzz = acc.ZZZ;
  return true;
}

// out_ok[i] = x_ok and y(R) = y_num * zzz_inv is even
NMSM_HD void schnorr_finish(uint32_t i, bool x_ok, const SchF& y_num, const SchF& zzz_inv, uint8_t* out_ok) {
  bool ok = false;
  if (x_ok) {
    uint32_t y[8];
    (y_num * zzz_inv).to_canonical(y);
    ok = (y[0] & 1u) == 0;
  }
  out_ok[i] = ok ? 1 : 0;
}

// serial statement of k_schnorr_check (one inversion per signature instead of one per warp)
template <int BITS = PT_BITS>
NMSM_HD void schnorr_check_serial(uint32_t n, const uint32_t* tbl, const uint32_t* ps, const uint32_t* ss,
                                  const uint32_t* us, const uint32_t* rs, uint8_t* out_ok, unsigned int* err) {
  for (uint32_t i = 0; i < n; i++) {
    SchF y = SchF::zero(), z;
    const bool x_ok = schnorr_check_lane<BITS>(i, tbl, ps, ss, us, rs, out_ok, y, z, err);
    schnorr_finish(i, x_ok, y, inv(z), out_ok);
  }
}

}  // namespace nmsm
