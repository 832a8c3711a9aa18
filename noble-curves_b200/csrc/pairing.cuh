// BLS12-381 optimal-ate pairing checks and BLS signature verification (SURVEY §8 row f7).
//
// The reference pairs one (P, Q) at a time (src/abstract/bls.ts `pairing` / `pairingBatch`, bls12-381.ts); here the
// question asked of the GPU is always "is this product of pairings 1", one verdict per check:
//   check j:  prod_{i in [off[j], off[j+1])} e(P_i, Q_i) == 1,   P_i in E(Fp), Q_i on the twist E'(Fp2): y^2 = x^3 + 4 xi
//   verify:   e(pk, H) e(-G1, sig) == 1                            (long signatures: pk in G1, sig and H = H(m) in G2)
//   short:    e(H, pk) e(sig, -G2) == 1                            (short signatures: pk in G2, sig and H = H(m) in G1)
//
// Miller loop: f_{|x|,Q}(P) over the bits of |x| = 0xd201000000010000 (x < 0): 63 doubling steps and 5 addition
// steps.  T runs in homogeneous projective coordinates on the twist (Costello-Lange-Naehrig doubling, mixed addition
// with the affine Q).  Untwisting (x', y') -> (x' / w^2, y' / w^3) turns every line, scaled by a factor of Fp4 that the
// final exponentiation removes, into l0 + l1 v + l4 v w with
//   doubling  l0 = Y^2 - 3 b' Z^2,  l1 = -3 X^2 xP,  l4 = 2 Y Z yP
//   addition  l0 = theta xQ - lambda yQ,  l1 = -theta xP,  l4 = lambda yP   (theta = Y - yQ Z, lambda = X - xQ Z)
// multiplied in sparsely (fp12_mul_by_014).  Vertical lines lie in Fp6 and are dropped.  Since x < 0, f is conjugated at
// the end (f_{x,Q} = 1 / f_{|x|,Q} up to a vertical line, and 1 / f = conj(f) after the easy part).
//
// Final exponentiation: f^(m (p^12 - 1) / r) with m = 3.
//   easy part  f^((p^6 - 1)(p^2 + 1)) = frob2(g) g, g = conj(f) / f  (one Fp12 inversion)
//   hard part  3 (p^4 - p^2 + 1) / r = l0 + l1 p + l2 p^2 + l3 p^3 with  l3 = (x - 1)^2, l2 = l3 x, l1 = l2 x - l3,
//              l0 = l1 x + 3  (an integer identity, checked by tests/test_bls_cpu.py), evaluated with five
//              exponentiations by x in the cyclotomic subgroup (a^x = conj(a^|x|)).
// m = 3 is coprime to r, so "== 1" verdicts are those of the exact pairing; the values tests/hostemu compares are
// those of oracle/bls_pairing_ref.py with the same m.
//
// A pair with an identity point (the affine (0, 0) encoding) contributes 1; the reference's pairing throws on it.
// Bodies are host/device so tests/hostemu can run them; the *_serial statements are what the kernels compute.  The
// check bodies shared with bn254 are pairing_check.cuh's, instantiated with BlsPairing.
#pragma once
#include "codec.cuh"
#include "pairing_check.cuh"

namespace nmsm {

using BlsT = Bls381Tower;
using BlsF = Fp<FpBls381>;
using BlsF2 = Fp2<FpBls381>;
using BlsF12 = Fp12<BlsT>;
static constexpr int BLS_F12_WORDS = BlsF12::WORDS;  // 144 words, 576 bytes
static constexpr uint32_t BLS_M = 3;                 // the final exponentiation computes e^BLS_M

struct BlsG2Proj {
  BlsF2 X, Y, Z;
};

template <class F>
NMSM_HD F times12(const F& a) {
  const F a2 = a + a, a4 = a2 + a2, a8 = a4 + a4;
  return a8 + a4;
}

// T <- 2T (coordinates scaled by 4, which projective coordinates absorb) and the tangent line at P = (xP, yP)
NMSM_HD_NOINLINE void bls_dbl_step(BlsG2Proj& T, const BlsF& neg_xp, const BlsF& yp, BlsF2& l0, BlsF2& l1, BlsF2& l4) {
  const BlsF2 B = sqr(T.Y), Cz = sqr(T.Z), E = times12(BlsT::mul_by_xi(Cz));  // E = 3 b' Z^2, b' = 4 xi
  const BlsF2 Fv = E + E + E, H = sqr(T.Y + T.Z) - B - Cz;                      // H = 2 Y Z
  const BlsF2 X2 = sqr(T.X), X2x3 = X2 + X2 + X2, XY = T.X * T.Y;
  l0 = B - E;
  l1 = BlsF2{X2x3.c0 * neg_xp, X2x3.c1 * neg_xp};
  l4 = BlsF2{H.c0 * yp, H.c1 * yp};
  const BlsF2 BF = B + Fv;
  T.X = (XY + XY) * (B - Fv);
  T.Y = sqr(BF) - times12(sqr(E));
  const BlsF2 BH = B * H;
  T.Z = (BH + BH) + (BH + BH);
}

// T <- T + Q (Q affine) and the line through T and Q at P
NMSM_HD_NOINLINE void bls_add_step(BlsG2Proj& T, const BlsF2& xq, const BlsF2& yq, const BlsF& neg_xp, const BlsF& yp,
                                   BlsF2& l0, BlsF2& l1, BlsF2& l4) {
  const BlsF2 theta = T.Y - yq * T.Z, lambda = T.X - xq * T.Z;
  l0 = theta * xq - lambda * yq;
  l1 = BlsF2{theta.c0 * neg_xp, theta.c1 * neg_xp};
  l4 = BlsF2{lambda.c0 * yp, lambda.c1 * yp};
  const BlsF2 C = sqr(theta), D = sqr(lambda), E = lambda * D, Fv = T.Z * C, G = T.X * D, H = E + Fv - (G + G);
  T.X = lambda * H;
  T.Y = theta * (G - H) - T.Y * E;
  T.Z = T.Z * E;
}

// f_{|x|,Q}(P), conjugated (x < 0).  g1_xy: P canonical (24 words); g2_xy: Q canonical (48 words); neither the identity.
NMSM_HD_NOINLINE BlsF12 bls_miller_loop(const uint32_t* g1_xy, const uint32_t* g2_xy) {
  const BlsF neg_xp = -BlsF::from_canonical(g1_xy), yp = BlsF::from_canonical(g1_xy + 12);
  const BlsF2 xq = BlsF2::from_canonical(g2_xy), yq = BlsF2::from_canonical(g2_xy + 24);
  BlsG2Proj T{xq, yq, BlsF2::one()};
  BlsF12 f = BlsF12::one();
  BlsF2 l0, l1, l4;
  for (int i = 62; i >= 0; i--) {
    if (i != 62) f = fp12_sqr(f);
    bls_dbl_step(T, neg_xp, yp, l0, l1, l4);
    f = fp12_mul_by_014(f, l0, l1, l4);
    const uint32_t bit = i >= 32 ? (Bls381G2Gls::Z(1) >> (i - 32)) & 1u : (Bls381G2Gls::Z(0) >> i) & 1u;
    if (bit) {
      bls_add_step(T, xq, yq, neg_xp, yp, l0, l1, l4);
      f = fp12_mul_by_014(f, l0, l1, l4);
    }
  }
  return fp12_conj(f);
}

// a^x for x = -|x| in the cyclotomic subgroup
NMSM_HD BlsF12 bls_exp_by_x(const BlsF12& a) { return fp12_conj(fp12_cyclotomic_exp_x(a)); }

// f^(3 (p^12 - 1) / r)
NMSM_HD_NOINLINE BlsF12 bls_final_exp(const BlsF12& f) {
  BlsF12 t = fp12_mul(fp12_conj(f), fp12_inv(f));  // f^(p^6 - 1)
  t = fp12_mul(fp12_frobenius<2>(t), t);            // ^(p^2 + 1): now in the cyclotomic subgroup
  BlsF12 a = fp12_mul(bls_exp_by_x(t), fp12_conj(t));                                  // t^(x - 1)
  a = fp12_mul(bls_exp_by_x(a), fp12_conj(a));                                         // t^l3
  const BlsF12 b = bls_exp_by_x(a);                                                    // t^l2
  const BlsF12 c = fp12_mul(bls_exp_by_x(b), fp12_conj(a));                            // t^l1
  const BlsF12 d = fp12_mul(bls_exp_by_x(c), fp12_mul(fp12_cyclotomic_sqr(t), t));     // t^l0
  return fp12_mul(fp12_mul(d, fp12_frobenius<1>(c)), fp12_mul(fp12_frobenius<2>(b), fp12_frobenius<3>(a)));
}

// the pairing policy of pairing_check.cuh
struct BlsPairing {
  using F12 = BlsF12;
  static constexpr int G1_WORDS = 24, G2_WORDS = 48;
  using G1Curve = CurveBls381G1Any;
  using G2Curve = CurveBls381G2Any;
  NMSM_HD static F12 miller_loop(const uint32_t* p, const uint32_t* q) { return bls_miller_loop(p, q); }
  NMSM_HD static F12 final_exp(const F12& f) { return bls_final_exp(f); }
};

// the generator of G1, negated: (Gx, p - Gy) canonical
NMSM_HD uint32_t bls_neg_g1(int k) {
  constexpr uint32_t W[24] = {0xdb22c6bbu, 0xfb3af00au, 0xf97a1aefu, 0x6c55e83fu, 0x171bac58u, 0xa14e3a3fu,
                              0x9774b905u, 0xc3688c4fu, 0x4fa9ac0fu, 0x2695638cu, 0x3197d794u, 0x17f1d3a7u,
                              0xb939c2cau, 0xad54dcd6u, 0x0ecb751bu, 0x4e6f38bau, 0xcaac4236u, 0x6655b9d5u,
                              0x1db507c9u, 0x67816aefu, 0xcf2e21f2u, 0xaa7d76c8u, 0x55d545a8u, 0x114d1d68u};
  return W[k];
}

// torsion_body's predicate (n P == O as (n - 1) P + P) for an in-range point the thread holds: torsion_body itself
// reads its point through the read-only global path, which a thread-local array cannot take
template <class Cv>
NMSM_HD bool bls_in_subgroup(const uint32_t* xy) {
  using G = typename Cv::G;
  uint32_t s[SCALAR_WORDS];
  for (int k = 0; k < SCALAR_WORDS; k++) s[k] = Cv::Fn::ORDER(k);
  s[0] -= 1u;  // the group order is odd
  const typename G::Affine P = G::prepare(xy);
  typename G::Acc acc = scalar_mul_acc<Cv>(P, s);
  nl_madd<G>(acc, P);
  return G::is_identity(acc);
}

// k_bls_verify_prepare, signature i: decode pk (48 B) and sig (96 B), reject identities and points outside the
// subgroups, range- and curve-check H (a caller error: err[0] = smallest bad index).  Writes the pairs 2i = (pk, H) and
// 2i + 1 = (-G1, sig), or two identity pairs when the signature is rejected, and pre_ok[i].
NMSM_HD void bls_verify_prepare_body(uint32_t i, const uint8_t* sigs96, const uint8_t* pks48, const uint32_t* msg_pts,
                                     uint32_t* g1, uint32_t* g2, uint8_t* pre_ok, unsigned int* err) {
  uint32_t pk[24], sig[48], h[48];
  load_words<48>(h, msg_pts + (size_t)i * 48);
  bool ok = true;
  if (!point_on_curve<CurveBls381G2Any>(h)) {
    atomic_min_u32(&err[0], i);
    ok = false;
  }
  ok = ok && !words_zero(h, 48);
  ok = ok && zcash_decode_bls12_381_g1(pks48 + (size_t)i * 48, pk) == 1;
  ok = ok && zcash_decode_bls12_381_g2(sigs96 + (size_t)i * 96, sig) == 1;
  ok = ok && bls_in_subgroup<CurveBls381G1Any>(pk);
  ok = ok && bls_in_subgroup<CurveBls381G2Any>(sig);
  uint32_t* p0 = g1 + (size_t)i * 48;
  uint32_t* q0 = g2 + (size_t)i * 96;
  for (int k = 0; k < 24; k++) {
    p0[k] = ok ? pk[k] : 0u;
    p0[24 + k] = ok ? bls_neg_g1(k) : 0u;
  }
  for (int k = 0; k < 48; k++) {
    q0[k] = ok ? h[k] : 0u;
    q0[48 + k] = ok ? sig[k] : 0u;
  }
  pre_ok[i] = ok ? 1 : 0;
}

// the generator of G2, negated: (Gx, -Gy) canonical in the G2 packing (x.c0, x.c1, y.c0, y.c1)
NMSM_HD uint32_t bls_neg_g2(int k) {
  constexpr uint32_t W[48] = {0xc121bdb8u, 0xd48056c8u, 0xa805bbefu, 0x0bac0326u, 0x7ae3d177u, 0xb4510b64u,
                              0xfa403b02u, 0xc6e47ad4u, 0x2dc51051u, 0x26080527u, 0xf08f0a91u, 0x024aa2b2u,
                              0x5d042b7eu, 0xe5ac7d05u, 0x13945d57u, 0x334cf112u, 0xdc7f5049u, 0xb5da61bbu,
                              0x9920b61au, 0x596bd0d0u, 0x88274f65u, 0x7dacd3a0u, 0x52719f60u, 0x13e02b60u,
                              0xf74782aau, 0xd86bab79u, 0x75a75d75u, 0x8c713632u, 0xa55024f7u, 0xf9ee3837u,
                              0x66c73f17u, 0xb679afdau, 0x691d77bcu, 0xbe51d9efu, 0xc7027888u, 0x0d1b3cc2u,
                              0x0fa030edu, 0x0f55f8a0u, 0x5467e25eu, 0xdf74f2d7u, 0x9f825c78u, 0x40bc3ff5u,
                              0x6dddaf10u, 0x99392306u, 0x1789213du, 0x186ed506u, 0x0ad8b1ceu, 0x13fa4d4au};
  return W[k];
}

// k_bls_short_verify_prepare, signature i (short signatures, bls_verify_prepare_body with the groups swapped): decode
// sig (48 B, G1) and pk (96 B, G2), reject identities and points outside the subgroups, range- and curve-check the G1
// point H (a caller error: err[0] = smallest bad index).  Writes the pairs 2i = (H, pk) and 2i + 1 = (sig, -G2), or two
// identity pairs when the signature is rejected, and pre_ok[i].
NMSM_HD void bls_short_verify_prepare_body(uint32_t i, const uint8_t* sigs48, const uint8_t* pks96,
                                           const uint32_t* msg_pts, uint32_t* g1, uint32_t* g2, uint8_t* pre_ok,
                                           unsigned int* err) {
  uint32_t sig[24], pk[48], h[24];
  load_words<24>(h, msg_pts + (size_t)i * 24);
  bool ok = true;
  if (!point_on_curve<CurveBls381G1Any>(h)) {
    atomic_min_u32(&err[0], i);
    ok = false;
  }
  ok = ok && !words_zero(h, 24);
  ok = ok && zcash_decode_bls12_381_g1(sigs48 + (size_t)i * 48, sig) == 1;
  ok = ok && zcash_decode_bls12_381_g2(pks96 + (size_t)i * 96, pk) == 1;
  ok = ok && bls_in_subgroup<CurveBls381G1Any>(sig);
  ok = ok && bls_in_subgroup<CurveBls381G2Any>(pk);
  uint32_t* p0 = g1 + (size_t)i * 48;
  uint32_t* q0 = g2 + (size_t)i * 96;
  for (int k = 0; k < 24; k++) {
    p0[k] = ok ? h[k] : 0u;
    p0[24 + k] = ok ? sig[k] : 0u;
  }
  for (int k = 0; k < 48; k++) {
    q0[k] = ok ? pk[k] : 0u;
    q0[48 + k] = ok ? bls_neg_g2(k) : 0u;
  }
  pre_ok[i] = ok ? 1 : 0;
}

// ---- serial statement (tests/hostemu): the kernels' work for pairs/checks in order, with chunks of `chunk` pairs ----
// W: (chunk + 2) * BLS_F12_WORDS words (the Miller values and two carry slots, as the library's workspace)
NMSM_HD void bls_check_serial(uint64_t n_checks, const uint64_t* off, const uint32_t* g1, const uint32_t* g2,
                              const uint8_t* pre_ok, uint64_t chunk, uint32_t* W, uint8_t* out_ok, unsigned int* err) {
  pairing_check_serial<BlsPairing>(n_checks, off, g1, g2, pre_ok, chunk, W, out_ok, err);
}

}  // namespace nmsm
