// bn254 optimal-ate pairing checks (SURVEY §8 row f8): Ethereum's ecPairing (EIP-197), Groth16 and KZG verification.
//
// The reference pairs one (P, Q) at a time (src/abstract/bls.ts `pairing` / `pairingBatch`, bn254.ts); here, as for
// BLS12-381 (pairing.cuh), the question asked of the GPU is always "is this product of pairings 1":
//   check j:  prod_{i in [off[j], off[j+1])} e(P_i, Q_i) == 1,   P_i in E(Fp): y^2 = x^3 + 3,
//                                                                 Q_i on the D-type twist E'(Fp2): y^2 = x^3 + 3 / xi
//
// Miller loop: f_{6u+2,Q}(P) over the non-adjacent form of 6u + 2 = 0x19d797039be763ba8 (u = 0x44e992b44a6909f1 > 0;
// 66 digits, 22 of them non-zero, tools/gen_consts.py Bn254Ate): 65 doubling steps and 21 addition steps with Q or -Q,
// then the two addition steps with Q1 = pi(Q) and -Q2 = -pi^2(Q) (pi(x', y') = (conj(x') xi^((p-1)/3),
// conj(y') xi^((p-1)/2)), -pi^2(x', y') = (x' xi^((p^2-1)/3), y'), Bn254Frob).  u > 0: no final conjugation.
// T runs in homogeneous projective coordinates on the twist with the same doubling and mixed-addition formulas as
// BLS12-381.  Untwisting (x', y') -> (x' w^2, y' w^3) turns every line, scaled by a factor of Fp2 that the final
// exponentiation removes, into l0 + l3 w + l4 v w with
//   doubling  l0 = 2 Y Z yP,  l3 = -3 X^2 xP,  l4 = Y^2 - 3 b' Z^2
//   addition  l0 = lambda yP,  l3 = -theta xP,  l4 = theta xQ - lambda yQ   (theta = Y - yQ Z, lambda = X - xQ Z)
// multiplied in sparsely (fp12_mul_by_034).  Vertical lines lie in Fp6 and are dropped; for Q in G2 the last step's line
// is vertical times w (T = pi^2(Q)), which the final exponentiation also removes.
//
// Final exponentiation: f^(M (p^12 - 1) / r) with M = 2u (6u^2 + 3u + 1), gcd(M, r) = 1.
//   easy part  f^((p^6 - 1)(p^2 + 1)) as for BLS12-381
//   hard part  M (p^4 - p^2 + 1) / r = l0 + l1 p + l2 p^2 + l3 p^3 (Fuentes-Castaneda, Knapp, Rodriguez-Henriquez) with
//              l0 = 1 + 6u + 12u^2 + 12u^3, l1 = 4u + 6u^2 + 12u^3, l2 = 6u + 6u^2 + 12u^3, l3 = -1 + 4u + 6u^2 + 12u^3
//              (checked by tests/test_bn254_pairing_cpu.py), evaluated with three exponentiations by u.
// "== 1" verdicts are those of the exact pairing; the values tests/hostemu compares are those of
// oracle/bn254_pairing_ref.py with the same M.
//
// A pair with an identity point (the affine (0, 0) encoding) contributes 1.  Bodies are host/device so tests/hostemu
// can run them; the check bodies are pairing_check.cuh's, instantiated with Bn254Pairing.
#pragma once
#include "pairing_check.cuh"

namespace nmsm {

using BnT = Bn254Tower;
using BnF = Fp<FpBn254>;
using BnF2 = Fp2<FpBn254>;
using BnF12 = Fp12<BnT>;
static constexpr int BN_F12_WORDS = BnF12::WORDS;  // 96 words, 384 bytes

struct BnG2Proj {
  BnF2 X, Y, Z;
};

NMSM_HD BnF2 bn_mul_fp(const BnF2& a, const BnF& b) { return BnF2{a.c0 * b, a.c1 * b}; }

// T <- 2T (coordinates scaled by 4, which projective coordinates absorb) and the tangent line at P = (xP, yP)
NMSM_HD_NOINLINE void bn_dbl_step(BnG2Proj& T, const BnF& neg_xp, const BnF& yp, BnF2& l0, BnF2& l3, BnF2& l4) {
  BnF2 b3;  // 3 b'
  for (int i = 0; i < 8; i++) {
    b3.c0.v[i] = Bn254Ate::B3_C0_MONT(i);
    b3.c1.v[i] = Bn254Ate::B3_C1_MONT(i);
  }
  const BnF2 B = sqr(T.Y), Cz = sqr(T.Z), E = b3 * Cz;  // E = 3 b' Z^2
  const BnF2 Fv = E + E + E, H = sqr(T.Y + T.Z) - B - Cz;  // H = 2 Y Z
  const BnF2 X2 = sqr(T.X), X2x3 = X2 + X2 + X2, XY = T.X * T.Y;
  l0 = bn_mul_fp(H, yp);
  l3 = bn_mul_fp(X2x3, neg_xp);
  l4 = B - E;
  const BnF2 BF = B + Fv, E2 = sqr(E), E4 = (E2 + E2) + (E2 + E2), E12 = E4 + E4 + E4;
  T.X = (XY + XY) * (B - Fv);
  T.Y = sqr(BF) - E12;
  const BnF2 BH = B * H;
  T.Z = (BH + BH) + (BH + BH);
}

// T <- T + Q (Q affine) and the line through T and Q at P
NMSM_HD_NOINLINE void bn_add_step(BnG2Proj& T, const BnF2& xq, const BnF2& yq, const BnF& neg_xp, const BnF& yp,
                                  BnF2& l0, BnF2& l3, BnF2& l4) {
  const BnF2 theta = T.Y - yq * T.Z, lambda = T.X - xq * T.Z;
  l0 = bn_mul_fp(lambda, yp);
  l3 = bn_mul_fp(theta, neg_xp);
  l4 = theta * xq - lambda * yq;
  const BnF2 C = sqr(theta), D = sqr(lambda), E = lambda * D, Fv = T.Z * C, G = T.X * D, H = E + Fv - (G + G);
  T.X = lambda * H;
  T.Y = theta * (G - H) - T.Y * E;
  T.Z = T.Z * E;
}

// f_{6u+2,Q}(P) l_{T,Q1}(P) l_{T+Q1,-Q2}(P).  g1_xy: P canonical (16 words); g2_xy: Q canonical (32 words); neither
// the identity.
NMSM_HD_NOINLINE BnF12 bn_miller_loop(const uint32_t* g1_xy, const uint32_t* g2_xy) {
  const BnF neg_xp = -BnF::from_canonical(g1_xy), yp = BnF::from_canonical(g1_xy + 8);
  const BnF2 xq = BnF2::from_canonical(g2_xy), yq = BnF2::from_canonical(g2_xy + 16), neg_yq = -yq;
  BnG2Proj T{xq, yq, BnF2::one()};
  BnF12 f = BnF12::one();
  BnF2 l0, l3, l4;
  for (int i = Bn254Ate::NAF_TOP - 1; i >= 0; i--) {
    if (i != Bn254Ate::NAF_TOP - 1) f = fp12_sqr(f);
    bn_dbl_step(T, neg_xp, yp, l0, l3, l4);
    f = fp12_mul_by_034(f, l0, l3, l4);
    const uint32_t pos = (Bn254Ate::NAF_POS(i >> 5) >> (i & 31)) & 1u, neg = (Bn254Ate::NAF_NEG(i >> 5) >> (i & 31)) & 1u;
    if (pos | neg) {
      bn_add_step(T, xq, pos ? yq : neg_yq, neg_xp, yp, l0, l3, l4);
      f = fp12_mul_by_034(f, l0, l3, l4);
    }
  }
  BnF2 tx1, ty1;
  BnF tx2;
  for (int i = 0; i < 8; i++) {
    tx1.c0.v[i] = Bn254Frob::TWIST_X1_C0_MONT(i);
    tx1.c1.v[i] = Bn254Frob::TWIST_X1_C1_MONT(i);
    ty1.c0.v[i] = Bn254Frob::TWIST_Y1_C0_MONT(i);
    ty1.c1.v[i] = Bn254Frob::TWIST_Y1_C1_MONT(i);
    tx2.v[i] = Bn254Frob::TWIST_X2_MONT(i);
  }
  bn_add_step(T, BnF2{xq.c0, -xq.c1} * tx1, BnF2{yq.c0, -yq.c1} * ty1, neg_xp, yp, l0, l3, l4);  // Q1 = pi(Q)
  f = fp12_mul_by_034(f, l0, l3, l4);
  bn_add_step(T, bn_mul_fp(xq, tx2), yq, neg_xp, yp, l0, l3, l4);  // -Q2 = -pi^2(Q)
  return fp12_mul_by_034(f, l0, l3, l4);
}

// f^(M (p^12 - 1) / r), M = 2u (6u^2 + 3u + 1)
NMSM_HD_NOINLINE BnF12 bn_final_exp(const BnF12& f) {
  BnF12 t = fp12_mul(fp12_conj(f), fp12_inv(f));  // f^(p^6 - 1)
  t = fp12_mul(fp12_frobenius<2>(t), t);           // ^(p^2 + 1): now in the cyclotomic subgroup
  const BnF12 a = fp12_cyclotomic_exp_x(t);                                      // t^u
  const BnF12 a2 = fp12_cyclotomic_sqr(a), a4 = fp12_cyclotomic_sqr(a2);         // t^2u, t^4u
  const BnF12 a6 = fp12_mul(a4, a2);                                             // t^6u
  const BnF12 b = fp12_cyclotomic_exp_x(a6);                                     // t^6u^2
  const BnF12 c = fp12_cyclotomic_exp_x(fp12_cyclotomic_sqr(b));                 // t^12u^3
  const BnF12 d = fp12_mul(c, b);                                                // t^(12u^3 + 6u^2)
  const BnF12 l2 = fp12_mul(d, a6), l1 = fp12_mul(d, a4);                        // t^l2, t^l1
  const BnF12 l0 = fp12_mul(fp12_mul(l2, b), t), l3 = fp12_mul(l1, fp12_conj(t));  // t^l0, t^l3
  return fp12_mul(fp12_mul(l0, fp12_frobenius<1>(l1)), fp12_mul(fp12_frobenius<2>(l2), fp12_frobenius<3>(l3)));
}

// the pairing policy of pairing_check.cuh
struct Bn254Pairing {
  using F12 = BnF12;
  static constexpr int G1_WORDS = 16, G2_WORDS = 32;
  using G1Curve = CurveBn254G1;
  using G2Curve = CurveBn254G2;
  NMSM_HD static F12 miller_loop(const uint32_t* p, const uint32_t* q) { return bn_miller_loop(p, q); }
  NMSM_HD static F12 final_exp(const F12& f) { return bn_final_exp(f); }
};

}  // namespace nmsm
