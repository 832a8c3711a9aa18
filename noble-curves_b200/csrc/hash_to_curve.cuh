// Hash to BLS12-381 G2 (SURVEY §8 row f10) and G1 (f13): RFC 9380 hash_to_curve with the suites
// BLS12381G2_XMD:SHA-256_SSWU_RO_ (§8.8.2) and BLS12381G1_XMD:SHA-256_SSWU_RO_ (§8.8.1), one message per thread.  The
// references are noble-curves' bls12_381.G2.hashToCurve / G1.hashToCurve(msg, { DST }) (abstract/hash-to-curve.ts,
// bls12-381.ts).
//   h2c_expand_to_fp    expand_message_xmd with SHA-256 and len_in_bytes = 64 NE (§5.3.1), started from the constant
//                       midstate of the 64-byte zero pad; NE 64-byte big-endian integers reduced mod p
//   G2 (Fp2, NE = 4):
//   h2c_hash_to_field   u0 = e0 + e1 u, u1 = e2 + e3 u
//   h2c_sswu            simplified SWU on the isogenous curve E2': y^2 = x^3 + A' x + B' (§6.6.2)
//   h2c_iso_map         the 3-isogeny E2' -> E2 (§E.3), straight into XYZZ coordinates (no inversion)
//   h2c_clear_cofactor  Budroni-Pintore (§G.3): [x^2 - x - 1] P + [x - 1] psi(P) + psi^2(2P), which is [h_eff] P on
//                       every point of E2(Fp2)
//   G1 (Fp, NE = 2):
//   h2c_sswu_g1         simplified SWU on E1' with Z = 11 and one exponentiation
//   h2c_iso_map_g1      the 11-isogeny E1' -> E1 (§E.2), straight into XYZZ coordinates
//   h2c_clear_cofactor_g1  [1 - x] P = P + [|x|] P
//   (kernels)           Q0 + Q1, cleared, made affine through one warp-shared inversion per 32 messages
// The additions and doublings are ec.cuh's XYZZ formulas with their explicit exceptional branches, so P = Q, P = -Q
// and identities (an isogeny kernel point, a cleared point of small order) all give the group law's result.
// Bodies are host/device so tests/hostemu can run them; h2c_hash_serial[_g1] are the kernels' work in order.
#pragma once
#include "ecdsa_verify.cuh"
#include "fp12.cuh"

namespace nmsm {

using H2cF = Fp<FpBls381>;
using H2cF2 = Fp2<FpBls381>;
using H2cG = CurveBls381G2Any::G;
static constexpr uint32_t H2C_MAX_DST = 255;  // longer tags are replaced on the host (RFC 9380 §5.3.3)

// SHA-256 state after one all-zero 64-byte block: the Z_pad prefix of msg_prime
NMSM_HD uint32_t h2c_zpad_midstate(int k) {
  constexpr uint32_t M[8] = {0xda5698beu, 0x17b9b469u, 0x62335799u, 0x779fbecau,
                             0x8ce5d491u, 0xc0d26243u, 0xbafef9eau, 0x1837a9d8u};
  return M[k];
}

// b_i = SHA-256(x || I2OSP(i, 1) || DST_prime) for the 32 bytes x (big-endian words); out: the digest's words
NMSM_HD_NOINLINE void h2c_xmd_block(const uint32_t* x, uint32_t i, const uint8_t* dst, uint32_t dlen, uint32_t* out) {
  uint32_t st[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
  uint8_t digest[32];
  auto byte_at = [&](uint64_t j) -> uint32_t {
    if (j < 32) return (x[j >> 2] >> (24 - 8 * (j & 3))) & 0xffu;
    if (j == 32) return i;
    return j - 33 < dlen ? dst[j - 33] : dlen;  // DST_prime = DST || I2OSP(len(DST), 1)
  };
  sha256_finish(st, 0, 34 + dlen, byte_at, digest);
  for (int k = 0; k < 8; k++) out[k] = st[k];
}

// e * R mod p (Montgomery form, canonical) for the 512-bit e = hi 2^384 + lo in little-endian words w[16]:
//   lo R^2 / R = lo R      lo < 2^384 = R and R^2 mod p < p, so lo R^2 < R p and the Montgomery product's one
//                          conditional subtraction leaves it below p
//   hi R^3 / R = hi 2^384 R   hi < 2^128, R^3 mod p < p: hi R^3 < R p likewise
// and the field addition of the two canonical halves reduces the sum.
NMSM_HD H2cF h2c_reduce512(const uint32_t* w) {
  H2cF lo, hi, r2, r3;
  for (int k = 0; k < 12; k++) {
    lo.v[k] = w[k];
    hi.v[k] = k < 4 ? w[12 + k] : 0u;
    r2.v[k] = FpBls381::R2(k);
    r3.v[k] = Bls381H2c::R3(k);
  }
  return lo * r2 + hi * r3;
}

// expand_message_xmd(msg, DST, 64 NE) (§5.3.1) cut into NE 64-byte big-endian integers, each reduced mod p: the
// count * m = NE elements of hash_to_field (§5.2, L = 64), e_k = OS2IP(b_{2k+1} || b_{2k+2}) mod p
template <int NE>
NMSM_HD void h2c_expand_to_fp(const uint8_t* msg, uint64_t mlen, const uint8_t* dst, uint32_t dlen, H2cF* e) {
  constexpr uint32_t LEN = 64 * NE;  // len_in_bytes
  uint32_t b0[8], prev[8], x[8];
  {
    // b_0 = H(Z_pad || msg || I2OSP(len_in_bytes, 2) || I2OSP(0, 1) || DST_prime)
    uint8_t digest[32];
    for (int k = 0; k < 8; k++) b0[k] = h2c_zpad_midstate(k);
    auto byte_at = [&](uint64_t j) -> uint32_t {
      if (j < mlen) return msg[j];
      j -= mlen;
      if (j < 3) return j == 0 ? LEN >> 8 : j == 1 ? LEN & 0xffu : 0u;
      j -= 3;
      return j < dlen ? dst[j] : dlen;
    };
    sha256_finish(b0, 64, mlen + 4 + dlen, byte_at, digest);
  }
  for (int k = 0; k < 8; k++) prev[k] = 0;  // b_1 hashes b_0 itself
#pragma unroll
  for (int k = 0; k < NE; k++) {
    uint32_t w[16];
#pragma unroll
    for (int h = 0; h < 2; h++) {  // b_i = H((b_0 xor b_{i-1}) || i || DST_prime)
      for (int t = 0; t < 8; t++) x[t] = b0[t] ^ prev[t];
      h2c_xmd_block(x, 2 * k + h + 1, dst, dlen, prev);
      for (int t = 0; t < 8; t++) w[8 * (1 - h) + 7 - t] = prev[t];  // the first digest is the high half
    }
    e[k] = h2c_reduce512(w);
  }
}

// hash_to_field(msg, 2) of §5.2 over Fp2 (len_in_bytes = 256): u0 = e0 + e1 u, u1 = e2 + e3 u
NMSM_HD void h2c_hash_to_field(const uint8_t* msg, uint64_t mlen, const uint8_t* dst, uint32_t dlen, H2cF2& u0,
                               H2cF2& u1) {
  H2cF e[4];
  h2c_expand_to_fp<4>(msg, mlen, dst, dlen, e);
  u0 = H2cF2{e[0], e[1]};
  u1 = H2cF2{e[2], e[3]};
}

// the Fp2 constants of tools/gen_consts.py Bls381H2c (coefficient k of a polynomial)
enum { H2C_A, H2C_B, H2C_Z, H2C_MB_OVER_A, H2C_B_OVER_ZA, H2C_XNUM, H2C_XDEN, H2C_YNUM, H2C_YDEN, H2C_SQRT_MZ };
template <int C>
NMSM_HD constexpr uint32_t h2c_word(int i) {
  if constexpr (C == H2C_A) return Bls381H2c::SSWU_A_MONT(i);
  else if constexpr (C == H2C_B) return Bls381H2c::SSWU_B_MONT(i);
  else if constexpr (C == H2C_Z) return Bls381H2c::SSWU_Z_MONT(i);
  else if constexpr (C == H2C_MB_OVER_A) return Bls381H2c::SSWU_MB_OVER_A_MONT(i);
  else if constexpr (C == H2C_B_OVER_ZA) return Bls381H2c::SSWU_B_OVER_ZA_MONT(i);
  else if constexpr (C == H2C_XNUM) return Bls381H2c::ISO_XNUM_MONT(i);
  else if constexpr (C == H2C_XDEN) return Bls381H2c::ISO_XDEN_MONT(i);
  else if constexpr (C == H2C_YNUM) return Bls381H2c::ISO_YNUM_MONT(i);
  else return Bls381H2c::ISO_YDEN_MONT(i);
}
template <int C>
NMSM_HD H2cF2 h2c_const(int k = 0) {
  H2cF2 r;
  for (int j = 0; j < 12; j++) {
    r.c0.v[j] = h2c_word<C>(24 * k + j);
    r.c1.v[j] = h2c_word<C>(24 * k + 12 + j);
  }
  return r;
}

// sgn0 of §4.1 for Fp2: sign_0 OR (zero_0 AND sign_1), on the canonical coordinates
NMSM_HD uint32_t h2c_sgn0(const H2cF2& a) {
  uint32_t c0[12], c1[12];
  a.c0.to_canonical(c0);
  a.c1.to_canonical(c1);
  return (c0[0] & 1u) | ((a.c0.is_zero() ? 1u : 0u) & c1[0] & 1u);
}

// simplified SWU (§6.6.2), the plain form: x1 = -B'/A' (1 + 1/tv1) with tv1 = Z^2 u^4 + Z u^2 (B'/(Z A') when tv1 = 0),
// then the square root of g(x1), or else of g(Z u^2 x1) = Z^3 u^6 g(x1), which is a square exactly when g(x1) is not;
// sgn0(y) = sgn0(u).
NMSM_HD_NOINLINE void h2c_sswu(const H2cF2& u, H2cF2& x, H2cF2& y) {
  const H2cF2 A = h2c_const<H2C_A>(), B = h2c_const<H2C_B>();
  const H2cF2 zu2 = h2c_const<H2C_Z>() * sqr(u);
  const H2cF2 tv1 = sqr(zu2) + zu2;
  const H2cF2 x1 = tv1.is_zero() ? h2c_const<H2C_B_OVER_ZA>() : h2c_const<H2C_MB_OVER_A>() * (H2cF2::one() + inv(tv1));
  x = x1;
  if (!fp2_sqrt<FpBls381>((sqr(x1) + A) * x1 + B, y)) {
    x = zu2 * x1;
    fp2_sqrt<FpBls381>((sqr(x) + A) * x + B, y);
  }
  if (h2c_sgn0(u) != h2c_sgn0(y)) y = -y;
}

// iso_map (§E.3) of the E2' point (x, y): x = xn / xd, y = y yn / yd, written as XYZZ with Z = xd yd:
//   ZZ = Z^2, ZZZ = Z^3, X = x ZZ = xn yd Z, Y = y ZZZ = y yn xd ZZ.  A kernel point (xd yd = 0) gives ZZ = 0: O.
NMSM_HD_NOINLINE H2cG::Acc h2c_iso_map(const H2cF2& x, const H2cF2& y) {
  H2cF2 xn = h2c_const<H2C_XNUM>(3), yn = h2c_const<H2C_YNUM>(3);
  for (int k = 2; k >= 0; k--) {
    xn = xn * x + h2c_const<H2C_XNUM>(k);
    yn = yn * x + h2c_const<H2C_YNUM>(k);
  }
  const H2cF2 xd = (x + h2c_const<H2C_XDEN>(1)) * x + h2c_const<H2C_XDEN>(0);
  const H2cF2 yd = ((x + h2c_const<H2C_YDEN>(2)) * x + h2c_const<H2C_YDEN>(1)) * x + h2c_const<H2C_YDEN>(0);
  const H2cF2 z = xd * yd, zz = sqr(z);
  return H2cG::Acc{xn * yd * z, y * yn * xd * zz, zz, zz * z};
}

// [|x|] P in the group G (G1 or G2) for the curve parameter |x| = 0xd201000000010000 (Bls381G2Gls::Z): 63 doublings and
// 5 additions
template <class G>
NMSM_HD_NOINLINE typename G::Acc h2c_mul_abs_x(const typename G::Acc& p) {
  typename G::Acc r = p;
  for (int i = 62; i >= 0; i--) {
    G::dbl(r);
    const uint32_t bit = i >= 32 ? (Bls381G2Gls::Z(1) >> (i - 32)) & 1u : (Bls381G2Gls::Z(0) >> i) & 1u;
    if (bit) G::add(r, p);
  }
  return r;
}

// psi(x, y) = (conj(x) PSI_X, conj(y) PSI_Y) on XYZZ coordinates: conjugation is a field automorphism, so
// x = X / ZZ maps to conj(X) / conj(ZZ), and conj(ZZ)^3 = conj(ZZZ)^2 still holds
NMSM_HD H2cG::Acc h2c_psi(const H2cG::Acc& p) {
  H2cF2 cx, cy;
  for (int k = 0; k < 12; k++) {
    cx.c0.v[k] = Bls381G2Gls::PSI_X_C0_MONT(k);
    cx.c1.v[k] = Bls381G2Gls::PSI_X_C1_MONT(k);
    cy.c0.v[k] = Bls381G2Gls::PSI_Y_C0_MONT(k);
    cy.c1.v[k] = Bls381G2Gls::PSI_Y_C1_MONT(k);
  }
  auto conj = [](const H2cF2& a) { return H2cF2{a.c0, -a.c1}; };
  return H2cG::Acc{conj(p.X) * cx, conj(p.Y) * cy, conj(p.ZZ), conj(p.ZZZ)};
}

// psi^2(x, y) = (x PSI2_X, -y), PSI2_X in Fp
NMSM_HD H2cG::Acc h2c_psi2(const H2cG::Acc& p) {
  H2cF c;
  for (int k = 0; k < 12; k++) c.v[k] = Bls381G2Gls::PSI2_X_MONT(k);
  return H2cG::Acc{H2cF2{p.X.c0 * c, p.X.c1 * c}, -p.Y, p.ZZ, p.ZZZ};
}

// clear_cofactor_bls12381_g2 (§G.3).  psi is a group endomorphism of E2, so [x] psi(P) = psi([x] P); with t1 = [x] P:
//   [x^2 - x - 1] P + [x - 1] psi(P) + psi^2(2P) = [x] t1 + psi(t1) - t1 + psi^2(2P) - psi(P) - P
// x < 0: [x] Q = -[|x|] Q.
NMSM_HD_NOINLINE H2cG::Acc h2c_clear_cofactor(const H2cG::Acc& p) {
  using G = H2cG;
  const G::Acc t1 = G::neg(h2c_mul_abs_x<G>(p));
  G::Acc r = p;
  G::dbl(r);
  r = h2c_psi2(r);
  G::add(r, G::neg(h2c_psi(p)));
  G::add(r, G::neg(p));
  G::add(r, h2c_psi(t1));
  G::add(r, G::neg(t1));
  G::Acc q = G::neg(h2c_mul_abs_x<G>(t1));
  G::add(q, r);
  return q;
}

// message i = msgs[msg_off[i], msg_off[i+1]) under the tag dst[0..dlen), 1 <= dlen <= H2C_MAX_DST:
// clear_cofactor(iso_map(sswu(u0)) + iso_map(sswu(u1))) in XYZZ coordinates
NMSM_HD H2cG::Acc h2c_hash_body(uint32_t i, const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* dst,
                                uint32_t dlen) {
  H2cF2 u0, u1, x, y;
  h2c_hash_to_field(msgs + msg_off[i], msg_off[i + 1] - msg_off[i], dst, dlen, u0, u1);
  h2c_sswu(u0, x, y);
  H2cG::Acc q = h2c_iso_map(x, y);
  h2c_sswu(u1, x, y);
  H2cG::add(q, h2c_iso_map(x, y));
  return h2c_clear_cofactor(q);
}

// point i in the G2 packing (x.c0, x.c1, y.c0, y.c1; 48 words) from q and zi = ZZZ^-1; the identity writes (0, 0)
NMSM_HD void h2c_store(uint32_t i, const H2cG::Acc& q, const H2cF2& zi, uint32_t* out) {
  uint32_t xy[48], inf;
  H2cG::to_affine_canonical_with_inv(q, zi, xy, &inf);
  store_words<48>(out + (size_t)i * 48, xy);
}

// serial statement of k_bls_hash_to_g2 (one inversion per message instead of one per warp)
NMSM_HD void h2c_hash_serial(uint32_t n, const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* dst, uint32_t dlen,
                             uint32_t* out) {
  for (uint32_t i = 0; i < n; i++) {
    const H2cG::Acc q = h2c_hash_body(i, msgs, msg_off, dst, dlen);
    h2c_store(i, q, inv(H2cG::inv_target(q)), out);
  }
}

// ---- hash to G1: suite BLS12381G1_XMD:SHA-256_SSWU_RO_ (§8.8.1) -------------------------------------------------
using H2cG1 = CurveBls381G1Any::G;

// the Fp constants of tools/gen_consts.py Bls381H2cG1 (coefficient k of a polynomial)
template <int C>
NMSM_HD constexpr uint32_t h2c_g1_word(int i) {
  if constexpr (C == H2C_A) return Bls381H2cG1::SSWU_A_MONT(i);
  else if constexpr (C == H2C_B) return Bls381H2cG1::SSWU_B_MONT(i);
  else if constexpr (C == H2C_Z) return Bls381H2cG1::SSWU_Z_MONT(i);
  else if constexpr (C == H2C_MB_OVER_A) return Bls381H2cG1::SSWU_MB_OVER_A_MONT(i);
  else if constexpr (C == H2C_B_OVER_ZA) return Bls381H2cG1::SSWU_B_OVER_ZA_MONT(i);
  else if constexpr (C == H2C_SQRT_MZ) return Bls381H2cG1::SSWU_SQRT_MZ_MONT(i);
  else if constexpr (C == H2C_XNUM) return Bls381H2cG1::ISO_XNUM_MONT(i);
  else if constexpr (C == H2C_XDEN) return Bls381H2cG1::ISO_XDEN_MONT(i);
  else if constexpr (C == H2C_YNUM) return Bls381H2cG1::ISO_YNUM_MONT(i);
  else return Bls381H2cG1::ISO_YDEN_MONT(i);
}
template <int C>
NMSM_HD H2cF h2c_g1_const(int k = 0) {
  H2cF r;
  for (int j = 0; j < 12; j++) r.v[j] = h2c_g1_word<C>(12 * k + j);
  return r;
}

// sgn0 of §4.1 for Fp: the parity of the canonical value
NMSM_HD uint32_t h2c_sgn0_fp(const H2cF& a) {
  uint32_t c[12];
  a.to_canonical(c);
  return c[0] & 1u;
}

// simplified SWU on E1': y^2 = x^3 + A' x + B', Z = 11 (§6.6.2), with one exponentiation (p = 3 mod 4, as §F.2.1.2):
// x1 = -B'/A' (1 + 1/tv1), tv1 = Z^2 u^4 + Z u^2 (B'/(Z A') when tv1 = 0), c = g(x1)^((p+1)/4).  When c^2 != g(x1),
// g(x1) is not a square and c^2 = -g(x1); then x2 = Z u^2 x1 has g(x2) = Z^3 u^6 g(x1), whose root is
// Z u^3 sqrt(-Z) c: (Z u^3 sqrt(-Z) c)^2 = -Z^3 u^6 c^2 = Z^3 u^6 g(x1).  sgn0(y) = sgn0(u).
NMSM_HD_NOINLINE void h2c_sswu_g1(const H2cF& u, H2cF& x, H2cF& y) {
  const H2cF A = h2c_g1_const<H2C_A>(), B = h2c_g1_const<H2C_B>();
  const H2cF zu2 = h2c_g1_const<H2C_Z>() * sqr(u);
  const H2cF tv1 = sqr(zu2) + zu2;
  const H2cF x1 =
      tv1.is_zero() ? h2c_g1_const<H2C_B_OVER_ZA>() : h2c_g1_const<H2C_MB_OVER_A>() * (H2cF::one() + inv(tv1));
  bool square;
  const H2cF c = fp_sqrt_3mod4<FpBls381>((sqr(x1) + A) * x1 + B, square);
  if (square) {
    x = x1;
    y = c;
  } else {
    x = zu2 * x1;
    y = zu2 * u * h2c_g1_const<H2C_SQRT_MZ>() * c;
  }
  if (h2c_sgn0_fp(u) != h2c_sgn0_fp(y)) y = -y;
}

// iso_map (§E.2), the 11-isogeny E1' -> E1 of the point (x, y): x = xn / xd, y = y yn / yd (xd, yd monic of degrees
// 10 and 15), written as XYZZ with Z = xd yd exactly as h2c_iso_map: a kernel point (xd yd = 0) gives ZZ = 0, O.
NMSM_HD_NOINLINE H2cG1::Acc h2c_iso_map_g1(const H2cF& x, const H2cF& y) {
  H2cF xn = h2c_g1_const<H2C_XNUM>(11), xd = x + h2c_g1_const<H2C_XDEN>(9);
  H2cF yn = h2c_g1_const<H2C_YNUM>(15), yd = x + h2c_g1_const<H2C_YDEN>(14);
#pragma unroll
  for (int k = 10; k >= 0; k--) xn = xn * x + h2c_g1_const<H2C_XNUM>(k);
#pragma unroll
  for (int k = 8; k >= 0; k--) xd = xd * x + h2c_g1_const<H2C_XDEN>(k);
#pragma unroll
  for (int k = 14; k >= 0; k--) yn = yn * x + h2c_g1_const<H2C_YNUM>(k);
#pragma unroll
  for (int k = 13; k >= 0; k--) yd = yd * x + h2c_g1_const<H2C_YDEN>(k);
  const H2cF z = xd * yd, zz = sqr(z);
  return H2cG1::Acc{xn * yd * z, y * yn * xd * zz, zz, zz * z};
}

// clear_cofactor for G1 (§8.8.1, h_eff = 1 - x = 0xd201000000010001): x < 0, so [1 - x] P = P + [|x|] P
NMSM_HD H2cG1::Acc h2c_clear_cofactor_g1(const H2cG1::Acc& p) {
  H2cG1::Acc q = h2c_mul_abs_x<H2cG1>(p);
  H2cG1::add(q, p);
  return q;
}

// message i as h2c_hash_body takes it: clear_cofactor(iso_map(sswu(u0)) + iso_map(sswu(u1))) for the two Fp elements
// of hash_to_field(msg, 2) (len_in_bytes = 128), in XYZZ coordinates
NMSM_HD H2cG1::Acc h2c_hash_body_g1(uint32_t i, const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* dst,
                                    uint32_t dlen) {
  H2cF u[2], x, y;
  h2c_expand_to_fp<2>(msgs + msg_off[i], msg_off[i + 1] - msg_off[i], dst, dlen, u);
  h2c_sswu_g1(u[0], x, y);
  H2cG1::Acc q = h2c_iso_map_g1(x, y);
  h2c_sswu_g1(u[1], x, y);
  H2cG1::add(q, h2c_iso_map_g1(x, y));
  return h2c_clear_cofactor_g1(q);
}

// point i in the G1 packing (x, y; 24 words) from q and zi = ZZZ^-1; the identity writes (0, 0)
NMSM_HD void h2c_store_g1(uint32_t i, const H2cG1::Acc& q, const H2cF& zi, uint32_t* out) {
  uint32_t xy[24], inf;
  H2cG1::to_affine_canonical_with_inv(q, zi, xy, &inf);
  store_words<24>(out + (size_t)i * 24, xy);
}

// serial statement of k_bls_hash_to_g1 (one inversion per message instead of one per warp)
NMSM_HD void h2c_hash_serial_g1(uint32_t n, const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* dst,
                                uint32_t dlen, uint32_t* out) {
  for (uint32_t i = 0; i < n; i++) {
    const H2cG1::Acc q = h2c_hash_body_g1(i, msgs, msg_off, dst, dlen);
    h2c_store_g1(i, q, inv(H2cG1::inv_target(q)), out);
  }
}

}  // namespace nmsm
