// Wire-format decoding on the GPU (SURVEY §8 row f2): bytes -> canonical affine (x, y) in the C-ABI packing,
// so callers can hand the encodings the reference's `fromBytes` consumes instead of bigints.
//   secp256k1  SEC1 compressed, 33 B      /root/reference/src/abstract/weierstrass.ts:565-588 (pointFromBytes)
//              (the same decoder serves P-256 and, 49 B, P-384 ECDSA keys, ecdsa_verify.cuh)
//   BLS12-381 G1  Zcash-flag compressed, 48 B   src/bls12-381.ts:377-468 (coder.decode, parseMask/validateMask)
//   BLS12-381 G2  Zcash-flag compressed, 96 B   same coder over Fp2 (c1 || c0, bls12-381.ts:354-367,488-491), Fp2 sqrt tower.ts:476-498
//   ed25519    RFC 8032 / ZIP-215, 32 B   src/abstract/edwards.ts:405-436  (ed25519_verify.cuh ed_decompress)
// Only the decode step is mirrored (coordinates from bytes); the reference's `Point.fromBytes` additionally runs
// assertValidity (subgroup membership for cofactor > 1), which is a scalar multiplication of its own.
#pragma once
#include "ed25519_verify.cuh"
#include "validate.cuh"

namespace nmsm {

// a^((p+1)/4) for p = 3 (mod 4); ok iff the result squares back to a  (weierstrass.ts:579 "y = y2 ^ (p+1)/4")
template <class P>
NMSM_HD Fp<P> fp_sqrt_3mod4(const Fp<P>& a, bool& ok) {
  constexpr int N = P::N;
  uint32_t e[N];  // (p + 1) >> 2
  {
    uint32_t t[N];
    t[0] = add_cc(P::P(0), 1u);
    for (int k = 1; k < N; k++) t[k] = addc_cc(P::P(k), 0u);
    uint32_t top = addc(0, 0);  // only non-zero for p = 2^(32N) - 1, which no supported prime is
    for (int k = 0; k < N - 1; k++) e[k] = (t[k] >> 2) | (t[k + 1] << 30);
    e[N - 1] = (t[N - 1] >> 2) | (top << 30);
  }
  Fp<P> r = Fp<P>::one();
  bool started = false;
  for (int i = N - 1; i >= 0; i--)
    for (int bit = 31; bit >= 0; bit--) {
      if (started) r = sqr(r);
      if ((e[i] >> bit) & 1) {
        r = r * a;
        started = true;
      }
    }
  ok = sqr(r) == a;
  return r;
}

template <int NBYTES>
NMSM_HD void words_from_be_bytes(uint32_t* w, const uint8_t* b) {  // big-endian integer -> little-endian words
  for (int k = 0; k < NBYTES / 4; k++) {
    const uint8_t* q = b + NBYTES - 4 * (k + 1);
    w[k] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | (uint32_t)q[3];
  }
}

// SEC1 compressed, 1 + 4 LIMBS bytes: 02/03 || x, y = sqrt(x^3 + a x + b) with the prefix's parity, for a prime field
// with p = 3 (mod 4) (secp256k1 and P-256: 33 B; P-384: 49 B).  status: 0 = invalid encoding, 1 = affine point written,
// 2 = point at infinity ((0,0) written)
template <class Cv>
NMSM_HD int sec1_decode_compressed(const uint8_t* enc, uint32_t* out_xy) {
  using F = typename Cv::G::Field;
  constexpr int L = F::LIMBS;
  const uint8_t head = enc[0];
  if (head != 0x02 && head != 0x03) return 0;
  uint32_t xw[L];
  words_from_be_bytes<4 * L>(xw, enc + 1);
  if (!F::canonical_in_range(xw)) return 0;  // Fp.fromBytes rejects x >= p
  const F x = F::from_canonical(xw);
  F rhs;
  if constexpr (Cv::ID == 0) {  // b from the generated Montgomery constant, not curve_b's conversion of 7
    F b;
    for (int k = 0; k < 8; k++) b.v[k] = Secp256k1Consts::B_MONT(k);
    rhs = sqr(x) * x + b;
  } else {
    rhs = sw_rhs<Cv>(x);
  }
  bool ok;
  F y = fp_sqrt_3mod4(rhs, ok);
  if (!ok) return 0;
  uint32_t yw[L];
  y.to_canonical(yw);
  if (((yw[0] & 1u) != 0) != ((head & 1u) != 0)) {
    y = -y;
    y.to_canonical(yw);
  }
  for (int k = 0; k < L; k++) {
    out_xy[k] = xw[k];
    out_xy[L + k] = yw[k];
  }
  return 1;
}
NMSM_HD int sec1_decode_secp256k1(const uint8_t* enc, uint32_t* out_xy) {
  return sec1_decode_compressed<CurveSecp256k1>(enc, out_xy);
}

// sortBit of a canonical BLS12-381 Fp element (12 words): y is the lexicographically larger root iff 2*y >= p
// (bls12-381.ts:347-352)
NMSM_HD bool bls12_381_sort_bit(const uint32_t* yw) {
  uint32_t d2[12];
  for (int k = 11; k >= 1; k--) d2[k] = (yw[k] << 1) | (yw[k - 1] >> 31);
  d2[0] = yw[0] << 1;  // 2y < 2^382: no overflow
  return !Fp<FpBls381>::canonical_in_range(d2);
}

NMSM_HD int zcash_decode_bls12_381_g1(const uint8_t* enc, uint32_t* out_xy) {
  using F = Fp<FpBls381>;
  const bool compressed = (enc[0] >> 7) & 1, infinity = (enc[0] >> 6) & 1, sort = (enc[0] >> 5) & 1;
  if (!compressed) return 0;                    // this entry point takes the 48-byte compressed form only
  if (compressed && infinity && sort) return 0;  // validateMask: 0xe0
  uint8_t v[48];
  for (int k = 0; k < 48; k++) v[k] = enc[k];
  v[0] &= 0x1f;
  if (infinity) {
    for (int k = 0; k < 48; k++)
      if (v[k]) return 0;  // non-canonical zero
    for (int k = 0; k < 24; k++) out_xy[k] = 0;
    return 2;
  }
  uint32_t xw[12];
  words_from_be_bytes<48>(xw, v);
  if (!F::canonical_in_range(xw)) return 0;
  const F x = F::from_canonical(xw);
  F b;
  for (int k = 0; k < 12; k++) b.v[k] = Bls381G1Consts::B_MONT(k);
  bool ok;
  F y = fp_sqrt_3mod4<FpBls381>(sqr(x) * x + b, ok);
  if (!ok) return 0;
  uint32_t yw[12];
  y.to_canonical(yw);
  if (bls12_381_sort_bit(yw) != sort) {
    y = -y;
    y.to_canonical(yw);
  }
  for (int k = 0; k < 12; k++) {
    out_xy[k] = xw[k];
    out_xy[12 + k] = yw[k];
  }
  return 1;
}

// Square root in Fp2 = Fp[u]/(u^2 + 1), p = 3 (mod 4): the reference's complex method (tower.ts:476-498).  Returns
// false when `n` is not a square; which of the two roots comes back is irrelevant to the caller, the wire format's
// sort bit selects the sign afterwards.
template <class P>
NMSM_HD bool fp2_sqrt(const Fp2<P>& n, Fp2<P>& out) {
  using B = Fp<P>;
  bool ok;
  if (n.c1.is_zero()) {
    B r = fp_sqrt_3mod4<P>(n.c0, ok);  // c0 a residue: (sqrt(c0), 0)
    if (ok) {
      out = Fp2<P>{r, B::zero()};
      return true;
    }
    r = fp_sqrt_3mod4<P>(-n.c0, ok);   // else c0 / (-1) is one: (0, sqrt(-c0))
    out = Fp2<P>{B::zero(), r};
    return ok;
  }
  const B a = fp_sqrt_3mod4<P>(sqr(n.c0) + sqr(n.c1), ok);  // sqrt of the norm c0^2 - c1^2 * (-1)
  if (!ok) return false;
  uint32_t hw[P::N];  // (p + 1) / 2 = 1/2 mod p
  {
    uint32_t t[P::N];
    t[0] = add_cc(P::P(0), 1u);
    for (int k = 1; k < P::N; k++) t[k] = addc_cc(P::P(k), 0u);
    const uint32_t top = addc(0, 0);
    for (int k = 0; k < P::N - 1; k++) hw[k] = (t[k] >> 1) | (t[k + 1] << 31);
    hw[P::N - 1] = (t[P::N - 1] >> 1) | (top << 31);
  }
  const B half = B::from_canonical(hw);
  B d = (a + n.c0) * half;
  B a0 = fp_sqrt_3mod4<P>(d, ok);
  if (!ok) {  // legendre(d) == -1 (tower.ts:489)
    d = d - a;
    a0 = fp_sqrt_3mod4<P>(d, ok);
    if (!ok) return false;
  }
  out = Fp2<P>{a0, n.c1 * half * inv(a0)};
  const Fp2<P> chk = out * out;
  return chk == n;
}

// BLS12-381 G2, 96-byte compressed: x = c1 || c0 big-endian (bls12-381.ts:354-367), flags in the top three bits,
// y = sqrt(x^3 + 4(1 + u)) with the sort bit taken over [y.c1, y.c0] (bls12-381.ts:347-352,488-491).
// out: x.c0, x.c1, y.c0, y.c1 as 12 little-endian words each (the C-ABI packing of a G2 point).
NMSM_HD int zcash_decode_bls12_381_g2(const uint8_t* enc, uint32_t* out_xy) {
  using B = Fp<FpBls381>;
  using F2 = Fp2<FpBls381>;
  const bool compressed = (enc[0] >> 7) & 1, infinity = (enc[0] >> 6) & 1, sort = (enc[0] >> 5) & 1;
  if (!compressed) return 0;                    // this entry point takes the 96-byte compressed form only
  if (compressed && infinity && sort) return 0;  // validateMask: 0xe0
  uint8_t v[96];
  for (int k = 0; k < 96; k++) v[k] = enc[k];
  v[0] &= 0x1f;
  if (infinity) {
    for (int k = 0; k < 96; k++)
      if (v[k]) return 0;  // non-canonical zero
    for (int k = 0; k < 48; k++) out_xy[k] = 0;
    return 2;
  }
  uint32_t xw[24];
  words_from_be_bytes<48>(xw + 12, v);      // c1 comes first on the wire
  words_from_be_bytes<48>(xw, v + 48);      // then c0
  if (!B::canonical_in_range(xw) || !B::canonical_in_range(xw + 12)) return 0;
  const F2 x = F2::from_canonical(xw);
  uint32_t four[12] = {4, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  const B b4 = B::from_canonical(four);
  const F2 rhs = x * x * x + F2{b4, b4};
  F2 y;
  if (!fp2_sqrt<FpBls381>(rhs, y)) return 0;
  uint32_t yw[24];
  y.to_canonical(yw);
  // sortBit over [c1, c0]: the first non-zero part decides, larger iff 2 * part >= p
  const uint32_t* part = yw + 12;
  bool c1_zero = true;
  for (int k = 0; k < 12; k++) c1_zero &= (yw[12 + k] == 0);
  if (c1_zero) part = yw;
  uint32_t d2[12];
  for (int k = 11; k >= 1; k--) d2[k] = (part[k] << 1) | (part[k - 1] >> 31);
  d2[0] = part[0] << 1;
  bool all_zero = true;
  for (int k = 0; k < 12; k++) all_zero &= (part[k] == 0);
  const bool larger = !all_zero && !B::canonical_in_range(d2);
  if (larger != sort) {
    y = -y;
    y.to_canonical(yw);
  }
  for (int k = 0; k < 24; k++) {
    out_xy[k] = xw[k];
    out_xy[24 + k] = yw[k];
  }
  return 1;
}

// zip215 = false: the reference's default `fromBytes(bytes, zip215 = false)` (edwards.ts:405-436): y must be < p and
// x = 0 with the sign bit set is rejected; zip215 = true: the ZIP-215 acceptance rules ed25519.verify uses by default.
NMSM_HD int ed25519_decode(const uint8_t* enc, uint32_t* out_xy, bool zip215 = false) {
  return ed_decompress(enc, out_xy, zip215) ? 1 : 0;
}

}  // namespace nmsm
