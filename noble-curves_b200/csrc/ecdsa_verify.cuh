// ECDSA batch verification for secp256k1 (SURVEY §8 row f5), P-256 and P-384: one independent verdict per signature.
//
// The reference verifies one signature at a time: weierstrass.ts `ecdsa().verify` (noble-curves v2), with
// format 'compact' and the options { prehash, lowS } (both default true for secp256k1; p256 and p384 default to lowS
// false).  For a curve with W-word field elements and scalars (W = 8, or 12 for P-384):
//   sig = r || s (8W B, big-endian); inside the reference's try (any failure = false):
//   1 <= r, s < n;  P = Point.fromBytes(publicKey)  (1 + 4W B 02/03 + sqrt, or 1 + 8W B 04 + curve equation);
//   lowS && s > n/2 -> false;  h = bits2int_modN(prehash ? hash(msg) : msg)  (SHA-256, or SHA-384 for P-384;
//   bits2int takes the first min(len, 4W) bytes, and throws above 8192 bytes);
//   w = s^-1,  u1 = h w,  u2 = r w  (mod n);  R = u1 G + u2 P;  R == O -> false;  accept iff R.x mod n == r.
// ECDSA has no batch equation (R's y is not in the signature), so the batch is data-parallel: per signature
//   ecdsa_prepare_body  parse + range checks, lowS, key decode, prehash, bits2int mod n
//   (kernel)            s^-1 through one warp-shared inversion per 32 signatures (msm.cuh warp_batch_inverse)
//   ecdsa_store         u1, u2
//   ecdsa_check_body    u1 G from the fixed-point table of G (table_mul_body), u2 Q (scalar_mul_acc: GLV on
//                       secp256k1, plain windows on P-256 and P-384), complete addition, and the x comparison in
//                       XYZZ coordinates without an inversion.
// The two halves run as two kernels (inst_secp256k1.cu, inst_p256.cu, inst_p384.cu) so the hash / square-root state
// stays out of the scalar multiplication's registers.  Bodies are host/device so tests/hostemu can run them.  They are
// templates on the curve policy (CurveSecp256k1 by default, CurveP256 or CurveP384); what differs per curve is the
// group and its width, the scalar modulus n and the prehash (EcdsaScalar) and the SEC1 key decoders.
#pragma once
#include "codec.cuh"
#include "validate.cuh"

namespace nmsm {

static constexpr int ECDSA_PREHASH = 1;  // include/nmsm.h NMSM_ECDSA_PREHASH
static constexpr int ECDSA_LOW_S = 2;    // include/nmsm.h NMSM_ECDSA_LOW_S
static constexpr uint64_t ECDSA_MAX_RAW_MSG = 8192;  // bits2int: "input is too large" above this many bytes

// ---- SHA-256 (FIPS 180-4) ---------------------------------------------------------------------
NMSM_HD uint32_t sha256_k(int i) {
  constexpr uint32_t K[64] = {
      0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
      0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
      0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
      0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
      0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
      0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
      0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
      0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};
  return K[i];
}
NMSM_HD uint32_t rotr32(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

// One SHA-256 compression: st <- st + the 64 rounds over the block w[16] (big-endian words; w is overwritten).
NMSM_HD void sha256_compress(uint32_t* st, uint32_t* w) {
  uint32_t a = st[0], bb = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
  for (int i = 0; i < 64; i++) {
    if (i >= 16) {
      const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
      const uint32_t s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
      const uint32_t s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
      w[i & 15] = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
    }
    const uint32_t S1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
    const uint32_t ch = (e & f) ^ (~e & g);
    const uint32_t t1 = h + S1 + ch + sha256_k(i) + w[i & 15];
    const uint32_t S0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
    const uint32_t mj = (a & bb) ^ (a & c) ^ (bb & c);
    const uint32_t t2 = S0 + mj;
    h = g; g = f; f = e; e = d + t1; d = c; c = bb; bb = a; a = t1 + t2;
  }
  st[0] += a; st[1] += bb; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// Finish a SHA-256 whose first `done` bytes (a multiple of 64) are already compressed into st: absorb the `len` bytes
// byte_at(0 .. len), pad for a total of done + len bytes, and write the digest (its byte order) to out[32].
template <class ByteAt>
NMSM_HD void sha256_finish(uint32_t* st, uint64_t done, uint64_t len, const ByteAt& byte_at, uint8_t* out) {
  const uint64_t nblocks = (len + 1 + 8 + 63) / 64;
  const uint64_t end = nblocks * 64, bits = (done + len) * 8;
  auto padded = [&](uint64_t j) -> uint32_t {  // j-th byte of the padded tail
    if (j < len) return byte_at(j);
    if (j == len) return 0x80u;
    if (j >= end - 8) return (uint32_t)((bits >> (8 * (end - 1 - j))) & 0xff);  // 64-bit big-endian bit length
    return 0u;
  };
  for (uint64_t b = 0; b < nblocks; b++) {
    uint32_t w[16];
    for (int i = 0; i < 16; i++) {
      uint32_t x = 0;
      for (int k = 0; k < 4; k++) x = (x << 8) | padded(b * 64 + 4 * i + k);
      w[i] = x;
    }
    sha256_compress(st, w);
  }
  for (int i = 0; i < 8; i++)
    for (int k = 0; k < 4; k++) out[4 * i + k] = (uint8_t)(st[i] >> (24 - 8 * k));
}

// SHA-256(msg[0..len)) -> out[32], the digest's byte order
NMSM_HD void sha256(const uint8_t* msg, uint64_t len, uint8_t* out) {
  uint32_t st[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
  sha256_finish(st, 0, len, [&](uint64_t j) -> uint32_t { return msg[j]; }, out);
}

// The per-curve ECDSA policy: the scalar modulus n (s^-1, u1, u2 mod n) and the prehash with its digest length
template <class Cv>
struct EcdsaScalar;
template <>
struct EcdsaScalar<CurveSecp256k1> {
  using Mod = FnSecp256k1Mod;
  static constexpr int DIGEST_BYTES = 32;
  NMSM_HD static void prehash(const uint8_t* m, uint64_t len, uint8_t* out) { sha256(m, len, out); }
};
template <>
struct EcdsaScalar<CurveP256> {
  using Mod = FnP256Mod;
  static constexpr int DIGEST_BYTES = 32;
  NMSM_HD static void prehash(const uint8_t* m, uint64_t len, uint8_t* out) { sha256(m, len, out); }
};
template <>
struct EcdsaScalar<CurveP384> {
  using Mod = FnP384Mod;
  static constexpr int DIGEST_BYTES = 48;
  NMSM_HD static void prehash(const uint8_t* m, uint64_t len, uint8_t* out) { sha384(m, len, out); }
};
template <class Cv>
using EcdsaS = Fp<typename EcdsaScalar<Cv>::Mod>;
using EcS = EcdsaS<CurveSecp256k1>;
// words of the curve's scalars (r, s, h, u1, u2) and of its field elements (the key's x, y).  Equal on every ECDSA curve
// here (n and p have the same bit length), which lets r be compared with R.x in Fp.
template <class Cv>
NMSM_HD constexpr int ecdsa_sw() { return EcdsaS<Cv>::LIMBS; }
template <class Cv>
NMSM_HD constexpr int ecdsa_fw() { return Cv::G::Field::LIMBS; }

// SEC1 uncompressed, 1 + 8 LIMBS bytes (65 B; 97 B on P-384): 04 || x || y, x < p, y < p, on the curve
// (weierstrass.ts pointFromBytes, `isValidXY`).  (0, 0) is rejected although point_on_curve accepts it as the identity
// encoding: b != 0 on every ECDSA curve.  status as sec1_decode_compressed: 0 = invalid, 1 = affine point written
// (canonical x, y words).
template <class Cv>
NMSM_HD int sec1_decode_uncompressed(const uint8_t* enc, uint32_t* out_xy) {
  constexpr int L = Cv::G::Field::LIMBS;
  if (enc[0] != 0x04) return 0;
  uint32_t xy[2 * L];
  words_from_be_bytes<4 * L>(xy, enc + 1);
  words_from_be_bytes<4 * L>(xy + L, enc + 1 + 4 * L);
  uint32_t any = 0;
  for (int k = 0; k < 2 * L; k++) any |= xy[k];
  if (any == 0 || !point_on_curve<Cv>(xy)) return 0;
  for (int k = 0; k < 2 * L; k++) out_xy[k] = xy[k];
  return 1;
}
NMSM_HD int sec1_decode_secp256k1_uncompressed(const uint8_t* enc, uint32_t* out_xy) {
  return sec1_decode_uncompressed<CurveSecp256k1>(enc, out_xy);
}

template <int W>
NMSM_HD bool words_nonzero(const uint32_t* a) {
  uint32_t t = 0;
  for (int k = 0; k < W; k++) t |= a[k];
  return t != 0;
}
NMSM_HD bool words8_nonzero(const uint32_t* a) { return words_nonzero<8>(a); }
// a > (n >> 1): the high-S test (Signature.hasHighS)
template <class Cv = CurveSecp256k1>
NMSM_HD bool ecdsa_high_s(const uint32_t* s) {
  using Mod = typename EcdsaScalar<Cv>::Mod;
  constexpr int SW = ecdsa_sw<Cv>();
  for (int k = SW - 1; k >= 0; k--) {
    const uint32_t half = (Mod::P(k) >> 1) | (k < SW - 1 ? Mod::P(k + 1) << 31 : 0u);
    if (s[k] != half) return s[k] > half;
  }
  return false;
}

// h = bits2int_modN(prehash ? hash(m) : m) for the message m[0..mlen): the big-endian integer of the first
// min(len, 4 SW) bytes (32, or 48 on P-384: n has 32 SW bits), reduced mod n.  False for a raw message over
// ECDSA_MAX_RAW_MSG bytes (bits2int throws).
template <class Cv = CurveSecp256k1>
NMSM_HD bool ecdsa_msg_hash(const uint8_t* m, uint64_t mlen, int flags, uint32_t* h) {
  using Pol = EcdsaScalar<Cv>;
  using Mod = typename Pol::Mod;
  constexpr int SW = ecdsa_sw<Cv>(), NB = 4 * SW;
  uint8_t digest[Pol::DIGEST_BYTES];
  if (flags & ECDSA_PREHASH) {
    Pol::prehash(m, mlen, digest);
    m = digest;
    mlen = Pol::DIGEST_BYTES;
  } else if (mlen > ECDSA_MAX_RAW_MSG) {
    return false;
  }
  const int take = mlen < NB ? (int)mlen : NB;
  for (int k = 0; k < SW; k++) h[k] = 0;
  for (int j = 0; j < take; j++) {
    const int bit = 8 * (take - 1 - j);
    h[bit >> 5] |= (uint32_t)m[j] << (bit & 31);
  }
  if (!EcdsaS<Cv>::canonical_in_range(h)) {  // h < 2^(32 SW) < 2n: one subtraction reduces it
    h[0] = sub_cc(h[0], Mod::P(0));
    for (int k = 1; k < SW; k++) h[k] = subc_cc(h[k], Mod::P(k));
  }
  return true;
}

// Signature i: r, s, h (SW words each), the public key Q (2 FW canonical affine words) and h = bits2int_modN(m).  False = the reference's
// verify returns false before any scalar multiplication; the outputs are then unspecified.
template <class Cv = CurveSecp256k1>
NMSM_HD bool ecdsa_prepare_body(uint32_t i, const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off,
                                const uint8_t* msgs, const uint64_t* msg_off, int flags, uint32_t* q_xy, uint32_t* r,
                                uint32_t* s, uint32_t* h) {
  constexpr int SW = ecdsa_sw<Cv>(), FW = ecdsa_fw<Cv>();
  const uint8_t* sig = sigs + (size_t)i * (8 * SW);
  words_from_be_bytes<4 * SW>(r, sig);
  words_from_be_bytes<4 * SW>(s, sig + 4 * SW);
  // Signature.fromBytes: 1 <= r < n, 1 <= s < n;  then lowS
  using S = EcdsaS<Cv>;
  if (!words_nonzero<SW>(r) || !S::canonical_in_range(r) || !words_nonzero<SW>(s) || !S::canonical_in_range(s))
    return false;
  if ((flags & ECDSA_LOW_S) && ecdsa_high_s<Cv>(s)) return false;
  // Point.fromBytes
  const uint8_t* pk = pks + pk_off[i];
  const uint64_t pk_len = pk_off[i + 1] - pk_off[i];
  if (pk_len == 1 + 4 * FW) {
    if (sec1_decode_compressed<Cv>(pk, q_xy) != 1) return false;
  } else if (pk_len == 1 + 8 * FW) {
    if (sec1_decode_uncompressed<Cv>(pk, q_xy) != 1) return false;
  } else {
    return false;
  }
  return ecdsa_msg_hash<Cv>(msgs + msg_off[i], msg_off[i + 1] - msg_off[i], flags, h);
}

// Given w = s^-1 (Montgomery form mod n): u1 = h w, u2 = r w, and the per-signature state k_ecdsa_check reads.
// ok_out[i] carries the prepare verdict to the check, which overwrites it with the final one.
template <class Cv = CurveSecp256k1>
NMSM_HD void ecdsa_store(uint32_t i, bool ok, const uint32_t* q_xy, const uint32_t* r, const uint32_t* h,
                         const EcdsaS<Cv>& w, uint32_t* qs, uint32_t* u1s, uint32_t* u2s, uint32_t* rs, uint8_t* ok_out) {
  using S = EcdsaS<Cv>;
  constexpr int SW = ecdsa_sw<Cv>(), FW = ecdsa_fw<Cv>();
  ok_out[i] = ok ? 1 : 0;
  if (!ok) return;
  uint32_t u1[SW], u2[SW];
  (S::from_canonical(h) * w).to_canonical(u1);
  (S::from_canonical(r) * w).to_canonical(u2);
  store_words<2 * FW>(qs + (size_t)i * (2 * FW), q_xy);
  store_words<SW>(u1s + (size_t)i * SW, u1);
  store_words<SW>(u2s + (size_t)i * SW, u2);
  store_words<SW>(rs + (size_t)i * SW, r);
}

// serial statement of k_ecdsa_prepare / k_p256_ecdsa_prepare / k_p384_ecdsa_prepare (one inversion per signature
// instead of one per warp)
template <class Cv = CurveSecp256k1>
NMSM_HD void ecdsa_prepare_serial(uint32_t n, const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off,
                                  const uint8_t* msgs, const uint64_t* msg_off, int flags, uint32_t* qs, uint32_t* u1s,
                                  uint32_t* u2s, uint32_t* rs, uint8_t* ok_out) {
  constexpr int SW = ecdsa_sw<Cv>(), FW = ecdsa_fw<Cv>();
  for (uint32_t i = 0; i < n; i++) {
    uint32_t q[2 * FW], r[SW], s[SW], h[SW];
    const bool ok = ecdsa_prepare_body<Cv>(i, sigs, pks, pk_off, msgs, msg_off, flags, q, r, s, h);
    using S = EcdsaS<Cv>;
    ecdsa_store<Cv>(i, ok, q, r, h, ok ? inv(S::from_canonical(s)) : S::one(), qs, u1s, u2s, rs, ok_out);
  }
}

// R.x mod n == r for R = acc (XYZZ, x = X / ZZ), without an inversion: X == r ZZ, or, when r + n < p (R.x >= n is
// possible because n < p < 2n on every curve here: p - n < 2^128 on the 256-bit curves, < 2^190 on P-384),
// X == (r + n) ZZ.  R = O (ZZ = 0) is false.
template <class Cv = CurveSecp256k1>
NMSM_HD bool ecdsa_x_matches(const typename Cv::G::Acc& acc, const uint32_t* r) {
  using F = typename Cv::G::Field;
  using Mod = typename EcdsaScalar<Cv>::Mod;
  constexpr int W = ecdsa_fw<Cv>();
  static_assert(ecdsa_sw<Cv>() == W, "ecdsa_x_matches: r and R.x must have the same width");
  if (Cv::G::is_identity(acc)) return false;
  if (acc.X == F::from_canonical(r) * acc.ZZ) return true;  // r < n < p
  uint32_t rn[W];
  rn[0] = add_cc(r[0], Mod::P(0));
  for (int k = 1; k < W; k++) rn[k] = addc_cc(r[k], Mod::P(k));
  const uint32_t carry = addc(0, 0);
  if (carry || !F::canonical_in_range(rn)) return false;
  return acc.X == F::from_canonical(rn) * acc.ZZ;
}

// Signature i after ecdsa_store: R = u1 G + u2 Q, out_ok[i] = verdict.  tbl: the fixed-point table of G
// (table_mul_body layout, BITS-bit digits; BITS is a parameter only so that tests/hostemu can use a small table).
// u2 Q: GLV windows on secp256k1, plain 4-bit windows on P-256 and P-384 (scalar_mul_acc).
template <int BITS = PT_BITS, class Cv = CurveSecp256k1>
NMSM_HD void ecdsa_check_body(uint32_t i, const uint32_t* tbl, const uint32_t* qs, const uint32_t* u1s,
                              const uint32_t* u2s, const uint32_t* rs, uint8_t* out_ok, unsigned int* err) {
  using G = typename Cv::G;
  constexpr int SW = ecdsa_sw<Cv>(), FW = ecdsa_fw<Cv>();
  static_assert(scalar_words<typename Cv::Fn>() == SW, "ecdsa_check_body: table_mul_body reads SW-word scalars");
  if (!out_ok[i]) return;
  typename G::Acc acc;
  table_mul_body<Cv, BITS>(i, tbl, u1s, 1, acc, err);  // u1 < n always; u1 = 0 (h = 0 mod n) gives O
  uint32_t q[2 * FW], u2[SW], r[SW];
  load_words<2 * FW>(q, qs + (size_t)i * (2 * FW));
  load_words<SW>(u2, u2s + (size_t)i * SW);
  load_words<SW>(r, rs + (size_t)i * SW);
  nl_add<G>(acc, scalar_mul_acc<Cv>(G::prepare(q), u2));  // complete: doubles when u1 G == u2 Q
  out_ok[i] = ecdsa_x_matches<Cv>(acc, r) ? 1 : 0;
}

template <int BITS = PT_BITS, class Cv = CurveSecp256k1>
NMSM_HD void ecdsa_check_serial(uint32_t n, const uint32_t* tbl, const uint32_t* qs, const uint32_t* u1s,
                                const uint32_t* u2s, const uint32_t* rs, uint8_t* out_ok, unsigned int* err) {
  for (uint32_t i = 0; i < n; i++) ecdsa_check_body<BITS, Cv>(i, tbl, qs, u1s, u2s, rs, out_ok, err);
}

}  // namespace nmsm
