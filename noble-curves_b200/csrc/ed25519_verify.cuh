// Ed25519 batch verification front/back end (SURVEY §8 row f1, "next" after the MSM path).
//
// The reference has NO batch verification (SURVEY §3.4); it verifies one signature at a time:
//   /root/reference/src/abstract/edwards.ts:942-989  verify(): decode A, R (fromBytes :405-436, ZIP-215 by
//   default for ed25519, src/ed25519.ts:168), 0 <= s < l, k = SHA-512(R || A || M) mod l (:900-906),
//   accept iff [8](R + k*A - s*B) == O.
// Batch form (random 128-bit z_i from the caller):
//   [8]( sum z_i*R_i + sum (z_i*k_i mod l)*A_i - (sum z_i*s_i mod l)*B ) == O
// which holds for every z iff every individual equation holds (and with probability <= 2^-128 otherwise),
// so parity is defined as: batch accepts <=> every individual reference verify accepts.
//
// Pieces (thread bodies are host/device like msm_body.cuh so tests/hostemu can run them):
//   ed_decompress      RFC 8032 5.1.3 + uvRatio (src/ed25519.ts:104-121), ZIP-215 acceptance rules
//   sha512_rAM         SHA-512 over R || A || M
//   ed_terms_body      per signature: k, z*k mod l, z*s mod l (Montgomery arithmetic mod l), s < l check
//   k_ed_finish        c = -(sum z*s) mod l, appends (c, B)
// followed by the generic Edwards MSM of 2n+1 terms and a cofactor-clearing identity check.
#pragma once
#include "msm_body.cuh"

namespace nmsm {

using EdF = Fp<FpEd25519>;
using EdS = Fp<FnEd25519Mod>;

// x^(2^252 - 3) (the (p-5)/8 power), addition chain of src/ed25519.ts:66-98 `ed25519_pow_2_252_3`
NMSM_HD EdF ed_pow_p58(const EdF& x) {
  auto sqn = [](EdF v, int n) {
    for (int i = 0; i < n; i++) v = sqr(v);
    return v;
  };
  EdF x2 = sqr(x);
  EdF b2 = x2 * x;               // x^3
  EdF b4 = sqn(b2, 2) * b2;      // x^(2^4 - 1)
  EdF b5 = sqr(b4) * x;          // x^(2^5 - 1)
  EdF b10 = sqn(b5, 5) * b5;
  EdF b20 = sqn(b10, 10) * b10;
  EdF b40 = sqn(b20, 20) * b20;
  EdF b80 = sqn(b40, 40) * b40;
  EdF b160 = sqn(b80, 80) * b80;
  EdF b240 = sqn(b160, 80) * b80;
  EdF b250 = sqn(b240, 10) * b10;
  return sqn(b250, 2) * x;       // x^(2^252 - 3)
}

NMSM_HD EdF ed_d() {
  EdF r;
  for (int k = 0; k < 8; k++) r.v[k] = Ed25519Consts::D_MONT(k);
  return r;
}
NMSM_HD EdF ed_sqrt_m1() {
  EdF r;
  for (int k = 0; k < 8; k++) r.v[k] = Ed25519Consts::SQRT_M1_MONT(k);
  return r;
}

// Point.fromBytes(bytes, zip215) (edwards.ts:405-436).  zip215 = true: any 255-bit y is accepted and reduced,
// x = 0 with the sign bit set is accepted (what ed25519.verify decodes with by default, ed25519.ts:168).
// zip215 = false (RFC 8032 / the reference's fromBytes default): y >= p is rejected (`aInRange('point.y', y, 0, p)`
// :421) and so is x = 0 with the sign bit set (:431-433).  Writes canonical (x, y) little-endian words; false if
// rejected or y^2 - 1 / (d y^2 + 1) is not a square.
NMSM_HD bool ed_decompress(const uint8_t* enc, uint32_t* out_xy, bool zip215 = true) {
  uint32_t yw[8];
  for (int k = 0; k < 8; k++)
    yw[k] = (uint32_t)enc[4 * k] | ((uint32_t)enc[4 * k + 1] << 8) | ((uint32_t)enc[4 * k + 2] << 16) |
            ((uint32_t)enc[4 * k + 3] << 24);
  const bool sign = (yw[7] >> 31) != 0;
  yw[7] &= 0x7fffffffu;
  if (!EdF::canonical_in_range(yw)) {  // y in [p, 2^255): reduce (ZIP-215 allows unreduced encodings)
    if (!zip215) return false;
    yw[0] = sub_cc(yw[0], FpEd25519::P(0));
    for (int k = 1; k < 8; k++) yw[k] = subc_cc(yw[k], FpEd25519::P(k));
  }
  const EdF one = EdF::one();
  const EdF y = EdF::from_canonical(yw);
  const EdF y2 = sqr(y);
  const EdF u = y2 - one;
  const EdF v = ed_d() * y2 + one;  // d*y^2 - a, a = -1
  // uvRatio
  const EdF v3 = sqr(v) * v;
  const EdF v7 = sqr(v3) * v;
  const EdF pw = ed_pow_p58(u * v7);
  EdF x = u * v3 * pw;
  const EdF vx2 = v * sqr(x);
  const EdF sqrt_m1 = ed_sqrt_m1();
  const EdF neg_u = -u;
  const bool use1 = vx2 == u;
  const bool use2 = vx2 == neg_u;
  const bool no_root = vx2 == neg_u * sqrt_m1;
  if (use2 || no_root) x = x * sqrt_m1;
  if (!(use1 || use2)) return false;
  uint32_t xc[8];
  x.to_canonical(xc);
  bool x_odd = (xc[0] & 1u) != 0;
  if (x_odd) {  // isNegativeLE -> take the even root
    x = -x;
    x.to_canonical(xc);
    x_odd = (xc[0] & 1u) != 0;  // false unless x == 0 (then still false)
  }
  if (!zip215 && sign && x.is_zero()) return false;  // edwards.ts:431-433 "bad point: x=0 and x_0=1"
  if (sign != x_odd) {
    x = -x;
    x.to_canonical(xc);
  }
  for (int k = 0; k < 8; k++) {
    out_xy[k] = xc[k];
    out_xy[8 + k] = yw[k];
  }
  return true;
}

// ---- SHA-512 -----------------------------------------------------------------------------------
NMSM_HD uint64_t sha512_k(int i) {
  constexpr uint64_t K[80] = {
      0x428a2f98d728ae22ULL, 0x7137449123ef65cdULL, 0xb5c0fbcfec4d3b2fULL, 0xe9b5dba58189dbbcULL, 0x3956c25bf348b538ULL,
      0x59f111f1b605d019ULL, 0x923f82a4af194f9bULL, 0xab1c5ed5da6d8118ULL, 0xd807aa98a3030242ULL, 0x12835b0145706fbeULL,
      0x243185be4ee4b28cULL, 0x550c7dc3d5ffb4e2ULL, 0x72be5d74f27b896fULL, 0x80deb1fe3b1696b1ULL, 0x9bdc06a725c71235ULL,
      0xc19bf174cf692694ULL, 0xe49b69c19ef14ad2ULL, 0xefbe4786384f25e3ULL, 0x0fc19dc68b8cd5b5ULL, 0x240ca1cc77ac9c65ULL,
      0x2de92c6f592b0275ULL, 0x4a7484aa6ea6e483ULL, 0x5cb0a9dcbd41fbd4ULL, 0x76f988da831153b5ULL, 0x983e5152ee66dfabULL,
      0xa831c66d2db43210ULL, 0xb00327c898fb213fULL, 0xbf597fc7beef0ee4ULL, 0xc6e00bf33da88fc2ULL, 0xd5a79147930aa725ULL,
      0x06ca6351e003826fULL, 0x142929670a0e6e70ULL, 0x27b70a8546d22ffcULL, 0x2e1b21385c26c926ULL, 0x4d2c6dfc5ac42aedULL,
      0x53380d139d95b3dfULL, 0x650a73548baf63deULL, 0x766a0abb3c77b2a8ULL, 0x81c2c92e47edaee6ULL, 0x92722c851482353bULL,
      0xa2bfe8a14cf10364ULL, 0xa81a664bbc423001ULL, 0xc24b8b70d0f89791ULL, 0xc76c51a30654be30ULL, 0xd192e819d6ef5218ULL,
      0xd69906245565a910ULL, 0xf40e35855771202aULL, 0x106aa07032bbd1b8ULL, 0x19a4c116b8d2d0c8ULL, 0x1e376c085141ab53ULL,
      0x2748774cdf8eeb99ULL, 0x34b0bcb5e19b48a8ULL, 0x391c0cb3c5c95a63ULL, 0x4ed8aa4ae3418acbULL, 0x5b9cca4f7763e373ULL,
      0x682e6ff3d6b2b8a3ULL, 0x748f82ee5defb2fcULL, 0x78a5636f43172f60ULL, 0x84c87814a1f0ab72ULL, 0x8cc702081a6439ecULL,
      0x90befffa23631e28ULL, 0xa4506cebde82bde9ULL, 0xbef9a3f7b2c67915ULL, 0xc67178f2e372532bULL, 0xca273eceea26619cULL,
      0xd186b8c721c0c207ULL, 0xeada7dd6cde0eb1eULL, 0xf57d4f7fee6ed178ULL, 0x06f067aa72176fbaULL, 0x0a637dc5a2c898a6ULL,
      0x113f9804bef90daeULL, 0x1b710b35131c471bULL, 0x28db77f523047d84ULL, 0x32caab7b40c72493ULL, 0x3c9ebe0a15c9bebcULL,
      0x431d67c49c100d4cULL, 0x4cc5d4becb3e42b6ULL, 0x597f299cfc657e2aULL, 0x5fcb6fab3ad6faecULL, 0x6c44198c4a475817ULL};
  return K[i];
}
NMSM_HD uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

// One SHA-512 compression (FIPS 180-4 §6.4.2): st <- st + the 80 rounds over the block w[16] (big-endian 64-bit words;
// w is overwritten).  SHA-512 and SHA-384 share it.
NMSM_HD void sha512_compress(uint64_t* st, uint64_t* w) {
  uint64_t a = st[0], bb = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
  for (int i = 0; i < 80; i++) {
    if (i >= 16) {
      const uint64_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
      const uint64_t s0 = rotr64(w15, 1) ^ rotr64(w15, 8) ^ (w15 >> 7);
      const uint64_t s1 = rotr64(w2, 19) ^ rotr64(w2, 61) ^ (w2 >> 6);
      w[i & 15] = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
    }
    const uint64_t S1 = rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41);
    const uint64_t ch = (e & f) ^ (~e & g);
    const uint64_t t1 = h + S1 + ch + sha512_k(i) + w[i & 15];
    const uint64_t S0 = rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39);
    const uint64_t mj = (a & bb) ^ (a & c) ^ (bb & c);
    const uint64_t t2 = S0 + mj;
    h = g; g = f; f = e; e = d + t1; d = c; c = bb; bb = a; a = t1 + t2;
  }
  st[0] += a; st[1] += bb; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// SHA-512(R || A || M); digest as 64 bytes little-endian-interpretable words out[0..15] (u32, byte order of the digest)
NMSM_HD void sha512_rAM(const uint8_t* r32, const uint8_t* a32, const uint8_t* msg, uint64_t mlen, uint8_t* digest) {
  uint64_t st[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                    0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
  const uint64_t total = 64 + mlen;
  const uint64_t nblocks = (total + 1 + 16 + 127) / 128;
  auto byte_at = [&](uint64_t j) -> uint32_t {  // j-th byte of the padded message
    if (j < 32) return r32[j];
    if (j < 64) return a32[j - 32];
    if (j < total) return msg[j - 64];
    if (j == total) return 0x80u;
    const uint64_t end = nblocks * 128;
    if (j >= end - 8) return (uint32_t)(((total * 8) >> (8 * (end - 1 - j))) & 0xff);  // 128-bit length, high half zero
    return 0u;
  };
  for (uint64_t b = 0; b < nblocks; b++) {
    uint64_t w[16];
    for (int i = 0; i < 16; i++) {
      uint64_t x = 0;
      for (int k = 0; k < 8; k++) x = (x << 8) | byte_at(b * 128 + 8 * i + k);
      w[i] = x;
    }
    sha512_compress(st, w);
  }
  for (int i = 0; i < 8; i++)
    for (int k = 0; k < 8; k++) digest[8 * i + k] = (uint8_t)(st[i] >> (56 - 8 * k));
}

// SHA-384(msg[0..len)) -> out[48], the digest's byte order: SHA-512's compression from the FIPS 180-4 §5.3.4 initial
// value, truncated to the first six state words (the P-384 ECDSA prehash, ecdsa_verify.cuh)
NMSM_HD void sha384(const uint8_t* msg, uint64_t len, uint8_t* out) {
  uint64_t st[8] = {0xcbbb9d5dc1059ed8ULL, 0x629a292a367cd507ULL, 0x9159015a3070dd17ULL, 0x152fecd8f70e5939ULL,
                    0x67332667ffc00b31ULL, 0x8eb44a8768581511ULL, 0xdb0c2e0d64f98fa7ULL, 0x47b5481dbefa4fa4ULL};
  const uint64_t nblocks = (len + 1 + 16 + 127) / 128;
  const uint64_t end = nblocks * 128;
  auto byte_at = [&](uint64_t j) -> uint32_t {  // j-th byte of the padded message
    if (j < len) return msg[j];
    if (j == len) return 0x80u;
    if (j >= end - 8) return (uint32_t)(((len * 8) >> (8 * (end - 1 - j))) & 0xff);  // 128-bit length, high half zero
    return 0u;
  };
  for (uint64_t b = 0; b < nblocks; b++) {
    uint64_t w[16];
    for (int i = 0; i < 16; i++) {
      uint64_t x = 0;
      for (int k = 0; k < 8; k++) x = (x << 8) | byte_at(b * 128 + 8 * i + k);
      w[i] = x;
    }
    sha512_compress(st, w);
  }
  for (int i = 0; i < 6; i++)
    for (int k = 0; k < 8; k++) out[8 * i + k] = (uint8_t)(st[i] >> (56 - 8 * k));
}

NMSM_HD void words_from_le_bytes(uint32_t* w, const uint8_t* b, int nwords) {
  for (int k = 0; k < nwords; k++)
    w[k] = (uint32_t)b[4 * k] | ((uint32_t)b[4 * k + 1] << 8) | ((uint32_t)b[4 * k + 2] << 16) | ((uint32_t)b[4 * k + 3] << 24);
}

// Montgomery form (mod l) of an arbitrary 256-bit integer
NMSM_HD EdS eds_to_mont(const uint32_t* x) {
  EdS a, r2;
  for (int k = 0; k < 8; k++) {
    a.v[k] = x[k];
    r2.v[k] = FnEd25519Mod::R2(k);
  }
  return a * r2;
}

// k = SHA-512(R || A || M) mod l in Montgomery form, over the signature's R bytes and the key bytes as given (not
// re-encoded: ZIP-215 accepts non-canonical encodings, and the hash must see them as sent)
NMSM_HD EdS ed_challenge(const uint8_t* r32, const uint8_t* a32, const uint8_t* msg, uint64_t mlen) {
  uint8_t digest[64];
  sha512_rAM(r32, a32, msg, mlen, digest);
  uint32_t lo[8], hi[8];
  words_from_le_bytes(lo, digest, 8);  // k = little-endian integer of the 64-byte digest (edwards.ts:867)
  words_from_le_bytes(hi, digest + 32, 8);
  EdS r2;
  for (int k = 0; k < 8; k++) r2.v[k] = FnEd25519Mod::R2(k);
  return eds_to_mont(lo) + eds_to_mont(hi) * r2;  // (lo + hi * 2^256) mod l
}

// Per-signature scalars.  Layout of the MSM that follows (2n+1 terms):
//   points  [0,n) = R_i   [n,2n) = A_i   [2n] = B
//   scalars [0,n) = z_i   [n,2n) = z_i*k_i mod l   [2n] = -(sum z_i*s_i) mod l
// bad[0] receives the smallest index whose signature cannot be accepted individually
// (undecodable R or A, or s >= l): edwards.ts:963-971 returns false for those.
NMSM_HD void ed_terms_body(uint32_t i, uint32_t n, const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs,
                           const uint64_t* msg_off, const uint8_t* z16, uint32_t* pts, uint32_t* scalars,
                           uint32_t* zs_mont, unsigned int* bad) {
  const uint8_t* sig = sigs + (size_t)i * 64;
  const uint8_t* pk = pks + (size_t)i * 32;
  bool ok = ed_decompress(sig, pts + (size_t)i * 16);
  ok = ed_decompress(pk, pts + (size_t)(n + i) * 16) && ok;
  uint32_t s[8];
  words_from_le_bytes(s, sig + 32, 8);
  if (!EdS::canonical_in_range(s)) ok = false;  // s >= l (multiplyUnsafe range check, edwards.ts:573)
  if (!ok) {
    atomic_min_u32(&bad[0], i);
    for (int k = 0; k < 8; k++) zs_mont[(size_t)i * 8 + k] = 0;  // keep the rest of the batch well-defined
    for (int k = 0; k < 16; k++) {  // identity points, zero scalars
      pts[(size_t)i * 16 + k] = (k == 8) ? 1u : 0u;
      pts[(size_t)(n + i) * 16 + k] = (k == 8) ? 1u : 0u;
    }
    for (int k = 0; k < 8; k++) scalars[(size_t)i * 8 + k] = scalars[(size_t)(n + i) * 8 + k] = 0;
    return;
  }
  const EdS k_m = ed_challenge(sig, pk, msgs + msg_off[i], msg_off[i + 1] - msg_off[i]);
  uint32_t z[8];
  words_from_le_bytes(z, z16 + (size_t)i * 16, 4);
  for (int k = 4; k < 8; k++) z[k] = 0;
  const EdS z_m = eds_to_mont(z);
  const EdS zk = z_m * k_m;
  const EdS zs = z_m * eds_to_mont(s);
  uint32_t zk_c[8];
  zk.to_canonical(zk_c);
  for (int k = 0; k < 8; k++) {
    scalars[(size_t)i * 8 + k] = z[k];
    scalars[(size_t)(n + i) * 8 + k] = zk_c[k];
    zs_mont[(size_t)i * 8 + k] = zs.v[k];
  }
}

// c = -(sum_i zs_i) mod l and the base-point term; serial statement (the kernel strides + tree-reduces)
NMSM_HD void ed_finish_serial(uint32_t n, const uint32_t* zs_mont, uint32_t* pts, uint32_t* scalars) {
  EdS acc = EdS::zero();
  for (uint32_t i = 0; i < n; i++) {
    EdS t;
    for (int k = 0; k < 8; k++) t.v[k] = zs_mont[(size_t)i * 8 + k];
    acc = acc + t;
  }
  acc = -acc;
  uint32_t c[8];
  acc.to_canonical(c);
  for (int k = 0; k < 8; k++) {
    scalars[(size_t)(2 * n) * 8 + k] = c[k];
    pts[(size_t)(2 * n) * 16 + k] = Ed25519Consts::GX(k);
    pts[(size_t)(2 * n) * 16 + 8 + k] = Ed25519Consts::GY(k);
  }
}

// ---- one verdict per signature (nmsm_ed25519_verify_each) ------------------------------------------------------
// The batch equation above answers for the whole batch; a caller holding signatures from untrusted senders needs to
// know WHICH one fails.  Per signature, as edwards.ts:942-989 states it:
//   ed_verify_prepare_body  decode A and R, s < l, (strict) [8]A != O, k = SHA-512(R || A || M) mod l
//   ed_verify_check_body    [8](s B - k A - R) == O: s B from the fixed-point table of B, k A by 4-bit signed windows
// Two kernels (inst_ed25519.cu), as for ECDSA: the SHA-512 and square-root state stays out of the scalar
// multiplication's registers.  No inversion: the identity test works on projective coordinates.
static constexpr int ED_VERIFY_STRICT = 1;  // include/nmsm.h NMSM_ED25519_VERIFY_STRICT

// [8]P == O for canonical affine (x, y): the strict mode's small-order test of A (verify's `!zip215 && A.isSmallOrder()`)
NMSM_HD bool ed_small_order(const uint32_t* xy) {
  using G = CurveEd25519::G;
  G::Acc p = G::from_affine(G::prepare(xy));
  for (int j = 0; j < 3; j++) nl_dbl<G>(p);
  return G::is_identity(p);
}

// Signature i: A, R (canonical affine words), s and k (canonical words mod l), and the prepare verdict in ok_out[i].
// flags & ED_VERIFY_STRICT: RFC 8032 decoding and small-order A rejected ({ zip215: false }); else ZIP-215 decoding.
NMSM_HD void ed_verify_prepare_body(uint32_t i, const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs,
                                    const uint64_t* msg_off, int flags, uint32_t* as, uint32_t* rs, uint32_t* ss,
                                    uint32_t* ks, uint8_t* ok_out) {
  const uint8_t* sig = sigs + (size_t)i * 64;
  const uint8_t* pk = pks + (size_t)i * 32;
  const bool zip215 = (flags & ED_VERIFY_STRICT) == 0;
  uint32_t a[16], r[16], s[8];
  bool ok = ed_decompress(pk, a, zip215);
  ok = ed_decompress(sig, r, zip215) && ok;
  words_from_le_bytes(s, sig + 32, 8);
  ok = ok && EdS::canonical_in_range(s);  // s >= l is false; s = 0 is allowed (multiplyUnsafe, edwards.ts:573)
  if (ok && !zip215 && ed_small_order(a)) ok = false;
  ok_out[i] = ok ? 1 : 0;
  if (!ok) return;
  uint32_t k[8];
  ed_challenge(sig, pk, msgs + msg_off[i], msg_off[i + 1] - msg_off[i]).to_canonical(k);
  store_words<16>(as + (size_t)i * 16, a);
  store_words<16>(rs + (size_t)i * 16, r);
  store_words<8>(ss + (size_t)i * 8, s);
  store_words<8>(ks + (size_t)i * 8, k);
}

// Signature i after the prepare: out_ok[i] = [8](s B - k A - R) == O, the cofactored equation of both modes.
// tbl: the fixed-point table of B (table_mul_body layout, BITS-bit digits; BITS is a parameter only so that
// tests/hostemu can use a small table).
template <int BITS = PT_BITS>
NMSM_HD void ed_verify_check_body(uint32_t i, const uint32_t* tbl, const uint32_t* as, const uint32_t* rs,
                                  const uint32_t* ss, const uint32_t* ks, uint8_t* out_ok, unsigned int* err) {
  using Cv = CurveEd25519;
  using G = Cv::G;
  if (!out_ok[i]) return;
  G::Acc acc;
  table_mul_body<Cv, BITS>(i, tbl, ss, 1, acc, err);  // s < l always; s = 0 gives O
  uint32_t a[16], r[16], k[8];
  load_words<16>(a, as + (size_t)i * 16);
  load_words<16>(r, rs + (size_t)i * 16);
  load_words<8>(k, ks + (size_t)i * 8);
  nl_add<G>(acc, scalar_mul_acc<Cv>(G::neg(G::prepare(a)), k));  // complete formulas: any A, including small order
  nl_madd<G>(acc, G::neg(G::prepare(r)));
  for (int j = 0; j < 3; j++) nl_dbl<G>(acc);
  out_ok[i] = G::is_identity(acc) ? 1 : 0;
}

// serial statements of k_ed_verify_prepare / k_ed_verify_check
NMSM_HD void ed_verify_prepare_serial(uint32_t n, const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs,
                                      const uint64_t* msg_off, int flags, uint32_t* as, uint32_t* rs, uint32_t* ss,
                                      uint32_t* ks, uint8_t* ok_out) {
  for (uint32_t i = 0; i < n; i++) ed_verify_prepare_body(i, sigs, pks, msgs, msg_off, flags, as, rs, ss, ks, ok_out);
}
template <int BITS = PT_BITS>
NMSM_HD void ed_verify_check_serial(uint32_t n, const uint32_t* tbl, const uint32_t* as, const uint32_t* rs,
                                    const uint32_t* ss, const uint32_t* ks, uint8_t* out_ok, unsigned int* err) {
  for (uint32_t i = 0; i < n; i++) ed_verify_check_body<BITS>(i, tbl, as, rs, ss, ks, out_ok, err);
}

}  // namespace nmsm
