// EIP-4844 KZG proof verification on BLS12-381 (SURVEY §8 row f15): the point-evaluation precompile (0x0A) and
// verify_blob_kzg_proof of the consensus specs (Deneb polynomial-commitments.md), one verdict per item.
//
//   challenge  z = int_be(SHA-256("FSBLOBVERIFY_V1_" || u128_be(4096) || blob || C)) mod r
//   eval       y = f(z) for the blob's 4096 evaluations f_i over the bit-reversed domain w_i = omega^brp(i):
//              f_k when z = w_k, else (z^4096 - 1) / 4096 * sum_i f_i w_i / (z - w_i)
//   check      e(C - y G1, -G2) e(pi, [tau] G2 - z G2) == 1, computed as e(Q, -G2) e(pi, [tau] G2) == 1 with
//              Q = C - y G1 + z pi, so every scalar multiplication is in G1 and both G2 points are fixed per call
//
// k_kzg_challenge runs one thread per blob: SHA-256 cannot be split within one message, so its ~2050 compressions run
// one after another.  k_kzg_eval runs one block per blob and sums the 4096 fractions f_i w_i / d_i (d_i = z - w_i)
// as one fraction num / den, (a/b + c/d) = (a d + c b) / (b d): per lane over its 16 elements, then over the lanes by
// shuffles and shared memory, so the blob costs 5 multiplications per element and ONE inversion, with nothing stored
// per element (Montgomery's batch inversion would need the 4096 prefix products and a back-sweep for the same single
// inversion).  k_kzg_prepare runs one thread per check: decoding with validate_kzg_g1 semantics (the identity
// 0xc0 || 0..0 is allowed, anything else must decode and lie in G1), range checks of z and y, the optional versioned
// hash, and Q; the Miller and final kernels are the BLS pairing checks' (pairing.cuh), two pairs per check.
//
// Bodies are host/device so tests/hostemu can run them; the *_serial statements are what the kernels compute.
#pragma once
#include "ecdsa_verify.cuh"
#include "pairing.cuh"

namespace nmsm {

using KzgFr = Fp<FrBls381>;
using KzgG = CurveBls381G1Any::G;
static constexpr uint32_t KZG_N = 4096;                    // FIELD_ELEMENTS_PER_BLOB
static constexpr uint64_t KZG_BLOB_BYTES = 32ull * KZG_N;  // BYTES_PER_BLOB
static constexpr int KZG_EVAL_THREADS = 256;               // k_kzg_eval: one block per blob
static constexpr int KZG_PER_LANE = KZG_N / KZG_EVAL_THREADS;

// big-endian word at a 4-byte aligned address
NMSM_HD uint32_t kzg_be32(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
  return __byte_perm(*reinterpret_cast<const uint32_t*>(p), 0, 0x0123);
#else
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3];
#endif
}

// a 32-byte big-endian field element at a 4-byte aligned address -> 8 little-endian words
NMSM_HD void kzg_load_fr(uint32_t* w, const uint8_t* b) {
  for (int k = 0; k < 8; k++) w[k] = kzg_be32(b + 28 - 4 * k);
}

NMSM_HD void kzg_store_fr(uint8_t* b, const uint32_t* w) {
  for (int k = 0; k < 8; k++)
    for (int j = 0; j < 4; j++) b[31 - 4 * k - j] = (uint8_t)(w[k] >> (8 * j));
}

// a^e for the exponent's low `bits` bits (e little-endian words)
NMSM_HD KzgFr kzg_pow(const KzgFr& a, const uint32_t* e, int bits) {
  KzgFr r = KzgFr::one();
  for (int b = bits - 1; b >= 0; b--) {
    r = sqr(r);
    if ((e[b >> 5] >> (b & 31)) & 1u) r = r * a;
  }
  return r;
}

// w_i = omega^brp(i) in Montgomery form, omega = 7^((r - 1) / 4096): the spec's bit-reversed domain
NMSM_HD KzgFr kzg_root(uint32_t i) {
  uint32_t e[8], seven[8] = {7, 0, 0, 0, 0, 0, 0, 0};
  for (int k = 0; k < 8; k++) {  // (r - 1) >> 12; the low word of r is 1
    const uint32_t lo = k == 0 ? FrBls381::P(0) - 1u : FrBls381::P(k), hi = k < 7 ? FrBls381::P(k + 1) : 0u;
    e[k] = (lo >> 12) | (hi << 20);
  }
  const KzgFr omega = kzg_pow(KzgFr::from_canonical(seven), e, 243);
  uint32_t j = 0;
  for (int b = 0; b < 12; b++) j |= ((i >> b) & 1u) << (11 - b);
  return kzg_pow(omega, &j, 12);
}

// ---- compute_challenge ------------------------------------------------------------------------------------------
// blob i (4-byte aligned) and its 48-byte commitment -> z as a canonical 32-byte big-endian value
NMSM_HD void kzg_challenge_body(uint32_t i, const uint8_t* blobs, const uint8_t* commitments48, uint8_t* zs32) {
  const uint8_t* blob = blobs + (size_t)i * KZG_BLOB_BYTES;
  const uint8_t* c = commitments48 + (size_t)i * 48;
  uint32_t st[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
  uint32_t w[16];
  // block 0: "FSBLOBVERIFY_V1_", 4096 as 16 big-endian bytes, blob[0, 32); block b: blob[64 b - 32, 64 b + 32)
  constexpr uint32_t HEAD[8] = {0x4653424cu, 0x4f425645u, 0x52494659u, 0x5f56315fu, 0u, 0u, 0u, KZG_N};
  for (int k = 0; k < 8; k++) {
    w[k] = HEAD[k];
    w[8 + k] = kzg_be32(blob + 4 * k);
  }
  sha256_compress(st, w);
  constexpr uint32_t FULL = (uint32_t)((32 + KZG_BLOB_BYTES) / 64);  // 2048 blocks; 32 blob bytes remain
  for (uint32_t b = 1; b < FULL; b++) {
    const uint8_t* p = blob + 64 * (size_t)b - 32;
    for (int k = 0; k < 16; k++) w[k] = kzg_be32(p + 4 * k);
    sha256_compress(st, w);
  }
  const uint8_t* tail = blob + KZG_BLOB_BYTES - 32;
  uint8_t d[32];
  sha256_finish(st, 64ull * FULL, 80, [&](uint64_t j) -> uint32_t { return j < 32 ? tail[j] : c[j - 32]; }, d);
  uint32_t z[8];
  words_from_be_bytes<32>(z, d);
  while (!KzgFr::canonical_in_range(z)) {  // 2^256 < 3 r: at most two subtractions
    z[0] = sub_cc(z[0], FrBls381::P(0));
    for (int k = 1; k < 8; k++) z[k] = subc_cc(z[k], FrBls381::P(k));
  }
  kzg_store_fr(zs32 + (size_t)i * 32, z);
}

// ---- evaluate_polynomial_in_evaluation_form ---------------------------------------------------------------------
struct KzgFrac {
  KzgFr num, den;
};

NMSM_HD KzgFrac kzg_frac_add(const KzgFrac& a, const KzgFrac& b) {
  return KzgFrac{a.num * b.den + b.num * a.den, a.den * b.den};
}

// lane t's elements t + 256 j: the sum of f_i w_i / d_i as one fraction, with a zero d_k (z = w_k) taken as 1 and k
// reported in `hit`; bad when an element is >= r.  roots: the 4096 w_i in Montgomery form (kzg_root).
NMSM_HD KzgFrac kzg_eval_lane(uint32_t t, const uint8_t* blob, const KzgFr& z, const uint32_t* roots, bool& bad,
                              int& hit) {
  KzgFrac s{KzgFr::zero(), KzgFr::one()};
  for (int j = 0; j < KZG_PER_LANE; j++) {
    const uint32_t e = t + KZG_EVAL_THREADS * j;
    uint32_t fw[8];
    kzg_load_fr(fw, blob + 32 * (size_t)e);
    bad |= !KzgFr::canonical_in_range(fw);
    KzgFr w;
    load_words<8>(w.v, roots + 8 * (size_t)e);
    KzgFr d = z - w;
    if (d.is_zero()) {
      hit = (int)e;
      d = KzgFr::one();
    }
    const KzgFr fwi = KzgFr::from_canonical(fw) * w;
    s.num = s.num * d + fwi * s.den;
    s.den = s.den * d;
  }
  return s;
}

// y for the whole blob from the lanes' sum s (or f_hit), written as 32 big-endian bytes with ok = !bad
NMSM_HD void kzg_eval_finish(const uint8_t* blob, const KzgFr& z, const KzgFrac& s, int hit, bool bad, uint8_t* y32,
                             uint8_t* ok) {
  uint32_t y[8];
  if (hit >= 0) {
    kzg_load_fr(y, blob + 32 * (size_t)hit);
  } else {
    KzgFr zn = z;
    for (int k = 0; k < 12; k++) zn = sqr(zn);  // z^4096
    uint32_t w[8] = {KZG_N, 0, 0, 0, 0, 0, 0, 0};
    const KzgFr v = (zn - KzgFr::one()) * s.num * inv(KzgFr::from_canonical(w) * s.den);
    v.to_canonical(y);
  }
  kzg_store_fr(y32, y);
  *ok = bad ? 0 : 1;
}

// serial statement of k_kzg_eval for blob i (the lanes one after another)
NMSM_HD void kzg_eval_serial(uint32_t i, const uint8_t* blobs, const uint8_t* zs32, const uint32_t* roots,
                             uint8_t* ys32, uint8_t* item_ok) {
  const uint8_t* blob = blobs + (size_t)i * KZG_BLOB_BYTES;
  uint32_t zw[8];
  kzg_load_fr(zw, zs32 + (size_t)i * 32);
  const KzgFr z = KzgFr::from_canonical(zw);
  bool bad = false;
  int hit = -1;
  KzgFrac s{KzgFr::zero(), KzgFr::one()};
  for (uint32_t t = 0; t < KZG_EVAL_THREADS; t++) s = kzg_frac_add(s, kzg_eval_lane(t, blob, z, roots, bad, hit));
  kzg_eval_finish(blob, z, s, hit, bad, ys32 + (size_t)i * 32, item_ok + i);
}

// ---- verify_kzg_proof -------------------------------------------------------------------------------------------
// validate_kzg_g1 + decompression: 1 = a point of G1 other than the identity, 2 = the identity 0xc0 || 0..0 (xy = 0),
// 0 = rejected (bad encoding, off the curve, outside G1)
NMSM_HD int kzg_decode_g1(const uint8_t* b48, uint32_t* xy) {
  const int r = zcash_decode_bls12_381_g1(b48, xy);
  return r == 1 && !bls_in_subgroup<CurveBls381G1Any>(xy) ? 0 : r;
}

// the setup point [tau] G2: decodes to a point other than the identity and lies in G2
NMSM_HD bool kzg_setup_body(const uint8_t* g2_96, uint32_t* xy) {
  return zcash_decode_bls12_381_g2(g2_96, xy) == 1 && bls_in_subgroup<CurveBls381G2Any>(xy);
}

// vh == 0x01 || SHA-256(C)[1:]  (kzg_to_versioned_hash)
NMSM_HD bool kzg_versioned_hash_ok(const uint8_t* c48, const uint8_t* vh) {
  uint8_t d[32];
  sha256(c48, 48, d);
  bool ok = vh[0] == 0x01;
  for (int k = 1; k < 32; k++) ok &= vh[k] == d[k];
  return ok;
}

// s xy for an affine point of G1 other than the identity (24 canonical words) and s < r
NMSM_HD_NOINLINE KzgG::Acc kzg_mul(const uint32_t* xy, const uint32_t* s) {
  return scalar_mul_acc<CurveBls381G1Any>(KzgG::prepare(xy), s);
}

// the generator of G1, negated (pairing.cuh bls_neg_g1)
NMSM_HD void kzg_neg_g1(uint32_t* xy) {
  for (int k = 0; k < 24; k++) xy[k] = bls_neg_g1(k);
}

// k_kzg_prepare, check i: item_ok (optional: the blob evaluation's verdict), z and y < r, the versioned hash
// (optional), C and pi through kzg_decode_g1; then q = C - y G1 + z pi and pi's affine words.  false: rejected.
NMSM_HD bool kzg_prepare_body(uint32_t i, const uint8_t* commitments48, const uint8_t* zs32, const uint8_t* ys32,
                              const uint8_t* proofs48, const uint8_t* vhs32, const uint8_t* item_ok, KzgG::Acc& q,
                              uint32_t* pi) {
  if (item_ok && !item_ok[i]) return false;
  uint32_t z[8], y[8];
  words_from_be_bytes<32>(z, zs32 + (size_t)i * 32);
  words_from_be_bytes<32>(y, ys32 + (size_t)i * 32);
  if (!KzgFr::canonical_in_range(z) || !KzgFr::canonical_in_range(y)) return false;
  const uint8_t* c48 = commitments48 + (size_t)i * 48;
  if (vhs32 && !kzg_versioned_hash_ok(c48, vhs32 + (size_t)i * 32)) return false;
  uint32_t c[24];
  const int rc = kzg_decode_g1(c48, c);
  if (rc == 0) return false;
  const int rp = kzg_decode_g1(proofs48 + (size_t)i * 48, pi);
  if (rp == 0) return false;
  uint32_t g[24];
  kzg_neg_g1(g);
  q = kzg_mul(g, y);
  if (rp == 1) nl_add<KzgG>(q, kzg_mul(pi, z));
  if (rc == 1) nl_madd<KzgG>(q, KzgG::prepare(c));
  return true;
}

// the two pairs of check i: 2i = (Q, -G2), 2i + 1 = (pi, [tau] G2), or two identity pairs and pre_ok 0 when rejected.
// zi: 1 / the inversion target of q.  setup_xy: [tau] G2 in the G2 packing (48 words).
NMSM_HD void kzg_store_pairs(uint32_t i, bool ok, const KzgG::Acc& q, const BlsF& zi, const uint32_t* pi,
                             const uint32_t* setup_xy, uint32_t* g1, uint32_t* g2, uint8_t* pre_ok) {
  uint32_t qxy[24], inf;
  KzgG::to_affine_canonical_with_inv(q, zi, qxy, &inf);
  uint32_t* p0 = g1 + (size_t)i * 48;
  uint32_t* q0 = g2 + (size_t)i * 96;
  for (int k = 0; k < 24; k++) {
    p0[k] = ok ? qxy[k] : 0u;
    p0[24 + k] = ok ? pi[k] : 0u;
  }
  for (int k = 0; k < 48; k++) {
    q0[k] = ok ? bls_neg_g2(k) : 0u;
    q0[48 + k] = ok ? setup_xy[k] : 0u;
  }
  pre_ok[i] = ok ? 1 : 0;
}

// serial statement of k_kzg_prepare (one inversion per check instead of one per warp)
NMSM_HD void kzg_prepare_serial(uint32_t n, const uint8_t* commitments48, const uint8_t* zs32, const uint8_t* ys32,
                                const uint8_t* proofs48, const uint8_t* vhs32, const uint8_t* item_ok,
                                const uint32_t* setup_xy, uint32_t* g1, uint32_t* g2, uint8_t* pre_ok) {
  for (uint32_t i = 0; i < n; i++) {
    KzgG::Acc q = KzgG::identity();
    uint32_t pi[24] = {};
    const bool ok = kzg_prepare_body(i, commitments48, zs32, ys32, proofs48, vhs32, item_ok, q, pi);
    kzg_store_pairs(i, ok, q, inv(ok ? KzgG::inv_target(q) : BlsF::one()), pi, setup_xy, g1, g2, pre_ok);
  }
}

}  // namespace nmsm
