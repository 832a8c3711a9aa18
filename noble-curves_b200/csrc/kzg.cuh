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
// The prover (SURVEY §8 row f16; blob_to_kzg_commitment, compute_kzg_proof, compute_blob_kzg_proof) is at the end: the
// setup table of the Lagrange points, the comb lincomb over it, the quotient by Montgomery's batch inversion, and the
// G1 compression of the results.
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

// i with its 12 bits reversed: the index map of bit_reversal_permutation over 4096 elements (an involution)
NMSM_HD uint32_t kzg_brp(uint32_t i) {
  uint32_t j = 0;
  for (int b = 0; b < 12; b++) j |= ((i >> b) & 1u) << (11 - b);
  return j;
}

// w_i = omega^brp(i) in Montgomery form, omega = 7^((r - 1) / 4096): the spec's bit-reversed domain
NMSM_HD KzgFr kzg_root(uint32_t i) {
  uint32_t e[8], seven[8] = {7, 0, 0, 0, 0, 0, 0, 0};
  for (int k = 0; k < 8; k++) {  // (r - 1) >> 12; the low word of r is 1
    const uint32_t lo = k == 0 ? FrBls381::P(0) - 1u : FrBls381::P(k), hi = k < 7 ? FrBls381::P(k + 1) : 0u;
    e[k] = (lo >> 12) | (hi << 20);
  }
  const KzgFr omega = kzg_pow(KzgFr::from_canonical(seven), e, 243);
  const uint32_t j = kzg_brp(i);
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

// ---- the prover: blob_to_kzg_commitment, compute_kzg_proof, compute_blob_kzg_proof -----------------------------------
// Every commitment and proof is g1_lincomb(bit_reversal_permutation(KZG_SETUP_G1_LAGRANGE), s) over 4096 scalars s:
// the blob's elements or the quotient's.  The setup table holds d 2^(b j) P_p for every setup point P_p (already in
// bit-reversed order), level j < ceil(256 / b) and d in [1, 2^(b-1)], level-major: entry (j, p, d) at
// ((j * 4096 + p) 2^(b-1) + d - 1) * 24 words in the prepared affine layout.  A lincomb is then one gathered mixed
// addition per point and level (table_walk_acc over the signed b-bit digits of s_p) and no doubling.
using KzgCv = CurveBls381G1Any;
static constexpr int KZG_COMB_BITS = 8;  // b: 4096 x 32 levels x 128 entries x 96 B = 1.61 GB (DESIGN.md §4h)

template <int BITS = KZG_COMB_BITS>
NMSM_HD constexpr uint64_t kzg_table_bytes(uint32_t npts) {
  return (uint64_t)point_table_levels<KzgCv, BITS>() * npts * (1u << (BITS - 1)) * KzgG::AFF_WORDS * 4;
}

// setup point i (natural order, 48-byte compressed) -> canonical affine words at position brp(i) of `xy` (k_prepare
// then converts them to the prepared layout); false when it does not decode, is the identity or lies outside G1
NMSM_HD bool kzg_setup_point_body(uint32_t i, const uint8_t* g1_48, uint32_t* xy) {
  return kzg_decode_g1(g1_48 + 48 * (size_t)i, xy + 24 * (size_t)kzg_brp(i)) == 1;
}

// level 0, entry t = p 2^(b-1) + d - 1: d P_p (table_base_body per point)
template <int BITS = KZG_COMB_BITS>
NMSM_HD void kzg_table_base_body(uint32_t t, const uint32_t* aff, uint32_t* tbl) {
  constexpr uint32_t HALF = 1u << (BITS - 1);
  const uint32_t p = t / HALF;
  table_base_body<KzgCv, BITS>(t % HALF, aff + (size_t)p * KzgG::AFF_WORDS, tbl + (size_t)p * HALF * KzgG::AFF_WORDS);
}

// lane t of S: acc += s_p P_p over the points p = t, t + S, ... < NPTS, s_p the 32-byte big-endian scalars; bad when
// one of them is >= r
template <int BITS = KZG_COMB_BITS, uint32_t NPTS = KZG_N>
NMSM_HD void kzg_lincomb_lane(uint32_t t, uint32_t S, const uint8_t* scalars_be, const uint32_t* tbl, KzgG::Acc& acc,
                              bool& bad) {
  constexpr size_t HALF = 1u << (BITS - 1);
  for (uint32_t p = t; p < NPTS; p += S) {
    uint32_t s[8];
    kzg_load_fr(s, scalars_be + 32 * (size_t)p);
    bad |= !KzgFr::canonical_in_range(s);
    table_walk_acc<KzgCv, BITS, NPTS * HALF>(tbl + p * HALF * KzgG::AFF_WORDS, s, acc);
  }
}

// The 48-byte Zcash-flag compressed encoding of a canonical affine point (24 words): x big-endian with 0x80, plus 0x20
// when y > (p - 1) / 2; the identity is 0xc0 || 0..0
NMSM_HD void kzg_g1_compress(const uint32_t* xy, bool inf, uint8_t* out48) {
  for (int k = 0; k < 48; k++) out48[k] = 0;
  if (inf) {
    out48[0] = 0xc0;
    return;
  }
  for (int k = 0; k < 12; k++)
    for (int j = 0; j < 4; j++) out48[47 - 4 * k - j] = (uint8_t)(xy[k] >> (8 * j));
  out48[0] |= bls12_381_sort_bit(xy + 12) ? 0xa0 : 0x80;
}

// the sum of P accumulators stored one after another
NMSM_HD_NOINLINE KzgG::Acc kzg_sum_parts(const uint32_t* parts, uint32_t P) {
  KzgG::Acc acc = KzgG::identity();
  for (uint32_t k = 0; k < P; k++) nl_add<KzgG>(acc, load_acc<KzgG>(parts + (size_t)k * KzgG::ACC_WORDS));
  return acc;
}

// a lincomb's accumulator, normalised with zi = 1 / inv_target(acc), compressed
NMSM_HD_NOINLINE void kzg_store_g1(const KzgG::Acc& acc, const KzgG::Field& zi, uint8_t* out48) {
  uint32_t xy[24], inf;
  KzgG::to_affine_canonical_with_inv(acc, zi, xy, &inf);
  kzg_g1_compress(xy, inf != 0, out48);
}

// serial statement of k_kzg_lincomb + k_kzg_lincomb_finish for blob i (S lanes one after another)
template <int BITS = KZG_COMB_BITS, uint32_t NPTS = KZG_N>
NMSM_HD void kzg_lincomb_serial(uint32_t i, uint32_t S, const uint8_t* scalars_be, const uint32_t* tbl, uint8_t* out48,
                                uint8_t* item_ok) {
  KzgG::Acc sum = KzgG::identity();
  bool bad = false;
  for (uint32_t t = 0; t < S; t++) {
    KzgG::Acc acc = KzgG::identity();
    kzg_lincomb_lane<BITS, NPTS>(t, S, scalars_be + (size_t)i * 32 * NPTS, tbl, acc, bad);
    nl_add<KzgG>(sum, acc);
  }
  if (bad) item_ok[i] = 0;
  kzg_store_g1(sum, inv(KzgG::inv_target(sum)), out48 + 48 * (size_t)i);
}

// ---- compute_kzg_proof_impl's quotient q_i = (f_i - y) / (w_i - z), in place of the blob ------------------------------
// z and y of blob i in Montgomery form; false when the blob failed its range vote (item_ok) or z >= r
NMSM_HD bool kzg_quotient_start(uint32_t i, const uint8_t* zs32, const uint8_t* ys32, const uint8_t* item_ok, KzgFr& z,
                                KzgFr& y) {
  uint32_t zw[8], yw[8];
  kzg_load_fr(zw, zs32 + (size_t)i * 32);
  kzg_load_fr(yw, ys32 + (size_t)i * 32);
  if (!item_ok[i] || !KzgFr::canonical_in_range(zw)) return false;
  z = KzgFr::from_canonical(zw);
  y = KzgFr::from_canonical(yw);
  return true;
}

// Montgomery's batch inversion over lane t's elements e_j = t + 256 j.  Forward: d_j = w_j - z (a zero d_m, z = w_m,
// taken as 1 and m reported in hit, as kzg_eval_lane does), P_j = d_0 ... d_j, and element e_j overwritten by
// P_(j-1) (f_j - y) as 8 Montgomery words.  Returns P_15.
NMSM_HD KzgFr kzg_quotient_fwd(uint32_t t, uint8_t* blob, const KzgFr& z, const KzgFr& y, const uint32_t* roots,
                               int& hit) {
  KzgFr pre = KzgFr::one();
  for (int j = 0; j < KZG_PER_LANE; j++) {
    const uint32_t e = t + KZG_EVAL_THREADS * j;
    uint32_t fw[8];
    kzg_load_fr(fw, blob + 32 * (size_t)e);
    KzgFr w;
    load_words<8>(w.v, roots + 8 * (size_t)e);
    KzgFr d = w - z;
    if (d.is_zero()) {
      hit = (int)e;
      d = KzgFr::one();
    }
    const KzgFr m = pre * (KzgFr::from_canonical(fw) - y);
    store_words<8>(reinterpret_cast<uint32_t*>(blob + 32 * (size_t)e), m.v);
    pre = pre * d;
  }
  return pre;
}

// Back-sweep from ri = 1 / P_15: q_j = P_(j-1) (f_j - y) / P_j, then 1 / P_(j-1) = d_j / P_j; q_j stored as 32
// big-endian bytes.  With `sum`: returns sum_j q_j w_j, the term of the within-domain quotient.
NMSM_HD KzgFr kzg_quotient_back(uint32_t t, uint8_t* blob, const KzgFr& z, const uint32_t* roots, KzgFr ri, bool sum) {
  KzgFr acc = KzgFr::zero();
  for (int j = KZG_PER_LANE - 1; j >= 0; j--) {
    const uint32_t e = t + KZG_EVAL_THREADS * j;
    KzgFr m, w;
    load_words_rw<8>(m.v, reinterpret_cast<const uint32_t*>(blob + 32 * (size_t)e));
    load_words<8>(w.v, roots + 8 * (size_t)e);
    KzgFr d = w - z;
    if (d.is_zero()) d = KzgFr::one();
    const KzgFr q = m * ri;
    ri = ri * d;
    if (sum) acc = acc + q * w;
    uint32_t qw[8];
    q.to_canonical(qw);
    kzg_store_fr(blob + 32 * (size_t)e, qw);
  }
  return acc;
}

// z = w_m: q_m = compute_quotient_eval_within_domain(z, f, y) = sum_(i != m) (f_i - y) w_i / (z (z - w_i))
// = -(1 / z) sum_i q_i w_i (the back-sweep left q_m = 0, since y = f_m)
NMSM_HD void kzg_quotient_in_domain(uint8_t* blob, int m, const KzgFr& z, const KzgFr& sum) {
  uint32_t qw[8];
  (-(sum * inv(z))).to_canonical(qw);
  kzg_store_fr(blob + 32 * (size_t)m, qw);
}

// serial statement of k_kzg_quotient for blob i (one inversion per lane instead of one per warp)
NMSM_HD void kzg_quotient_serial(uint32_t i, uint8_t* blobs, const uint8_t* zs32, const uint8_t* ys32,
                                 const uint32_t* roots, uint8_t* item_ok) {
  uint8_t* blob = blobs + (size_t)i * KZG_BLOB_BYTES;
  KzgFr z, y;
  if (!kzg_quotient_start(i, zs32, ys32, item_ok, z, y)) {
    item_ok[i] = 0;
    return;
  }
  int hit = -1;
  KzgFr pre[KZG_EVAL_THREADS];
  for (uint32_t t = 0; t < KZG_EVAL_THREADS; t++) pre[t] = kzg_quotient_fwd(t, blob, z, y, roots, hit);
  KzgFr sum = KzgFr::zero();
  for (uint32_t t = 0; t < KZG_EVAL_THREADS; t++) sum = sum + kzg_quotient_back(t, blob, z, roots, inv(pre[t]), hit >= 0);
  if (hit >= 0) kzg_quotient_in_domain(blob, hit, z, sum);
}

}  // namespace nmsm
