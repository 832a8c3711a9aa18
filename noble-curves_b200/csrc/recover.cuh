// secp256k1 ECDSA public-key recovery (SURVEY §8 row f9) and Ethereum's ecrecover precompile (0x01), batched.
//
// The reference recovers one key at a time: weierstrass.ts `Signature.recoverPublicKey` (noble-curves v2), reached
// through secp256k1.recoverPublicKey(signature, message, { prehash }) with the 65-byte 'recovered' format
// rec || r || s.  Inside the reference every failure throws; in the batch it is a 0 verdict:
//   rec in {0, 1, 2, 3};  1 <= r, s < n;  x = rec & 2 ? r + n : r, x < p;
//   R = the SEC1 decode of (rec & 1 ? 03 : 02) || x (fails when x^3 + 7 is not a square);
//   h = bits2int_modN(prehash ? sha256(m) : m) (a raw message over 8192 bytes fails, as in verify);
//   u1 = -h r^-1, u2 = s r^-1 (mod n);  Q = u1 G + u2 R;  Q = O fails.
// No lowS rule applies, and Q is on the curve by construction.  ecrecover (Yellow Paper appendix E, ECREC) takes
// h || v || r || s (32 B each, big-endian): v must be 27 or 28 as a 256-bit integer, rec = v - 27, h is the 32 raw
// bytes (no prehash), and the output is 12 zero bytes || the last 20 bytes of keccak256(x || y) of Q, big-endian.
//
// As for ECDSA verification (ecdsa_verify.cuh) the batch is data-parallel, split into two kernels
// (inst_secp256k1.cu):
//   recover_prepare_body  parse, range checks, x = r (+ n), lift R (sec1_decode_secp256k1), h
//   (kernel)              r^-1 through one warp-shared inversion per 32 items (msm.cuh warp_batch_inverse)
//   recover_store         R, u1, u2
//   recover_check_lane    Q = u1 G (fixed-point table of G) + u2 R (GLV scalar_mul_acc), complete addition, Q != O
//   (kernel)              ZZZ^-1 through one warp-shared inversion per 32 items
//   recover_finish        canonical affine Q, or for ecrecover the address word (keccak256_64)
// Bodies are host/device so tests/hostemu can run them; the *_serial statements invert once per item.
#pragma once
#include "ecdsa_verify.cuh"

namespace nmsm {

// ---- Keccak-256 of a 64-byte input (the original Keccak padding 0x01, not SHA-3's 0x06) --------------------------
NMSM_HD uint64_t keccak_rc(int round) {
  constexpr uint64_t RC[24] = {
      0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808aull, 0x8000000080008000ull,
      0x000000000000808bull, 0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull,
      0x000000000000008aull, 0x0000000000000088ull, 0x0000000080008009ull, 0x000000008000000aull,
      0x000000008000808bull, 0x800000000000008bull, 0x8000000000008089ull, 0x8000000000008003ull,
      0x8000000000008002ull, 0x8000000000000080ull, 0x000000000000800aull, 0x800000008000000aull,
      0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull};
  return RC[round];
}
NMSM_HD uint64_t rotl64(uint64_t x, int n) { return (x << n) | (x >> (64 - n)); }  // 1 <= n <= 63

// Keccak-f[1600] on the 25 lanes a[x + 5 y].  The lane walk of rho + pi (positions and rotations along the
// (x, y) -> (y, 2x + 3y) orbit of lane 1) is unrolled so that the state stays in registers.
NMSM_HD void keccak_f1600(uint64_t* a) {
  constexpr int PI[24] = {10, 7, 11, 17, 18, 3, 5, 16, 8, 21, 24, 4, 15, 23, 19, 13, 12, 2, 20, 14, 22, 9, 6, 1};
  constexpr int RHO[24] = {1, 3, 6, 10, 15, 21, 28, 36, 45, 55, 2, 14, 27, 41, 56, 8, 25, 43, 62, 18, 39, 61, 20, 44};
  for (int round = 0; round < 24; round++) {
    uint64_t c[5];
#pragma unroll
    for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
#pragma unroll
    for (int x = 0; x < 5; x++) {
      const uint64_t d = c[(x + 4) % 5] ^ rotl64(c[(x + 1) % 5], 1);
#pragma unroll
      for (int y = 0; y < 25; y += 5) a[x + y] ^= d;
    }
    uint64_t cur = a[1];
#pragma unroll
    for (int t = 0; t < 24; t++) {
      const uint64_t next = a[PI[t]];
      a[PI[t]] = rotl64(cur, RHO[t]);
      cur = next;
    }
#pragma unroll
    for (int y = 0; y < 25; y += 5) {
      uint64_t b[5];
#pragma unroll
      for (int x = 0; x < 5; x++) b[x] = a[y + x];
#pragma unroll
      for (int x = 0; x < 5; x++) a[y + x] = b[x] ^ (~b[(x + 1) % 5] & b[(x + 2) % 5]);
    }
    a[0] ^= keccak_rc(round);
  }
}

// keccak256(in[0..64)) -> out[32]: one absorb into the 136-byte rate (64 data bytes, the pad byte 0x01 at 64, 0x80
// in the last rate byte 135) and one permutation
NMSM_HD void keccak256_64(const uint8_t* in, uint8_t* out) {
  uint64_t a[25];
#pragma unroll
  for (int k = 0; k < 25; k++) a[k] = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    uint64_t w = 0;
#pragma unroll
    for (int j = 7; j >= 0; j--) w = (w << 8) | in[8 * k + j];
    a[k] = w;
  }
  a[8] = 0x01ull;
  a[16] = 0x80ull << 56;
  keccak_f1600(a);
#pragma unroll
  for (int k = 0; k < 32; k++) out[k] = (uint8_t)(a[k >> 3] >> (8 * (k & 7)));
}

// ---- recovery ----------------------------------------------------------------------------------------------------
// The two input layouts of one prepare body: RECOVER_SIG65 = rec || r || s (65 B) plus message i of msgs / msg_off
// under `flags`; RECOVER_ECREC = the 128-byte precompile input h || v || r || s.
static constexpr int RECOVER_SIG65 = 0;
static constexpr int RECOVER_ECREC = 1;

// Item i: the point R (canonical affine words), r, s and h.  False = the reference throws before any scalar
// multiplication; the outputs are then unspecified.
template <int LAYOUT>
NMSM_HD bool recover_prepare_body(uint32_t i, const uint8_t* in, const uint8_t* msgs, const uint64_t* msg_off,
                                  int flags, uint32_t* r_xy, uint32_t* r, uint32_t* s, uint32_t* h) {
  const uint8_t* rs_be;
  uint32_t rec;
  if (LAYOUT == RECOVER_ECREC) {
    const uint8_t* w = in + (size_t)i * 128;
    uint32_t v_high = 0;  // v < 2^8 as a 256-bit integer
    for (int k = 32; k < 63; k++) v_high |= w[k];
    if (v_high != 0 || (w[63] != 27 && w[63] != 28)) return false;
    rec = w[63] - 27u;
    rs_be = w + 64;
  } else {
    const uint8_t* w = in + (size_t)i * 65;
    rec = w[0];
    if (rec > 3) return false;
    rs_be = w + 1;
  }
  words_from_be_bytes<32>(r, rs_be);
  words_from_be_bytes<32>(s, rs_be + 32);
  if (!words8_nonzero(r) || !EcS::canonical_in_range(r) || !words8_nonzero(s) || !EcS::canonical_in_range(s))
    return false;
  // x = r or r + n; the SEC1 decoder rejects x >= p
  uint32_t x[8];
  for (int k = 0; k < 8; k++) x[k] = r[k];
  if (rec & 2u) {
    x[0] = add_cc(r[0], FnSecp256k1Mod::P(0));
    for (int k = 1; k < 8; k++) x[k] = addc_cc(r[k], FnSecp256k1Mod::P(k));
    if (addc(0, 0)) return false;  // r + n >= 2^256 > p
  }
  uint8_t enc[33];
  enc[0] = (uint8_t)(0x02u | (rec & 1u));
  for (int j = 0; j < 32; j++) enc[1 + j] = (uint8_t)(x[(31 - j) >> 2] >> (8 * ((31 - j) & 3)));
  if (sec1_decode_secp256k1(enc, r_xy) != 1) return false;
  if (LAYOUT == RECOVER_ECREC) return ecdsa_msg_hash(in + (size_t)i * 128, 32, 0, h);
  return ecdsa_msg_hash(msgs + msg_off[i], msg_off[i + 1] - msg_off[i], flags, h);
}

// Given w = r^-1 (Montgomery form mod n): u1 = -h w, u2 = s w, and the per-item state k_recover_check reads.
// ok_out[i] carries the prepare verdict to the check, which overwrites it with the final one.
NMSM_HD void recover_store(uint32_t i, bool ok, const uint32_t* r_xy, const uint32_t* s, const uint32_t* h,
                           const EcS& w, uint32_t* rpts, uint32_t* u1s, uint32_t* u2s, uint8_t* ok_out) {
  ok_out[i] = ok ? 1 : 0;
  if (!ok) return;
  uint32_t u1[8], u2[8];
  (-(EcS::from_canonical(h) * w)).to_canonical(u1);
  (EcS::from_canonical(s) * w).to_canonical(u2);
  store_words<16>(rpts + (size_t)i * 16, r_xy);
  store_words<8>(u1s + (size_t)i * 8, u1);
  store_words<8>(u2s + (size_t)i * 8, u2);
}

// serial statement of k_recover_prepare (one inversion per item instead of one per warp)
template <int LAYOUT>
NMSM_HD void recover_prepare_serial(uint32_t n, const uint8_t* in, const uint8_t* msgs, const uint64_t* msg_off,
                                    int flags, uint32_t* rpts, uint32_t* u1s, uint32_t* u2s, uint8_t* ok_out) {
  for (uint32_t i = 0; i < n; i++) {
    uint32_t rxy[16], r[8], s[8], h[8];
    const bool ok = recover_prepare_body<LAYOUT>(i, in, msgs, msg_off, flags, rxy, r, s, h);
    recover_store(i, ok, rxy, s, h, ok ? inv(EcS::from_canonical(r)) : EcS::one(), rpts, u1s, u2s, ok_out);
  }
}

// The per-lane part of the check for item i after recover_store: acc = Q = u1 G + u2 R.  True iff prepare accepted
// and Q != O.  acc is the identity for a lane that prepare rejected, so G::inv_target(acc) = 1 for it.
// tbl: the fixed-point table of G (table_mul_body layout, BITS-bit digits; BITS is a parameter only so that
// tests/hostemu can use a small table).
template <int BITS = PT_BITS>
NMSM_HD bool recover_check_lane(uint32_t i, const uint32_t* tbl, const uint32_t* rpts, const uint32_t* u1s,
                                const uint32_t* u2s, const uint8_t* ok_in, typename CurveSecp256k1::G::Acc& acc,
                                unsigned int* err) {
  using Cv = CurveSecp256k1;
  using G = Cv::G;
  acc = G::identity();
  if (!ok_in[i]) return false;
  table_mul_body<Cv, BITS>(i, tbl, u1s, 1, acc, err);  // u1 = 0 (h = 0 mod n) gives O
  uint32_t rxy[16], u2[8];
  load_words<16>(rxy, rpts + (size_t)i * 16);
  load_words<8>(u2, u2s + (size_t)i * 8);
  nl_add<G>(acc, scalar_mul_acc<Cv>(G::prepare(rxy), u2));  // complete: doubles when u1 G == u2 R
  return !G::is_identity(acc);
}

// Item i's output from Q = acc and zi = ZZZ^-1: out_ok[i], and either the recovered key (16 words: the canonical
// affine packing of nmsm_mul_batch) or, for ecrecover, the 32-byte address word (8 words).  A failed item writes 0
// and zero words.
template <int LAYOUT>
NMSM_HD void recover_finish(uint32_t i, bool ok, const typename CurveSecp256k1::G::Acc& acc,
                            const typename CurveSecp256k1::G::Field& zi, uint32_t* out, uint8_t* out_ok) {
  uint32_t xy[16];
  for (int k = 0; k < 16; k++) xy[k] = 0;
  if (ok) {
    uint32_t inf;
    CurveSecp256k1::G::to_affine_canonical_with_inv(acc, zi, xy, &inf);
  }
  if (LAYOUT == RECOVER_ECREC) {
    uint32_t word[8];
    for (int k = 0; k < 8; k++) word[k] = 0;
    if (ok) {
      uint8_t be[64], digest[32];
      for (int j = 0; j < 32; j++) {
        be[j] = (uint8_t)(xy[(31 - j) >> 2] >> (8 * ((31 - j) & 3)));
        be[32 + j] = (uint8_t)(xy[8 + ((31 - j) >> 2)] >> (8 * ((31 - j) & 3)));
      }
      keccak256_64(be, digest);
      for (int j = 12; j < 32; j++) word[j >> 2] |= (uint32_t)digest[j] << (8 * (j & 3));  // byte j of the word
    }
    store_words<8>(out + (size_t)i * 8, word);
  } else {
    store_words<16>(out + (size_t)i * 16, xy);
  }
  out_ok[i] = ok ? 1 : 0;
}

// serial statement of k_recover_check (one inversion per item instead of one per warp)
template <int LAYOUT, int BITS = PT_BITS>
NMSM_HD void recover_check_serial(uint32_t n, const uint32_t* tbl, const uint32_t* rpts, const uint32_t* u1s,
                                  const uint32_t* u2s, uint8_t* ok, uint32_t* out, unsigned int* err) {
  using G = CurveSecp256k1::G;
  for (uint32_t i = 0; i < n; i++) {
    G::Acc acc;
    const bool q_ok = recover_check_lane<BITS>(i, tbl, rpts, u1s, u2s, ok, acc, err);
    recover_finish<LAYOUT>(i, q_ok, acc, inv(G::inv_target(acc)), out, ok);
  }
}

}  // namespace nmsm
