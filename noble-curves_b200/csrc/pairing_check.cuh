// Batch pairing-product checks for any pairing curve: the curve-independent bodies of the Miller and final kernels
// and their serial statement (tests/hostemu), as templates over a pairing policy P (pairing.cuh BlsPairing,
// pairing_bn254.cuh Bn254Pairing) that provides
//   F12                    the Fp12 type, F12::WORDS words per value
//   G1_WORDS, G2_WORDS     canonical affine point sizes in words
//   G1Curve, G2Curve       the curve policies whose equations validate the points (validate.cuh)
//   miller_loop(p, q)      the Miller value of one pair, neither point the identity
//   final_exp(f)           the final exponentiation (any power coprime to r of the exact pairing's)
//
//   check j:  prod_{i in [off[j], off[j+1])} e(P_i, Q_i) == 1
// Miller values of a chunk of pairs sit in a workspace W; a check that spans a chunk boundary carries its partial
// product to the next chunk in one of two alternating carry slots after the chunk's values.
#pragma once
#include "fp12.cuh"
#include "msm_body.cuh"
#include "validate.cuh"

namespace nmsm {

NMSM_HD bool words_zero(const uint32_t* w, int n) {
  uint32_t t = 0;
  for (int k = 0; k < n; k++) t |= w[k];
  return t == 0;
}

// pair i: validates both points (err[0] = smallest bad G1 index, err[1] = smallest bad G2 index) and writes f_i to out
// (F12::WORDS words); rejected and identity pairs write 1.
template <class P>
NMSM_HD void pairing_miller_body(uint64_t i, const uint32_t* g1, const uint32_t* g2, uint32_t* out, unsigned int* err) {
  using F12 = typename P::F12;
  uint32_t p[P::G1_WORDS], q[P::G2_WORDS];
  load_words<P::G1_WORDS>(p, g1 + i * P::G1_WORDS);
  load_words<P::G2_WORDS>(q, g2 + i * P::G2_WORDS);
  const bool ok1 = point_on_curve<typename P::G1Curve>(p), ok2 = point_on_curve<typename P::G2Curve>(q);
  if (!ok1) atomic_min_u32(&err[0], (uint32_t)i);
  if (!ok2) atomic_min_u32(&err[1], (uint32_t)i);
  F12 f = F12::one();
  if (ok1 && ok2 && !words_zero(p, P::G1_WORDS) && !words_zero(q, P::G2_WORDS)) f = P::miller_loop(p, q);
  f.store(out);
}

// pairs of check j: [off[j], off[j+1]); off == nullptr means two pairs per check (verification)
NMSM_HD uint64_t pairing_pair_off(const uint64_t* off, uint64_t j) { return off ? off[j] : 2 * j; }

// check j, over the pair chunk [q0, q1) whose Miller values are W[0 .. q1 - q0).  A check that began in an earlier
// chunk multiplies in carry_in; one that continues past q1 leaves its partial product in carry_out and no verdict.
// Empty checks are skipped (the caller pre-sets their verdict to 1).  pre_ok (optional) is ANDed in.
template <class P>
NMSM_HD void pairing_final_body(uint64_t j, const uint64_t* off, uint64_t q0, uint64_t q1, const uint32_t* W,
                                const uint32_t* carry_in, uint32_t* carry_out, const uint8_t* pre_ok, uint8_t* out_ok) {
  using F12 = typename P::F12;
  const uint64_t a = pairing_pair_off(off, j), b = pairing_pair_off(off, j + 1);
  if (a == b) return;
  F12 f = F12::one(), g;
  if (a < q0) f.load(carry_in);
  const uint64_t lo = a < q0 ? q0 : a, hi = b < q1 ? b : q1;
  for (uint64_t q = lo; q < hi; q++) {
    g.load(W + (q - q0) * F12::WORDS);
    f = fp12_mul(f, g);
  }
  if (b > q1) {
    f.store(carry_out);
    return;
  }
  const bool ok = P::final_exp(f).is_one() && (!pre_ok || pre_ok[j]);
  out_ok[j] = ok ? 1 : 0;
}

// ---- serial statement (tests/hostemu): the kernels' work for pairs/checks in order, with chunks of `chunk` pairs ----
// W: (chunk + 2) * F12::WORDS words (the Miller values and two carry slots, as the library's workspace)
template <class P>
NMSM_HD void pairing_check_serial(uint64_t n_checks, const uint64_t* off, const uint32_t* g1, const uint32_t* g2,
                                  const uint8_t* pre_ok, uint64_t chunk, uint32_t* W, uint8_t* out_ok,
                                  unsigned int* err) {
  constexpr int WORDS = P::F12::WORDS;
  const uint64_t total = pairing_pair_off(off, n_checks);
  for (uint64_t j = 0; j < n_checks; j++) out_ok[j] = 1;
  uint64_t c = 0;
  for (uint64_t q0 = 0; q0 < total; q0 += chunk, c++) {
    const uint64_t q1 = q0 + chunk < total ? q0 + chunk : total;
    for (uint64_t q = q0; q < q1; q++) pairing_miller_body<P>(q, g1, g2, W + (q - q0) * WORDS, err);
    uint32_t* carry_in = W + (chunk + ((c + 1) & 1)) * WORDS;
    uint32_t* carry_out = W + (chunk + (c & 1)) * WORDS;
    for (uint64_t j = 0; j < n_checks; j++)
      if (pairing_pair_off(off, j + 1) > q0 && pairing_pair_off(off, j) < q1)
        pairing_final_body<P>(j, off, q0, q1, W, carry_in, carry_out, pre_ok, out_ok);
  }
}

}  // namespace nmsm
