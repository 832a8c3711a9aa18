// nmsm::inv — the field inversion every kernel uses (to-affine of results, warp_batch_inverse, table building, decoders).
// Verified on the host against pow(x, -1, p) for all four base fields (tests/test_hostemu_parity.py::test_divsteps_inverse)
// and on the GPU through every bit-exact point result.  It replaced the binary extended GCD (field.cuh inv_xgcd, kept as
// fallback), which takes several times longer for a lone warp (tools/gpu/micro/tail_ops.cu times both).
//
// Modular inversion by batched division steps (Bernstein–Yang "safegcd" in its half-delta form): the state
// (f, g) = (p, x) is advanced 30 division steps at a time from the low 30 bits alone, the 2x2 transition matrix
// of a batch is then applied to the full-width (f, g) and, modulo p, to the Bezout pair (d, e).  Compared with the
// binary extended GCD in field.cuh this has no data-dependent branch inside a batch (all lanes of a warp execute
// the same instruction stream) and spends its full-width work in a few multiply-accumulate passes per batch
// instead of ~2 * BITS shift/subtract passes.  The outer loop stops when g == 0; should that not have happened
// after MAX_BATCHES batches (it cannot for inputs < p, the cap is far above the published worst case), the caller
// is told and falls back to field.cuh's inv.
//
// Numbers are held in signed 30-bit limbs (value = sum v[i] * 2^(30 i), every limb but the top in [0, 2^30), the top
// limb carries the sign).  The reference's counterpart is modular.ts:159-182 `invert` (extended Euclid on BigInt);
// results are identical: the unique x^-1 in [0, p).
#pragma once
#include <stdint.h>

#include "field.cuh"

namespace nmsm {

template <class C>
struct DivstepsInv {
  static constexpr int N = C::N;                       // 32-bit words of the field
  static constexpr int L = (32 * N + 2 + 29) / 30;     // 30-bit limbs: room for (-2p, 2p)
  static constexpr int32_t M30 = (int32_t)((1u << 30) - 1u);
  static constexpr int MAX_BATCHES = (49 * 32 * N + 57) / 17 / 30 + 2;  // Bernstein-Yang Thm 11.2 bound for the delta = 1 walk

  struct S30 {
    int32_t v[L];
  };
  struct Trans {
    int32_t u, v, q, r;
  };

  NMSM_HD static S30 from_words(const uint32_t* w) {  // 0 <= value < 2^(32 N)
    S30 r;
    for (int i = 0; i < L; i++) {
      const int bit = 30 * i, k = bit >> 5, sh = bit & 31;
      uint64_t lo = k < N ? w[k] : 0u, hi = (k + 1) < N ? w[k + 1] : 0u;
      r.v[i] = (int32_t)((uint32_t)(((lo | (hi << 32)) >> sh)) & (uint32_t)M30);
    }
    return r;
  }
  NMSM_HD static void to_words(const S30& a, uint32_t* w) {  // a in [0, 2^(32 N)), limbs normalised
    for (int k = 0; k < N; k++) w[k] = 0u;
    for (int i = 0; i < L; i++) {
      const int bit = 30 * i, k = bit >> 5, sh = bit & 31;
      const uint64_t val = (uint64_t)(uint32_t)a.v[i] << sh;
      if (k < N) w[k] |= (uint32_t)val;
      if (k + 1 < N) w[k + 1] |= (uint32_t)(val >> 32);
    }
  }
  NMSM_HD static S30 modulus() {
    uint32_t p[N];
    for (int k = 0; k < N; k++) p[k] = C::P(k);
    return from_words(p);
  }
  // p^-1 mod 2^30 by Newton iteration on the low word (p is odd)
  NMSM_HD static uint32_t modulus_inv30() {
    const uint32_t p0 = C::P(0);
    uint32_t x = p0;  // correct to 3 bits
    for (int i = 0; i < 5; i++) x *= 2u - p0 * x;
    return x & (uint32_t)M30;
  }

  // 30 division steps on the low bits; zeta = -(delta + 1/2).  Returns the new zeta, t = the transition matrix with
  // t * (f, g) = 2^30 * (f', g').
  NMSM_HD static int32_t divsteps_30(int32_t zeta, uint32_t f0, uint32_t g0, Trans& t) {
    uint32_t u = 1, v = 0, q = 0, r = 1;
    uint32_t f = f0, g = g0;
    for (int i = 0; i < 30; i++) {
      uint32_t c1 = (uint32_t)(zeta >> 31);  // all ones iff zeta < 0
      const uint32_t c2 = 0u - (g & 1u);     // all ones iff g is odd
      const uint32_t x = (f ^ c1) - c1, y = (u ^ c1) - c1, z = (v ^ c1) - c1;  // conditionally negated f, u, v
      g += x & c2;
      q += y & c2;
      r += z & c2;
      c1 &= c2;                                // swap only when zeta < 0 and g odd
      zeta = (int32_t)(((uint32_t)zeta ^ c1) - 1u);
      f += g & c1;
      u += q & c1;
      v += r & c1;
      g >>= 1;
      u <<= 1;
      v <<= 1;
    }
    t.u = (int32_t)u;
    t.v = (int32_t)v;
    t.q = (int32_t)q;
    t.r = (int32_t)r;
    return zeta;
  }

  // (f, g) <- t * (f, g) / 2^30, exact
  NMSM_HD static void update_fg(S30& f, S30& g, const Trans& t) {
    const int64_t u = t.u, v = t.v, q = t.q, r = t.r;
    int64_t cf = u * f.v[0] + v * g.v[0];
    int64_t cg = q * f.v[0] + r * g.v[0];
    cf >>= 30;
    cg >>= 30;
    for (int i = 1; i < L; i++) {
      cf += u * f.v[i] + v * g.v[i];
      cg += q * f.v[i] + r * g.v[i];
      f.v[i - 1] = (int32_t)cf & M30;
      g.v[i - 1] = (int32_t)cg & M30;
      cf >>= 30;
      cg >>= 30;
    }
    f.v[L - 1] = (int32_t)cf;
    g.v[L - 1] = (int32_t)cg;
  }

  // (d, e) <- t * (d, e) / 2^30 mod p, keeping both in (-2p, p)
  NMSM_HD static void update_de(S30& d, S30& e, const Trans& t, const S30& m, uint32_t m_inv30) {
    const int64_t u = t.u, v = t.v, q = t.q, r = t.r;
    const int32_t sd = d.v[L - 1] >> 31, se = e.v[L - 1] >> 31;  // sign masks
    int32_t md = (t.u & sd) + (t.v & se);
    int32_t me = (t.q & sd) + (t.r & se);
    int64_t cd = u * d.v[0] + v * e.v[0];
    int64_t ce = q * d.v[0] + r * e.v[0];
    // choose the multiples of p that clear the bottom 30 bits
    md -= (int32_t)((m_inv30 * (uint32_t)cd + (uint32_t)md) & (uint32_t)M30);
    me -= (int32_t)((m_inv30 * (uint32_t)ce + (uint32_t)me) & (uint32_t)M30);
    cd += (int64_t)m.v[0] * md;
    ce += (int64_t)m.v[0] * me;
    cd >>= 30;
    ce >>= 30;
    for (int i = 1; i < L; i++) {
      cd += u * d.v[i] + v * e.v[i] + (int64_t)m.v[i] * md;
      ce += q * d.v[i] + r * e.v[i] + (int64_t)m.v[i] * me;
      d.v[i - 1] = (int32_t)cd & M30;
      e.v[i - 1] = (int32_t)ce & M30;
      cd >>= 30;
      ce >>= 30;
    }
    d.v[L - 1] = (int32_t)cd;
    e.v[L - 1] = (int32_t)ce;
  }

  // bring a in (-2p, p) into [0, p), negating first if `negate`
  NMSM_HD static void normalize(S30& a, bool negate, const S30& m) {
    auto add_masked = [&](int32_t mask) {  // a += m & mask, then propagate carries
      int32_t carry = 0;
      for (int i = 0; i < L; i++) {
        int32_t x = a.v[i] + (m.v[i] & mask) + carry;
        if (i < L - 1) {
          carry = x >> 30;
          x &= M30;
        }
        a.v[i] = x;
      }
    };
    add_masked(a.v[L - 1] >> 31);  // a < 0: a += p  -> (-p, p)
    if (negate) {
      int32_t carry = 0;
      for (int i = 0; i < L; i++) {
        int32_t x = -a.v[i] + carry;
        if (i < L - 1) {
          carry = x >> 30;
          x &= M30;
        }
        a.v[i] = x;
      }
    }
    add_masked(a.v[L - 1] >> 31);  // still negative: one more p  -> [0, p)
  }

  NMSM_HD static bool is_zero(const S30& a) {
    int32_t t = 0;
    for (int i = 0; i < L; i++) t |= a.v[i];
    return t == 0;
  }

  // out = x^-1 mod p for 0 < x < p (plain integers, N little-endian words).  Returns false if the walk did not finish.
  NMSM_HD static bool inverse_words(const uint32_t* x, uint32_t* out, int* batches_used = nullptr) {
    const S30 m = modulus();
    const uint32_t mi = modulus_inv30();
    S30 f = m, g = from_words(x), d, e;
    for (int i = 0; i < L; i++) {
      d.v[i] = 0;
      e.v[i] = 0;
    }
    e.v[0] = 1;
    int32_t zeta = -1;
    bool done = false;
    for (int it = 0; it < MAX_BATCHES; it++) {
      Trans t;
      zeta = divsteps_30(zeta, (uint32_t)f.v[0] | ((uint32_t)f.v[1] << 30), (uint32_t)g.v[0] | ((uint32_t)g.v[1] << 30), t);
      update_de(d, e, t, m, mi);
      update_fg(f, g, t);
      if (is_zero(g)) {
        done = true;
        if (batches_used) *batches_used = it + 1;
        break;
      }
    }
    if (!done) return false;
    // f = +-1 (gcd); d * x = f (mod p)
    normalize(d, (f.v[L - 1] >> 31) != 0, m);
    to_words(d, out);
    return true;
  }

  // Montgomery form in, Montgomery form out (drop-in for nmsm::inv): (aR)^-1 = a^-1 R^-1, two multiplications by R^2 lift it back
  NMSM_HD static Fp<C> inverse(const Fp<C>& a) {
    if (a.is_zero()) return a;
    Fp<C> r, r2;
    if (!inverse_words(a.v, r.v)) return nmsm::inv_xgcd(a);
    for (int k = 0; k < N; k++) r2.v[k] = C::R2(k);
    return (r * r2) * r2;
  }
};

// Montgomery form in and out; 0 maps to 0 (modular.ts:159-182 `invert` computes the same inverse on BigInt)
template <class C>
NMSM_HD Fp<C> inv(const Fp<C>& a) {
  return DivstepsInv<C>::inverse(a);
}

}  // namespace nmsm
