// Prime-field arithmetic in Montgomery form on 32-bit register limbs (N = 8 for the 254/255/256-bit
// primes, N = 12 for the 381-bit BLS12-381 base field).
//
// Replaces (results identical after from-Montgomery) the reference's bigint field:
//   /root/reference/src/abstract/modular.ts:888-1038  `_Field` add/sub/neg/mul/sqr/inv/is0/eql
//   /root/reference/src/abstract/modular.ts:50-54     mod()
// The reference computes (a*b) % p on BigInt; here elements live as a*R mod p, R = 2^(32N), and
// every value handed to callers is fully reduced to [0, p) so equality is limb equality.
//
// mont_mul layout ("absolute even/odd columns"): two accumulator arrays indexed by absolute limb
// position.  A partial product x_j*w at position q goes to the array whose 64-bit slots are aligned
// to q's parity, so each row is one carry chain of (mad.lo.cc, madc.hi.cc) pairs = IMAD.WIDE.U32.X,
// with no per-product carry fix-up.  After step i the low limb of the slot array is zero and the
// high half is folded into the other array with an add.cc whose carry feeds that array's next
// chain.  Because indices are compile-time after unrolling, the "shift right by one limb per step"
// of CIOS is pure register renaming.  Cost: 2N^2 + N IMAD.WIDE-equivalents (N=12: 300, N=8: 136).
#pragma once
#include "bigint.cuh"

namespace nmsm {

// r = (top:r) - p if (top:r) >= p.  Requires (top:r) < 2p.
template <class C>
NMSM_HD void reduce_once(uint32_t* r, uint32_t top) {
  constexpr int N = C::N;
  uint32_t d[N];
  d[0] = sub_cc(r[0], C::P(0));
#pragma unroll
  for (int k = 1; k < N; k++) d[k] = subc_cc(r[k], C::P(k));
  uint32_t t = subc(top, 0);  // 0xffffffff iff (top:r) < p
  bool keep = (t >> 31) != 0;
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = keep ? r[k] : d[k];
}

template <class C>
NMSM_HD void mont_mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = C::N;
  static_assert(N % 2 == 0, "even limb count expected");
  uint32_t E[2 * N + 2], O[2 * N + 2];
#pragma unroll
  for (int k = 0; k < 2 * N + 2; k++) {
    E[k] = 0;
    O[k] = 0;
  }
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint32_t* P1 = (i & 1) ? O : E;  // slots aligned at position i
    uint32_t* P2 = (i & 1) ? E : O;  // slots aligned at position i+1; P2[i] = leftover high half
    const uint32_t w = b[i];
    // fold the leftover high half into limb i; carry continues into P2's chain at position i+1
    if (i > 0) P1[i] = add_cc(P1[i], P2[i]);
#pragma unroll
    for (int j = 1; j < N; j += 2) {
      P2[i + j] = (i == 0 && j == 1) ? mad_lo_cc(a[j], w, P2[i + j]) : madc_lo_cc(a[j], w, P2[i + j]);
      P2[i + j + 1] = madc_hi_cc(a[j], w, P2[i + j + 1]);
    }
    P2[i + N + 1] = addc(P2[i + N + 1], 0);
#pragma unroll
    for (int j = 0; j < N; j += 2) {
      P1[i + j] = (j == 0) ? mad_lo_cc(a[j], w, P1[i + j]) : madc_lo_cc(a[j], w, P1[i + j]);
      P1[i + j + 1] = madc_hi_cc(a[j], w, P1[i + j + 1]);
    }
    P1[i + N] = addc(P1[i + N], 0);
    // Montgomery quotient digit: makes limb i vanish
    const uint32_t m = P1[i] * C::INV;
#pragma unroll
    for (int j = 1; j < N; j += 2) {
      P2[i + j] = (j == 1) ? mad_lo_cc(m, C::P(j), P2[i + j]) : madc_lo_cc(m, C::P(j), P2[i + j]);
      P2[i + j + 1] = madc_hi_cc(m, C::P(j), P2[i + j + 1]);
    }
    P2[i + N + 1] = addc(P2[i + N + 1], 0);
#pragma unroll
    for (int j = 0; j < N; j += 2) {
      P1[i + j] = (j == 0) ? mad_lo_cc(m, C::P(j), P1[i + j]) : madc_lo_cc(m, C::P(j), P1[i + j]);
      P1[i + j + 1] = madc_hi_cc(m, C::P(j), P1[i + j + 1]);
    }
    P1[i + N] = addc(P1[i + N], 0);
  }
  // merge the two column arrays: limbs N..2N
  r[0] = add_cc(E[N], O[N]);
#pragma unroll
  for (int k = 1; k < N; k++) r[k] = addc_cc(E[N + k], O[N + k]);
  uint32_t top = addc(E[2 * N], O[2 * N]);
  reduce_once<C>(r, top);
}

// Montgomery squaring, SOS order: the n(n-1)/2 off-diagonal products are formed once and doubled
// (a one-bit shift of both column arrays), the n diagonal squares are added, then the n reduction rows
// run as in mont_mul.  IMAD.WIDE-equivalents: n(n-1)/2 + n + n^2 + n  (n = 12: 234 vs 300; n = 8: 108 vs 136).
// The reduction rows now add into limbs that already hold product bits, so their chain-end carries are
// collected in a separate small-count array (Cw) and merged at the end.
template <class C>
NMSM_HD void mont_sqr(uint32_t* r, const uint32_t* a) {
  constexpr int N = C::N;
  uint32_t E[2 * N + 2], O[2 * N + 2], Cw[2 * N + 2];
#pragma unroll
  for (int k = 0; k < 2 * N + 2; k++) {
    E[k] = 0;
    O[k] = 0;
    Cw[k] = 0;
  }
  // A1: off-diagonal products a_i * a_j (i < j) at absolute position i + j
#pragma unroll
  for (int i = 0; i < N - 1; i++) {
    // (i + j) even -> E
    if (i + 2 < N) {
#pragma unroll
      for (int j = i + 2; j < N; j += 2) {
        E[i + j] = (j == i + 2) ? mad_lo_cc(a[i], a[j], E[i + j]) : madc_lo_cc(a[i], a[j], E[i + j]);
        E[i + j + 1] = madc_hi_cc(a[i], a[j], E[i + j + 1]);
      }
      const int last = i + 2 + 2 * ((N - 1 - (i + 2)) / 2);  // largest j used
      E[i + last + 2] = addc(E[i + last + 2], 0);
    }
    // (i + j) odd -> O
#pragma unroll
    for (int j = i + 1; j < N; j += 2) {
      O[i + j] = (j == i + 1) ? mad_lo_cc(a[i], a[j], O[i + j]) : madc_lo_cc(a[i], a[j], O[i + j]);
      O[i + j + 1] = madc_hi_cc(a[i], a[j], O[i + j + 1]);
    }
    {
      const int last = i + 1 + 2 * ((N - 1 - (i + 1)) / 2);
      O[i + last + 2] = addc(O[i + last + 2], 0);
    }
  }
  // A2: double both column arrays (value(E) + value(O) is the off-diagonal sum)
#pragma unroll
  for (int k = 2 * N + 1; k >= 1; k--) {
    E[k] = (E[k] << 1) | (E[k - 1] >> 31);
    O[k] = (O[k] << 1) | (O[k - 1] >> 31);
  }
  E[0] <<= 1;
  O[0] <<= 1;
  // A3: diagonal squares a_i^2 at position 2i: one chain along E
#pragma unroll
  for (int i = 0; i < N; i++) {
    E[2 * i] = (i == 0) ? mad_lo_cc(a[i], a[i], E[2 * i]) : madc_lo_cc(a[i], a[i], E[2 * i]);
    E[2 * i + 1] = madc_hi_cc(a[i], a[i], E[2 * i + 1]);
  }
  E[2 * N] = addc(E[2 * N], 0);
  // B: Montgomery reduction rows
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint32_t* P1 = (i & 1) ? O : E;
    uint32_t* P2 = (i & 1) ? E : O;
    if (i > 0) P1[i] = add_cc(P1[i], P2[i]);  // carry continues into P2's chain at position i+1
    const uint32_t m = P1[i] * C::INV;
#pragma unroll
    for (int j = 1; j < N; j += 2) {
      P2[i + j] = (i == 0 && j == 1) ? mad_lo_cc(m, C::P(j), P2[i + j]) : madc_lo_cc(m, C::P(j), P2[i + j]);
      P2[i + j + 1] = madc_hi_cc(m, C::P(j), P2[i + j + 1]);
    }
    Cw[i + N + 1] = addc(Cw[i + N + 1], 0);
#pragma unroll
    for (int j = 0; j < N; j += 2) {
      P1[i + j] = (j == 0) ? mad_lo_cc(m, C::P(j), P1[i + j]) : madc_lo_cc(m, C::P(j), P1[i + j]);
      P1[i + j + 1] = madc_hi_cc(m, C::P(j), P1[i + j + 1]);
    }
    Cw[i + N] = addc(Cw[i + N], 0);
  }
  // merge limbs N..2N of E + O + Cw
  r[0] = add_cc(E[N], O[N]);
#pragma unroll
  for (int k = 1; k < N; k++) r[k] = addc_cc(E[N + k], O[N + k]);
  uint32_t top = addc(E[2 * N], O[2 * N]);
  r[0] = add_cc(r[0], Cw[N]);
#pragma unroll
  for (int k = 1; k < N; k++) r[k] = addc_cc(r[k], Cw[N + k]);
  top = addc(top, Cw[2 * N]);
  reduce_once<C>(r, top);
}

// ---- building blocks of the lazily reduced Fp2 multiplication (fp2.cuh) ----------------------------------------
// T = a * b as a plain 2N-limb integer (operands need not be reduced: any N-limb values).  Products are placed by the
// parity of their absolute position (i + j), so every row is one carry chain per column array, as in mont_sqr.
template <class C>
NMSM_HD void mul_wide(uint32_t* T, const uint32_t* a, const uint32_t* b) {
  constexpr int N = C::N;
  uint32_t E[2 * N + 2], O[2 * N + 2];
#pragma unroll
  for (int k = 0; k < 2 * N + 2; k++) {
    E[k] = 0;
    O[k] = 0;
  }
#pragma unroll
  for (int i = 0; i < N; i++) {
    const uint32_t w = b[i];
    const int j0e = i & 1, j0o = 1 - (i & 1);  // first j with (i + j) even / odd
#pragma unroll
    for (int j = j0e; j < N; j += 2) {
      E[i + j] = (j == j0e) ? mad_lo_cc(a[j], w, E[i + j]) : madc_lo_cc(a[j], w, E[i + j]);
      E[i + j + 1] = madc_hi_cc(a[j], w, E[i + j + 1]);
    }
    {
      const int last = j0e + 2 * ((N - 1 - j0e) / 2);
      E[i + last + 2] = addc(E[i + last + 2], 0);
    }
#pragma unroll
    for (int j = j0o; j < N; j += 2) {
      O[i + j] = (j == j0o) ? mad_lo_cc(a[j], w, O[i + j]) : madc_lo_cc(a[j], w, O[i + j]);
      O[i + j + 1] = madc_hi_cc(a[j], w, O[i + j + 1]);
    }
    {
      const int last = j0o + 2 * ((N - 1 - j0o) / 2);
      O[i + last + 2] = addc(O[i + last + 2], 0);
    }
  }
  T[0] = add_cc(E[0], O[0]);
#pragma unroll
  for (int k = 1; k < 2 * N; k++) T[k] = addc_cc(E[k], O[k]);
}

// r = T / R mod p, fully reduced, for a plain 2N-limb T < p * R / 2 (so that the result before the final conditional
// subtraction is below 2p): the N reduction rows of mont_sqr on E = T, O = 0.
template <class C>
NMSM_HD void mont_reduce_wide(uint32_t* r, const uint32_t* T) {
  constexpr int N = C::N;
  uint32_t E[2 * N + 2], O[2 * N + 2], Cw[2 * N + 2];
#pragma unroll
  for (int k = 0; k < 2 * N + 2; k++) {
    E[k] = k < 2 * N ? T[k] : 0u;
    O[k] = 0;
    Cw[k] = 0;
  }
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint32_t* P1 = (i & 1) ? O : E;
    uint32_t* P2 = (i & 1) ? E : O;
    if (i > 0) P1[i] = add_cc(P1[i], P2[i]);  // carry continues into P2's chain at position i+1
    const uint32_t m = P1[i] * C::INV;
#pragma unroll
    for (int j = 1; j < N; j += 2) {
      P2[i + j] = (i == 0 && j == 1) ? mad_lo_cc(m, C::P(j), P2[i + j]) : madc_lo_cc(m, C::P(j), P2[i + j]);
      P2[i + j + 1] = madc_hi_cc(m, C::P(j), P2[i + j + 1]);
    }
    Cw[i + N + 1] = addc(Cw[i + N + 1], 0);
#pragma unroll
    for (int j = 0; j < N; j += 2) {
      P1[i + j] = (j == 0) ? mad_lo_cc(m, C::P(j), P1[i + j]) : madc_lo_cc(m, C::P(j), P1[i + j]);
      P1[i + j + 1] = madc_hi_cc(m, C::P(j), P1[i + j + 1]);
    }
    Cw[i + N] = addc(Cw[i + N], 0);
  }
  r[0] = add_cc(E[N], O[N]);
#pragma unroll
  for (int k = 1; k < N; k++) r[k] = addc_cc(E[N + k], O[N + k]);
  uint32_t top = addc(E[2 * N], O[2 * N]);
  r[0] = add_cc(r[0], Cw[N]);
#pragma unroll
  for (int k = 1; k < N; k++) r[k] = addc_cc(r[k], Cw[N + k]);
  top = addc(top, Cw[2 * N]);
  reduce_once<C>(r, top);
}

// limb k of p * R / 4 = p << (32 N - 2) as a 2N-limb integer: the multiple of p added before a double-width
// subtraction so that the difference stays non-negative (p < R / 4 for every field here, hence p^2 <= p R / 4)
template <class C>
NMSM_HD constexpr uint32_t p_times_quarter_r(int k) {
  constexpr int N = C::N;
  const int w = k - (N - 1);  // p << 30 placed at word N - 1
  if (w < 0 || w > N) return 0u;
  const uint32_t lo = w >= 1 ? (C::P(w - 1) >> 2) : 0u;
  const uint32_t hi = w < N ? (C::P(w) << 30) : 0u;
  return lo | hi;
}

template <class C>
struct Fp;
#if defined(__CUDACC__)
template <class C>
__device__ __noinline__ Fp<C> mul_call(Fp<C> a, Fp<C> b);
template <class C>
__device__ __noinline__ Fp<C> sqr_call(Fp<C> a);
#endif

template <class C>
struct Fp {
  static constexpr int N = C::N;
  static constexpr int LIMBS = C::N;    // 32-bit words per element
  static constexpr int BASE_MULS = 1;   // base-field multiplications per mul (accounting)
  static constexpr int BASE_SQRS = 1;
  using Params = C;
  uint32_t v[N];

  NMSM_HD static Fp zero() {
    Fp r;
#pragma unroll
    for (int k = 0; k < N; k++) r.v[k] = 0;
    return r;
  }
  NMSM_HD static Fp one() {  // Montgomery form of 1
    Fp r;
#pragma unroll
    for (int k = 0; k < N; k++) r.v[k] = C::R1(k);
    return r;
  }
  NMSM_HD bool is_zero() const {
    uint32_t t = 0;
#pragma unroll
    for (int k = 0; k < N; k++) t |= v[k];
    return t == 0;
  }
  NMSM_HD bool operator==(const Fp& o) const {
    uint32_t t = 0;
#pragma unroll
    for (int k = 0; k < N; k++) t |= v[k] ^ o.v[k];
    return t == 0;
  }
  NMSM_HD bool operator!=(const Fp& o) const { return !(*this == o); }

  NMSM_HD friend Fp operator*(const Fp& a, const Fp& b) {
#if defined(__CUDA_ARCH__) && defined(NMSM_MUL_NOINLINE)
    return mul_call<C>(a, b);  // one shared copy of the 2N^2+N IMAD body: instruction-cache friendly
#else
    Fp r;
    mont_mul<C>(r.v, a.v, b.v);
    return r;
#endif
  }
  NMSM_HD friend Fp operator+(const Fp& a, const Fp& b) {
    Fp r;
    r.v[0] = add_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int k = 1; k < N; k++) r.v[k] = addc_cc(a.v[k], b.v[k]);
    uint32_t top = addc(0, 0);
    reduce_once<C>(r.v, top);
    return r;
  }
  NMSM_HD friend Fp operator-(const Fp& a, const Fp& b) {
    Fp r;
    r.v[0] = sub_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int k = 1; k < N; k++) r.v[k] = subc_cc(a.v[k], b.v[k]);
    uint32_t mask = subc(0, 0);  // all ones iff a < b
    r.v[0] = add_cc(r.v[0], C::P(0) & mask);
#pragma unroll
    for (int k = 1; k < N; k++) r.v[k] = addc_cc(r.v[k], C::P(k) & mask);
    return r;
  }
  NMSM_HD Fp operator-() const { return zero() - *this; }

  // canonical little-endian limbs <-> Montgomery
  NMSM_HD static Fp from_canonical(const uint32_t* x) {
    Fp a, r2;
#pragma unroll
    for (int k = 0; k < N; k++) {
      a.v[k] = x[k];
      r2.v[k] = C::R2(k);
    }
    return a * r2;
  }
  NMSM_HD void to_canonical(uint32_t* x) const {
    Fp o;
#pragma unroll
    for (int k = 0; k < N; k++) o.v[k] = (k == 0) ? 1u : 0u;
    Fp r = (*this) * o;
#pragma unroll
    for (int k = 0; k < N; k++) x[k] = r.v[k];
  }
  // x < p as canonical integer?
  NMSM_HD static bool canonical_in_range(const uint32_t* x) {
    uint32_t t = sub_cc(x[0], C::P(0));
#pragma unroll
    for (int k = 1; k < N; k++) t = subc_cc(x[k], C::P(k));
    (void)t;
    return subc(0, 0) != 0;  // borrow => x < p
  }
};

#if defined(__CUDACC__)
template <class C>
__device__ __noinline__ Fp<C> mul_call(Fp<C> a, Fp<C> b) {
  Fp<C> r;
  mont_mul<C>(r.v, a.v, b.v);
  return r;
}
template <class C>
__device__ __noinline__ Fp<C> sqr_call(Fp<C> a) {
  Fp<C> r;
  mont_sqr<C>(r.v, a.v);
  return r;
}
#endif

template <class C>
NMSM_HD Fp<C> sqr(const Fp<C>& a) {
#if defined(__CUDA_ARCH__) && defined(NMSM_MUL_NOINLINE)
  return sqr_call<C>(a);
#else
  Fp<C> r;
  mont_sqr<C>(r.v, a.v);
  return r;
#endif
}
template <class C>
NMSM_HD Fp<C> dbl(const Fp<C>& a) {
  return a + a;
}

// Modular inverse by a binary extended GCD on the limbs (modular.ts:980 `inv` -> :159-182; the reference runs extended
// Euclid on BigInt): ~2*BITS shift/subtract steps.  Since round 2 this is only the FALLBACK of nmsm::inv
// (inv_divsteps.cuh, batched division steps, several times faster for a lone warp).
// Input and output in Montgomery form; 0 maps to 0.
template <class C>
NMSM_HD Fp<C> inv_xgcd(const Fp<C>& a) {
  constexpr int N = C::N;
  if (a.is_zero()) return a;
  // invariants: a * x1 == u (mod p), a * x2 == v (mod p), with a taken as the raw limbs
  uint32_t u[N], v[N], x1[N], x2[N];
#pragma unroll
  for (int k = 0; k < N; k++) {
    u[k] = a.v[k];
    v[k] = C::P(k);
    x1[k] = (k == 0) ? 1u : 0u;
    x2[k] = 0u;
  }
  auto is_one = [](const uint32_t* x) {
    uint32_t t = x[0] ^ 1u;
#pragma unroll
    for (int k = 1; k < N; k++) t |= x[k];
    return t == 0;
  };
  auto halve = [](uint32_t* x, uint32_t top) {  // (top:x) >> 1
#pragma unroll
    for (int k = 0; k < N - 1; k++) x[k] = (x[k] >> 1) | (x[k + 1] << 31);
    x[N - 1] = (x[N - 1] >> 1) | (top << 31);
  };
  auto halve_mod = [&](uint32_t* x) {  // x/2 mod p
    uint32_t top = 0;
    if (x[0] & 1u) {
      x[0] = add_cc(x[0], C::P(0));
#pragma unroll
      for (int k = 1; k < N; k++) x[k] = addc_cc(x[k], C::P(k));
      top = addc(0, 0);
    }
    halve(x, top);
  };
  auto geq = [](const uint32_t* x, const uint32_t* y) {  // x >= y
    uint32_t t = sub_cc(x[0], y[0]);
#pragma unroll
    for (int k = 1; k < N; k++) t = subc_cc(x[k], y[k]);
    (void)t;
    return subc(0, 0) == 0;
  };
  auto sub_plain = [](uint32_t* x, const uint32_t* y) {  // x -= y (x >= y)
    x[0] = sub_cc(x[0], y[0]);
#pragma unroll
    for (int k = 1; k < N; k++) x[k] = subc_cc(x[k], y[k]);
  };
  auto sub_mod = [](uint32_t* x, const uint32_t* y) {  // x = x - y mod p
    x[0] = sub_cc(x[0], y[0]);
#pragma unroll
    for (int k = 1; k < N; k++) x[k] = subc_cc(x[k], y[k]);
    uint32_t mask = subc(0, 0);
    x[0] = add_cc(x[0], C::P(0) & mask);
#pragma unroll
    for (int k = 1; k < N; k++) x[k] = addc_cc(x[k], C::P(k) & mask);
  };
  while (!is_one(u) && !is_one(v)) {
    while (!(u[0] & 1u)) {
      halve(u, 0);
      halve_mod(x1);
    }
    while (!(v[0] & 1u)) {
      halve(v, 0);
      halve_mod(x2);
    }
    if (geq(u, v)) {
      sub_plain(u, v);
      sub_mod(x1, x2);
    } else {
      sub_plain(v, u);
      sub_mod(x2, x1);
    }
  }
  Fp<C> r, r2;
  const bool pick_u = is_one(u);
#pragma unroll
  for (int k = 0; k < N; k++) {
    r.v[k] = pick_u ? x1[k] : x2[k];
    r2.v[k] = C::R2(k);
  }
  // raw inverse of aR is a^-1 R^-1; two Montgomery multiplications by R^2 lift it to a^-1 R
  return (r * r2) * r2;
}

}  // namespace nmsm
