// The pairing towers over the BLS12-381 and bn254 base fields (SURVEY §8 rows f7, f8), the reference's
// src/abstract/tower.ts:
//   Fp6  = Fp2[v]/(v^3 - xi),  xi = 1 + u (BLS12-381), 9 + u (bn254)
//   Fp12 = Fp6[w]/(w^2 - v)
// An Fp12 element is c0 + c1 w with c0, c1 in Fp6; an Fp6 element is c0 + c1 v + c2 v^2 with coefficients in Fp2.  The
// memory order (c0.c0.c0, c0.c0.c1, c0.c1.c0, ..., c1.c2.c1; 12 Fp values of N words, Montgomery form) is the order
// the pairing workspace and tests/hostemu use.
//
// The tower is a template over a policy T (field parameters, multiplication by xi, Frobenius coefficients, the curve
// parameter x of the cyclotomic exponentiation): Bls381Tower and Bn254Tower.  The heavy operations are out of line on
// the device (NMSM_HD_NOINLINE): one copy of each body keeps the pairing kernels' code size and ptxas time reasonable.
// `inline` gives the host copies of the non-template ones (pairing.cuh) one definition per program, so more than one
// translation unit can include them (inst_bls381_pairing.cu and inst_kzg.cu); the device calls stay out of line.
#pragma once
#include "curve_consts.cuh"
#include "fp2.cuh"

namespace nmsm {

#if defined(__CUDACC__)
#define NMSM_HD_NOINLINE inline __host__ __device__ __noinline__
#else
#define NMSM_HD_NOINLINE inline
#endif

// Frobenius^K coefficients of a generated block Fr (tools/gen_consts.py Bls381Frob, Bn254Frob):
// v -> c1 v, v^2 -> c2 v^2, w -> cw w
template <class Fr, int K, class F2>
NMSM_HD void frob_coeffs_from(F2& c1, F2& c2, F2& cw) {
#define NMSM_FROB_LD(dst, NAME)          \
  dst.c0.v[i] = Fr::NAME##_C0_MONT(i); \
  dst.c1.v[i] = Fr::NAME##_C1_MONT(i)
  for (int i = 0; i < F2::Params::N; i++) {
    if constexpr (K == 1) {
      NMSM_FROB_LD(c1, FROB6_C1_1);
      NMSM_FROB_LD(c2, FROB6_C2_1);
      NMSM_FROB_LD(cw, FROB12_C1_1);
    } else if constexpr (K == 2) {
      NMSM_FROB_LD(c1, FROB6_C1_2);
      NMSM_FROB_LD(c2, FROB6_C2_2);
      NMSM_FROB_LD(cw, FROB12_C1_2);
    } else {
      static_assert(K == 3, "Frobenius powers 1..3");
      NMSM_FROB_LD(c1, FROB6_C1_3);
      NMSM_FROB_LD(c2, FROB6_C2_3);
      NMSM_FROB_LD(cw, FROB12_C1_3);
    }
  }
#undef NMSM_FROB_LD
}

struct Bls381Tower {
  using C = FpBls381;
  using F = Fp<FpBls381>;
  using F2 = Fp2<FpBls381>;
  NMSM_HD static F2 mul_by_xi(const F2& a) { return F2{a.c0 - a.c1, a.c0 + a.c1}; }  // (a0 + a1 u)(1 + u)
  template <int K>
  NMSM_HD static void frob_coeffs(F2& c1, F2& c2, F2& cw) {
    frob_coeffs_from<Bls381Frob, K>(c1, c2, cw);
  }
  // |x| = Bls381G2Gls::Z = 0xd201000000010000, the exponent of fp12_cyclotomic_exp_x
  static constexpr int X_BITS = 64;
  NMSM_HD static constexpr uint32_t X(int i) { return Bls381G2Gls::Z(i); }
};

struct Bn254Tower {
  using C = FpBn254;
  using F = Fp<FpBn254>;
  using F2 = Fp2<FpBn254>;
  NMSM_HD static F2 mul_by_xi(const F2& a) {  // (a0 + a1 u)(9 + u) = (9 a0 - a1) + (a0 + 9 a1) u
    const F2 a2 = a + a, a4 = a2 + a2, a9 = a4 + a4 + a;
    return F2{a9.c0 - a.c1, a.c0 + a9.c1};
  }
  template <int K>
  NMSM_HD static void frob_coeffs(F2& c1, F2& c2, F2& cw) {
    frob_coeffs_from<Bn254Frob, K>(c1, c2, cw);
  }
  // u = Bn254Ate::U = 0x44e992b44a6909f1, the exponent of fp12_cyclotomic_exp_x
  static constexpr int X_BITS = Bn254Ate::U_BITS;
  NMSM_HD static constexpr uint32_t X(int i) { return Bn254Ate::U(i); }
};

template <class T>
struct Fp6 {
  using F2 = typename T::F2;
  F2 c0, c1, c2;
  NMSM_HD static Fp6 zero() { return Fp6{F2::zero(), F2::zero(), F2::zero()}; }
  NMSM_HD static Fp6 one() { return Fp6{F2::one(), F2::zero(), F2::zero()}; }
  NMSM_HD friend Fp6 operator+(const Fp6& a, const Fp6& b) { return Fp6{a.c0 + b.c0, a.c1 + b.c1, a.c2 + b.c2}; }
  NMSM_HD friend Fp6 operator-(const Fp6& a, const Fp6& b) { return Fp6{a.c0 - b.c0, a.c1 - b.c1, a.c2 - b.c2}; }
  NMSM_HD Fp6 operator-() const { return Fp6{-c0, -c1, -c2}; }
  NMSM_HD bool operator==(const Fp6& o) const { return c0 == o.c0 && c1 == o.c1 && c2 == o.c2; }
};

template <class T>
struct Fp12 {
  using F6 = Fp6<T>;
  static constexpr int WORDS = 12 * T::C::N;
  F6 c0, c1;
  NMSM_HD static Fp12 one() { return Fp12{F6::one(), F6::zero()}; }
  NMSM_HD bool is_one() const { return c0 == F6::one() && c1 == F6::zero(); }
  NMSM_HD bool operator==(const Fp12& o) const { return c0 == o.c0 && c1 == o.c1; }
  NMSM_HD void load(const uint32_t* src) {
    uint32_t* d = reinterpret_cast<uint32_t*>(this);
    for (int k = 0; k < WORDS; k++) d[k] = src[k];
  }
  NMSM_HD void store(uint32_t* dst) const {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(this);
    for (int k = 0; k < WORDS; k++) dst[k] = s[k];
  }
};

// ---- Fp6 --------------------------------------------------------------------------------------------------------
template <class T>
NMSM_HD Fp6<T> fp6_mul_by_v(const Fp6<T>& a) {  // (c0 + c1 v + c2 v^2) v = xi c2 + c0 v + c1 v^2
  return Fp6<T>{T::mul_by_xi(a.c2), a.c0, a.c1};
}

// Karatsuba: 6 Fp2 multiplications
template <class T>
NMSM_HD_NOINLINE Fp6<T> fp6_mul(const Fp6<T>& a, const Fp6<T>& b) {
  using F2 = typename T::F2;
  const F2 t0 = a.c0 * b.c0, t1 = a.c1 * b.c1, t2 = a.c2 * b.c2;
  const F2 r0 = T::mul_by_xi((a.c1 + a.c2) * (b.c1 + b.c2) - t1 - t2) + t0;
  const F2 r1 = (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1 + T::mul_by_xi(t2);
  const F2 r2 = (a.c0 + a.c2) * (b.c0 + b.c2) - t0 - t2 + t1;
  return Fp6<T>{r0, r1, r2};
}

// Chung-Hasan SQR2: 2 Fp2 multiplications and 3 squarings
template <class T>
NMSM_HD_NOINLINE Fp6<T> fp6_sqr(const Fp6<T>& a) {
  using F2 = typename T::F2;
  const F2 s0 = sqr(a.c0), ab = a.c0 * a.c1, s1 = ab + ab, s2 = sqr(a.c0 - a.c1 + a.c2), bc = a.c1 * a.c2,
           s3 = bc + bc, s4 = sqr(a.c2);
  return Fp6<T>{s0 + T::mul_by_xi(s3), s1 + T::mul_by_xi(s4), s1 + s2 + s3 - s0 - s4};
}

// a (b0 + b1 v): 5 Fp2 multiplications
template <class T>
NMSM_HD Fp6<T> fp6_mul_by_01(const Fp6<T>& a, const typename T::F2& b0, const typename T::F2& b1) {
  using F2 = typename T::F2;
  const F2 t0 = a.c0 * b0, t1 = a.c1 * b1;
  return Fp6<T>{T::mul_by_xi(a.c2 * b1) + t0, (a.c0 + a.c1) * (b0 + b1) - t0 - t1, a.c2 * b0 + t1};
}

// a (b1 v): 3 Fp2 multiplications
template <class T>
NMSM_HD Fp6<T> fp6_mul_by_1(const Fp6<T>& a, const typename T::F2& b1) {
  return Fp6<T>{T::mul_by_xi(a.c2 * b1), a.c0 * b1, a.c1 * b1};
}

// through the norm to Fp2: a^-1 = (c0, c1, c2) / (a0 c0 + xi (a2 c1 + a1 c2))
template <class T>
NMSM_HD_NOINLINE Fp6<T> fp6_inv(const Fp6<T>& a) {
  using F2 = typename T::F2;
  const F2 c0 = sqr(a.c0) - T::mul_by_xi(a.c1 * a.c2);
  const F2 c1 = T::mul_by_xi(sqr(a.c2)) - a.c0 * a.c1;
  const F2 c2 = sqr(a.c1) - a.c0 * a.c2;
  const F2 t = inv(a.c0 * c0 + T::mul_by_xi(a.c2 * c1 + a.c1 * c2));
  return Fp6<T>{c0 * t, c1 * t, c2 * t};
}

// ---- Fp12 -------------------------------------------------------------------------------------------------------
// Karatsuba: 3 Fp6 multiplications
template <class T>
NMSM_HD_NOINLINE Fp12<T> fp12_mul(const Fp12<T>& a, const Fp12<T>& b) {
  using F6 = Fp6<T>;
  const F6 t0 = fp6_mul(a.c0, b.c0), t1 = fp6_mul(a.c1, b.c1);
  return Fp12<T>{t0 + fp6_mul_by_v(t1), fp6_mul(a.c0 + a.c1, b.c0 + b.c1) - t0 - t1};
}

// complex squaring: 2 Fp6 multiplications
template <class T>
NMSM_HD_NOINLINE Fp12<T> fp12_sqr(const Fp12<T>& a) {
  using F6 = Fp6<T>;
  const F6 t = fp6_mul(a.c0, a.c1);
  const F6 r0 = fp6_mul(a.c0 + a.c1, a.c0 + fp6_mul_by_v(a.c1)) - t - fp6_mul_by_v(t);
  return Fp12<T>{r0, t + t};
}

// f * (l0 + l1 v + l4 v w): the sparse shape of a Miller-loop line on the M-type twist (pairing.cuh)
template <class T>
NMSM_HD_NOINLINE Fp12<T> fp12_mul_by_014(const Fp12<T>& f, const typename T::F2& l0, const typename T::F2& l1,
                                         const typename T::F2& l4) {
  using F6 = Fp6<T>;
  const F6 t0 = fp6_mul_by_01(f.c0, l0, l1), t1 = fp6_mul_by_1(f.c1, l4);
  const F6 s = fp6_mul_by_01(f.c0 + f.c1, l0, l1 + l4);
  return Fp12<T>{t0 + fp6_mul_by_v(t1), s - t0 - t1};
}

// f * (l0 + l3 w + l4 v w): the sparse shape of a Miller-loop line on the D-type twist (pairing_bn254.cuh)
template <class T>
NMSM_HD_NOINLINE Fp12<T> fp12_mul_by_034(const Fp12<T>& f, const typename T::F2& l0, const typename T::F2& l3,
                                         const typename T::F2& l4) {
  using F6 = Fp6<T>;
  const F6 t0{f.c0.c0 * l0, f.c0.c1 * l0, f.c0.c2 * l0}, t1 = fp6_mul_by_01(f.c1, l3, l4);
  const F6 s = fp6_mul_by_01(f.c0 + f.c1, l0 + l3, l4);
  return Fp12<T>{t0 + fp6_mul_by_v(t1), s - t0 - t1};
}

template <class T>
NMSM_HD Fp12<T> fp12_conj(const Fp12<T>& a) {  // a^(p^6): w -> -w
  return Fp12<T>{a.c0, -a.c1};
}

template <class T>
NMSM_HD_NOINLINE Fp12<T> fp12_inv(const Fp12<T>& a) {  // (c0 - c1 w) / (c0^2 - v c1^2)
  using F6 = Fp6<T>;
  const F6 t = fp6_inv(fp6_sqr(a.c0) - fp6_mul_by_v(fp6_sqr(a.c1)));
  return Fp12<T>{fp6_mul(a.c0, t), -fp6_mul(a.c1, t)};
}

// a^(p^K), K = 1..3: conjugate every Fp2 coefficient K times, then scale the v, v^2 and w coordinates
template <int K, class T>
NMSM_HD_NOINLINE Fp12<T> fp12_frobenius(const Fp12<T>& a) {
  using F2 = typename T::F2;
  using F6 = Fp6<T>;
  F2 k1, k2, kw;
  T::template frob_coeffs<K>(k1, k2, kw);
  auto fr = [](const F2& x) { return (K & 1) ? F2{x.c0, -x.c1} : x; };
  auto fr6 = [&](const F6& x) { return F6{fr(x.c0), fr(x.c1) * k1, fr(x.c2) * k2}; };
  const F6 r0 = fr6(a.c0), r1 = fr6(a.c1);
  return Fp12<T>{r0, F6{r1.c0 * kw, r1.c1 * kw, r1.c2 * kw}};
}

// Granger-Scott squaring, valid in the cyclotomic subgroup (a^(p^6 + 1) = 1): Fp12 seen as Fp4^3 with
// Fp4 = Fp2[w^3]/((w^3)^2 - xi), three Fp4 squarings = 6 Fp2 squarings
template <class T>
NMSM_HD void fp4_sqr(const typename T::F2& a, const typename T::F2& b, typename T::F2& c0, typename T::F2& c1) {
  using F2 = typename T::F2;
  const F2 t0 = sqr(a), t1 = sqr(b);
  c0 = T::mul_by_xi(t1) + t0;
  c1 = sqr(a + b) - t0 - t1;
}

template <class T>
NMSM_HD_NOINLINE Fp12<T> fp12_cyclotomic_sqr(const Fp12<T>& f) {
  using F2 = typename T::F2;
  F2 z0 = f.c0.c0, z4 = f.c0.c1, z3 = f.c0.c2, z2 = f.c1.c0, z1 = f.c1.c1, z5 = f.c1.c2;
  F2 t0, t1, t2, t3;
  fp4_sqr<T>(z0, z1, t0, t1);
  z0 = t0 - z0;
  z0 = z0 + z0 + t0;
  z1 = t1 + z1;
  z1 = z1 + z1 + t1;
  fp4_sqr<T>(z2, z3, t0, t1);
  fp4_sqr<T>(z4, z5, t2, t3);
  z4 = t0 - z4;
  z4 = z4 + z4 + t0;
  z5 = t1 + z5;
  z5 = z5 + z5 + t1;
  t0 = T::mul_by_xi(t3);
  z2 = t0 + z2;
  z2 = z2 + z2 + t0;
  z3 = t2 - z3;
  z3 = z3 + z3 + t2;
  return Fp12<T>{Fp6<T>{z0, z4, z3}, Fp6<T>{z2, z1, z5}};
}

// a^x in the cyclotomic subgroup for the policy's exponent x = T::X (a top bit and X_BITS - 1 more): X_BITS - 1
// squarings and one multiplication per further set bit (BLS12-381 |x|: 63 and 5; bn254 u: 62 and 27)
template <class T>
NMSM_HD_NOINLINE Fp12<T> fp12_cyclotomic_exp_x(const Fp12<T>& a) {
  Fp12<T> r = a;
  for (int i = T::X_BITS - 2; i >= 0; i--) {
    r = fp12_cyclotomic_sqr(r);
    const uint32_t bit = i >= 32 ? (T::X(1) >> (i - 32)) & 1u : (T::X(0) >> i) & 1u;
    if (bit) r = fp12_mul(r, a);
  }
  return r;
}

}  // namespace nmsm
