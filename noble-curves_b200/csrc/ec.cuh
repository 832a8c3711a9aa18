// Group law policies used by every kernel (MSM buckets, batched scalar multiplication, folds).
//
// The reference (SURVEY §8 a7-a13) uses complete formulas on homogeneous projective / extended
// coordinates (weierstrass.ts:793-880 RCB, edwards.ts:505-545 hwcd).  Results are only defined up
// to the projective representative, so parity is on canonical affine (x, y) (test/point.test.ts:36-44).
// Here:
//   * short Weierstrass a = 0 (secp256k1, bn254 G1/G2, BLS12-381 G1/G2): XYZZ accumulators
//     (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2; identity <=> ZZ == 0) with affine mixed addition
//     madd-2008-s (8M+2S), add-2008-s (12M+2S), dbl-2008-s-1 (6M+3S for a=0), mdbl-2008-s-1.
//     The incomplete formulas are completed by explicit branches for P+P, P+(-P), O+P, P+O — all
//     of which occur in the reference's own tests (point.test.ts:269,842-853).
//   * twisted Edwards a = -1 (ed25519): extended coordinates with the unified, complete
//     add-2008-hwcd-3 on prepared affine inputs (y-x, y+x, 2dxy) (7M) and dbl-2008-hwcd (4M+4S).
#pragma once
#include "curve_consts.cuh"
#include "field.cuh"
#include "inv_divsteps.cuh"
#include "fp2.cuh"

namespace nmsm {

// ------------------------------------------------------------------------------------------
// Lane-parallel field multiplications for the latency-bound tails (k_horner_step / k_combine / k_fold, k_reduce2, the
// owner kernels of a sharded MSM).
// The multiply pipe is occupied per WARP instruction (a lone thread pays ~0.95 us per 381-bit
// mont_mul, measured), so latency-bound phases run each logical thread on a QUAD of 4 adjacent lanes
// holding the same replicated state; at each level of a point formula lane (l & 3) computes one of up
// to four independent products and the results are broadcast back inside the quad with warp shuffles
// (quad-scoped masks, so different quads of a warp may diverge).
// ------------------------------------------------------------------------------------------
#if defined(__CUDACC__)
// FULLWARP = true: all 32 lanes hold the same state (k_horner_step / k_fold) and shuffles use the full mask;
// false: quads are independent logical threads (k_reduce2, k_combine, the dense kernels) and shuffles are quad-scoped.
template <class F, bool FULLWARP>
struct Par4 {
  static constexpr int WORDS = sizeof(F) / 4;
  // broadcast from lane `src` (0..3) of the caller's quad (4 adjacent lanes); quads may be divergent
  __device__ static __forceinline__ F bcast(const F& z, int src) {
    F r;
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&z);
    uint32_t* d = reinterpret_cast<uint32_t*>(&r);
    const unsigned qbase = FULLWARP ? 0u : (threadIdx.x & 28u);  // blocks are multiples of 32 threads
    const unsigned qmask = FULLWARP ? 0xffffffffu : (0xFu << qbase);
#pragma unroll
    for (int k = 0; k < WORDS; k++) d[k] = __shfl_sync(qmask, s[k], qbase + src);
    return r;
  }
  // lane-dependent operand choice by masks: a ternary chain here compiles to divergent branches (one BSSY/BSYNC region
  // per word — measured: 2x the cost of the multiplication it feeds), and the quad's lanes must not diverge
  __device__ static __forceinline__ F pick(int l, const F& a0, const F& a1, const F& a2, const F& a3) {
    F r;
    const uint32_t* p0 = reinterpret_cast<const uint32_t*>(&a0);
    const uint32_t* p1 = reinterpret_cast<const uint32_t*>(&a1);
    const uint32_t* p2 = reinterpret_cast<const uint32_t*>(&a2);
    const uint32_t* p3 = reinterpret_cast<const uint32_t*>(&a3);
    uint32_t* d = reinterpret_cast<uint32_t*>(&r);
    const uint32_t m0 = 0u - (uint32_t)(l == 0), m1 = 0u - (uint32_t)(l == 1), m2 = 0u - (uint32_t)(l == 2),
                   m3 = 0u - (uint32_t)(l == 3);
#pragma unroll
    for (int k = 0; k < WORDS; k++) d[k] = (p0[k] & m0) | (p1[k] & m1) | (p2[k] & m2) | (p3[k] & m3);
    return r;
  }
  // r_k = a_k * b_k for k < 4, one product per lane, every lane receives all four
  __device__ static __forceinline__ void mul4(F& r0, F& r1, F& r2, F& r3, const F& a0, const F& b0, const F& a1,
                                              const F& b1, const F& a2, const F& b2, const F& a3, const F& b3) {
    const int l = threadIdx.x & 3;
    F x = pick(l, a0, a1, a2, a3), y = pick(l, b0, b1, b2, b3);
    F z = x * y;
    r0 = bcast(z, 0);
    r1 = bcast(z, 1);
    r2 = bcast(z, 2);
    r3 = bcast(z, 3);
  }
};
#endif

// ------------------------------------------------------------------------------------------
// Short Weierstrass, a = 0
// ------------------------------------------------------------------------------------------
template <class F>
struct SwXyzz {
  using Field = F;
  static constexpr int COORD_WORDS = F::LIMBS;
  static constexpr int IN_WORDS = 2 * F::LIMBS;   // canonical affine input (x, y)
  static constexpr int AFF_WORDS = 2 * F::LIMBS;  // prepared affine
  static constexpr int ACC_WORDS = 4 * F::LIMBS;
  // multiplication counts in field-mul equivalents (1S = 1M), SURVEY §8(d)
  static constexpr int COST_MADD = 10, COST_ADD = 14, COST_DBL = 9;
  static constexpr bool IS_EDWARDS = false;

  struct Affine {
    F x, y;
  };
  struct Acc {
    F X, Y, ZZ, ZZZ;
  };

  NMSM_HD static Acc identity() { return Acc{F::zero(), F::one(), F::zero(), F::zero()}; }
  NMSM_HD static bool is_identity(const Acc& p) { return p.ZZ.is_zero(); }
  NMSM_HD static bool affine_is_identity(const Affine& a) { return a.x.is_zero() && a.y.is_zero(); }
  // weierstrass.ts:716 — affine (0,0) encodes the point at infinity
  NMSM_HD static Affine prepare(const uint32_t* xy) {
    return Affine{F::from_canonical(xy), F::from_canonical(xy + F::LIMBS)};
  }
  NMSM_HD static bool input_in_range(const uint32_t* xy) {
    return F::canonical_in_range(xy) && F::canonical_in_range(xy + F::LIMBS);
  }
  NMSM_HD static Affine neg(const Affine& a) { return Affine{a.x, -a.y}; }
  NMSM_HD static Affine cneg(const Affine& a, bool n) {
    F ny = -a.y;
    return Affine{a.x, n ? ny : a.y};
  }
  NMSM_HD static Acc from_affine(const Affine& a) {
    if (affine_is_identity(a)) return identity();
    return Acc{a.x, a.y, F::one(), F::one()};
  }
  NMSM_HD static Acc neg(const Acc& p) { return Acc{p.X, -p.Y, p.ZZ, p.ZZZ}; }

  // 2*(x, y) for an affine point: mdbl-2008-s-1
  NMSM_HD static Acc dbl_affine(const Affine& a) {
    F U = nmsm::dbl(a.y);
    F V = sqr(U);
    F W = U * V;
    F S = a.x * V;
    F xx = sqr(a.x);
    F M = nmsm::dbl(xx) + xx;
    F X3 = sqr(M) - nmsm::dbl(S);
    F Y3 = M * (S - X3) - W * a.y;
    return Acc{X3, Y3, V, W};  // y == 0 gives ZZ = 0 (identity), as it must for a 2-torsion point
  }
  // dbl-2008-s-1, a = 0
  NMSM_HD static void dbl(Acc& p) {
    if (is_identity(p)) return;
    F U = nmsm::dbl(p.Y);
    F V = sqr(U);
    F W = U * V;
    F S = p.X * V;
    F xx = sqr(p.X);
    F M = nmsm::dbl(xx) + xx;
    F X3 = sqr(M) - nmsm::dbl(S);
    F Y3 = M * (S - X3) - W * p.Y;
    p.ZZ = V * p.ZZ;
    p.ZZZ = W * p.ZZZ;
    p.X = X3;
    p.Y = Y3;
  }
  // p += a (affine): madd-2008-s with the exceptional cases handled explicitly.  INL: the field products of the
  // general case are expanded in place (field.cuh mul_inline), for k_accumulate's loop; the rare doubling stays shared.
  template <bool INL = false>
  NMSM_HD static void madd(Acc& p, const Affine& a) {
    auto mul = [](const F& x, const F& y) -> F {
      if constexpr (INL) return mul_inline(x, y);
      else return x * y;
    };
    auto sq = [](const F& x) -> F {
      if constexpr (INL) return sqr_inline(x);
      else return sqr(x);
    };
    if (affine_is_identity(a)) return;
    if (is_identity(p)) {
      p = Acc{a.x, a.y, F::one(), F::one()};
      return;
    }
    F U2 = mul(a.x, p.ZZ);
    F S2 = mul(a.y, p.ZZZ);
    F P = U2 - p.X;
    F R = S2 - p.Y;
    if (P.is_zero()) {
      if (R.is_zero())
        p = dbl_affine(a);
      else
        p = identity();
      return;
    }
    F PP = sq(P);
    F PPP = mul(P, PP);
    F Q = mul(p.X, PP);
    F X3 = sq(R) - PPP - nmsm::dbl(Q);
    F Y3 = mul(R, Q - X3) - mul(p.Y, PPP);
    p.ZZ = mul(p.ZZ, PP);
    p.ZZZ = mul(p.ZZZ, PPP);
    p.X = X3;
    p.Y = Y3;
  }
  // p += q: add-2008-s with exceptional cases
  NMSM_HD static void add(Acc& p, const Acc& q) {
    if (is_identity(q)) return;
    if (is_identity(p)) {
      p = q;
      return;
    }
    F U1 = p.X * q.ZZ;
    F U2 = q.X * p.ZZ;
    F S1 = p.Y * q.ZZZ;
    F S2 = q.Y * p.ZZZ;
    F P = U2 - U1;
    F R = S2 - S1;
    if (P.is_zero()) {
      if (R.is_zero())
        dbl(p);
      else
        p = identity();
      return;
    }
    F PP = sqr(P);
    F PPP = P * PP;
    F Q = U1 * PP;
    F X3 = sqr(R) - PPP - nmsm::dbl(Q);
    F Y3 = R * (Q - X3) - S1 * PPP;
    p.ZZ = p.ZZ * q.ZZ * PP;
    p.ZZZ = p.ZZZ * q.ZZZ * PPP;
    p.X = X3;
    p.Y = Y3;
  }
#if defined(__CUDACC__)
  // Warp-replicated versions of dbl / add (see Par4): 3 and 4 multiplication levels instead of 9 / 14.
  template <bool FW>
  __device__ static void par_dbl(Acc& p) {
    if (is_identity(p)) return;
    using P4 = Par4<F, FW>;
    F U = nmsm::dbl(p.Y);
    F V, A, t2, t3;
    P4::mul4(V, A, t2, t3, U, U, p.X, p.X, U, U, U, U);
    F M = nmsm::dbl(A) + A;
    F W, S, MM;
    P4::mul4(W, S, MM, t3, U, V, p.X, V, M, M, M, M);
    F X3 = MM - nmsm::dbl(S);
    F y0, y1, zz, zzz;
    P4::mul4(y0, y1, zz, zzz, M, S - X3, W, p.Y, V, p.ZZ, W, p.ZZZ);
    p.X = X3;
    p.Y = y0 - y1;
    p.ZZ = zz;
    p.ZZZ = zzz;
  }
  template <bool FW>
  __device__ static void par_add(Acc& p, const Acc& q) {
    if (is_identity(q)) return;
    if (is_identity(p)) {
      p = q;
      return;
    }
    using P4 = Par4<F, FW>;
    F U1, U2, S1, S2;
    P4::mul4(U1, U2, S1, S2, p.X, q.ZZ, q.X, p.ZZ, p.Y, q.ZZZ, q.Y, p.ZZZ);
    F P = U2 - U1;
    F R = S2 - S1;
    if (P.is_zero()) {
      if (R.is_zero())
        par_dbl<FW>(p);
      else
        p = identity();
      return;
    }
    F PP, RR, ZZ12, ZZZ12;
    P4::mul4(PP, RR, ZZ12, ZZZ12, P, P, R, R, p.ZZ, q.ZZ, p.ZZZ, q.ZZZ);
    F PPP, Q, ZZ3, t3;
    P4::mul4(PPP, Q, ZZ3, t3, P, PP, U1, PP, ZZ12, PP, P, PP);
    F X3 = RR - PPP - nmsm::dbl(Q);
    F y0, y1, ZZZ3;
    P4::mul4(y0, y1, ZZZ3, t3, R, Q - X3, S1, PPP, ZZZ12, PPP, R, R);
    p.X = X3;
    p.Y = y0 - y1;
    p.ZZ = ZZ3;
    p.ZZZ = ZZZ3;
  }
#endif
  // the value whose inverse normalisation needs (batched across a warp by k_table_mul); never zero
  NMSM_HD static F inv_target(const Acc& p) { return is_identity(p) ? F::one() : p.ZZZ; }
  // canonical affine output; identity -> (0, 0), flag 1 (weierstrass.ts:966)
  NMSM_HD static void to_affine_canonical(const Acc& p, uint32_t* xy, uint32_t* is_inf) {
    if (is_identity(p)) {
      for (int k = 0; k < 2 * F::LIMBS; k++) xy[k] = 0;
      *is_inf = 1;
      return;
    }
    to_affine_canonical_with_inv(p, inv(p.ZZZ), xy, is_inf);
  }
  NMSM_HD static void to_affine_canonical_with_inv(const Acc& p, const F& i3, uint32_t* xy, uint32_t* is_inf) {
    if (is_identity(p)) {
      for (int k = 0; k < 2 * F::LIMBS; k++) xy[k] = 0;
      *is_inf = 1;
      return;
    }
    F t = p.ZZ * i3;         // 1/Z  (i3 = 1/Z^3)
    F x = p.X * sqr(t);      // X / Z^2
    F y = p.Y * i3;          // Y / Z^3
    x.to_canonical(xy);
    y.to_canonical(xy + F::LIMBS);
    *is_inf = 0;
  }
  // Montgomery-form affine (the layout k_accumulate gathers); identity -> (0, 0)
  NMSM_HD static Affine to_affine_prepared(const Acc& p) {
    if (is_identity(p)) return Affine{F::zero(), F::zero()};
    F i3 = inv(p.ZZZ);
    F t = p.ZZ * i3;
    return Affine{p.X * sqr(t), p.Y * i3};
  }
  NMSM_HD static void store_acc(uint32_t* dst, const Acc& p) {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&p);
    for (int k = 0; k < ACC_WORDS; k++) dst[k] = s[k];
  }
};

// ------------------------------------------------------------------------------------------
// Twisted Edwards, a = -1 (ed25519)
// ------------------------------------------------------------------------------------------
template <class F, class K>
struct EdExt {
  using Field = F;
  static constexpr int COORD_WORDS = F::LIMBS;
  static constexpr int IN_WORDS = 2 * F::LIMBS;
  static constexpr int AFF_WORDS = 3 * F::LIMBS;
  static constexpr int ACC_WORDS = 4 * F::LIMBS;
  static constexpr int COST_MADD = 7, COST_ADD = 9, COST_DBL = 8;
  static constexpr bool IS_EDWARDS = true;

  struct Affine {
    F ymx, ypx, t2d;  // y-x, y+x, 2d*x*y
  };
  struct Acc {
    F X, Y, Z, T;
  };

  NMSM_HD static F d2() {
    F r;
    for (int k = 0; k < F::N; k++) r.v[k] = K::D2_MONT(k);
    return r;
  }
  NMSM_HD static Acc identity() { return Acc{F::zero(), F::one(), F::one(), F::zero()}; }
  NMSM_HD static bool is_identity(const Acc& p) { return p.X.is_zero() && p.Y == p.Z; }
  NMSM_HD static bool affine_is_identity(const Affine& a) { return a.t2d.is_zero() && a.ymx == a.ypx; }
  NMSM_HD static Affine prepare(const uint32_t* xy) {
    F x = F::from_canonical(xy), y = F::from_canonical(xy + F::LIMBS);
    return Affine{y - x, y + x, x * y * d2()};
  }
  NMSM_HD static bool input_in_range(const uint32_t* xy) {
    return F::canonical_in_range(xy) && F::canonical_in_range(xy + F::LIMBS);
  }
  // -(x, y) = (-x, y)
  NMSM_HD static Affine neg(const Affine& a) { return Affine{a.ypx, a.ymx, -a.t2d}; }
  NMSM_HD static Affine cneg(const Affine& a, bool n) {
    F nt = -a.t2d;
    return Affine{n ? a.ypx : a.ymx, n ? a.ymx : a.ypx, n ? nt : a.t2d};
  }
  NMSM_HD static Acc neg(const Acc& p) { return Acc{-p.X, p.Y, p.Z, -p.T}; }
  NMSM_HD static Acc from_affine(const Affine& a) {
    Acc r = identity();
    madd(r, a);
    return r;
  }
  // dbl-2008-hwcd, a = -1 (edwards.ts:505-521)
  NMSM_HD static void dbl(Acc& p) {
    F A = sqr(p.X);
    F B = sqr(p.Y);
    F C = nmsm::dbl(sqr(p.Z));
    F D = -A;
    F E = sqr(p.X + p.Y) - A - B;
    F G = D + B;
    F Fv = G - C;
    F H = D - B;
    p.X = E * Fv;
    p.Y = G * H;
    p.T = E * H;
    p.Z = Fv * G;
  }
  // add-2008-hwcd-3 with Z2 = 1 and precomputed (y2-x2, y2+x2, 2d*x2*y2): complete for a=-1, d non-square
  NMSM_HD static void madd(Acc& p, const Affine& a) {
    F A = (p.Y - p.X) * a.ymx;
    F B = (p.Y + p.X) * a.ypx;
    F C = p.T * a.t2d;
    F D = nmsm::dbl(p.Z);
    F E = B - A;
    F Fv = D - C;
    F G = D + C;
    F H = B + A;
    p.X = E * Fv;
    p.Y = G * H;
    p.T = E * H;
    p.Z = Fv * G;
  }
  NMSM_HD static void add(Acc& p, const Acc& q) {
    F A = (p.Y - p.X) * (q.Y - q.X);
    F B = (p.Y + p.X) * (q.Y + q.X);
    F C = p.T * d2() * q.T;
    F D = nmsm::dbl(p.Z * q.Z);
    F E = B - A;
    F Fv = D - C;
    F G = D + C;
    F H = B + A;
    p.X = E * Fv;
    p.Y = G * H;
    p.T = E * H;
    p.Z = Fv * G;
  }
#if defined(__CUDACC__)
  // Warp-replicated versions (see Par4): 2 levels for doubling, 3 for addition.
  template <bool FW>
  __device__ static void par_dbl(Acc& p) {
    using P4 = Par4<F, FW>;
    F A, B, Zs, XY;
    F xy = p.X + p.Y;
    P4::mul4(A, B, Zs, XY, p.X, p.X, p.Y, p.Y, p.Z, p.Z, xy, xy);
    F C = nmsm::dbl(Zs);
    F D = -A;
    F E = XY - A - B;
    F G = D + B;
    F Fv = G - C;
    F H = D - B;
    P4::mul4(p.X, p.Y, p.T, p.Z, E, Fv, G, H, E, H, Fv, G);
  }
  template <bool FW>
  __device__ static void par_add(Acc& p, const Acc& q) {
    using P4 = Par4<F, FW>;
    F A, B, TT, ZZ;
    P4::mul4(A, B, TT, ZZ, p.Y - p.X, q.Y - q.X, p.Y + p.X, q.Y + q.X, p.T, q.T, p.Z, q.Z);
    F C = TT * d2();
    F D = nmsm::dbl(ZZ);
    F E = B - A;
    F Fv = D - C;
    F G = D + C;
    F H = B + A;
    P4::mul4(p.X, p.Y, p.T, p.Z, E, Fv, G, H, E, H, Fv, G);
  }
#endif
  NMSM_HD static F inv_target(const Acc& p) { return p.Z; }  // Z != 0 for every point of the complete formulas
  // canonical affine output; identity -> (0, 1), flag 1 (edwards.ts:606)
  NMSM_HD static void to_affine_canonical(const Acc& p, uint32_t* xy, uint32_t* is_inf) {
    to_affine_canonical_with_inv(p, inv(p.Z), xy, is_inf);
  }
  NMSM_HD static void to_affine_canonical_with_inv(const Acc& p, const F& iz, uint32_t* xy, uint32_t* is_inf) {
    F x = p.X * iz, y = p.Y * iz;
    x.to_canonical(xy);
    y.to_canonical(xy + F::LIMBS);
    *is_inf = (x.is_zero() && y == F::one()) ? 1u : 0u;
  }
  // prepared form (y - x, y + x, 2d*x*y) of an accumulator
  NMSM_HD static Affine to_affine_prepared(const Acc& p) {
    F iz = inv(p.Z);
    F x = p.X * iz, y = p.Y * iz;
    return Affine{y - x, y + x, x * y * d2()};
  }
  NMSM_HD static void store_acc(uint32_t* dst, const Acc& p) {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&p);
    for (int k = 0; k < ACC_WORDS; k++) dst[k] = s[k];
  }
};

// Curve policies; ID values are the curve ids of the C ABI (include/nmsm.h)
struct CurveSecp256k1 {
  // lattice GLV with the reference's own endomorphism data (secp256k1.ts:58-64)
  static constexpr bool GLV = true;
  static constexpr int GLV_KIND = 2;
  using Glv = Secp256k1Glv;
  using G = SwXyzz<Fp<FpSecp256k1>>;
  using Fn = Fn_secp256k1;
  static constexpr bool COFACTOR_ONE = true;  // the endomorphism acts as lambda on the WHOLE group E(Fp)
  static constexpr int ID = 0;
};
struct CurveEd25519 {
  static constexpr bool GLV = false;
  static constexpr int GLV_KIND = 0;
  using G = EdExt<Fp<FpEd25519>, Ed25519Consts>;
  using Fn = Fn_ed25519;
  static constexpr bool COFACTOR_ONE = false;  // the endomorphism acts as lambda on the WHOLE group E(Fp)
  static constexpr int ID = 1;
};
struct CurveBn254G1 {
  static constexpr bool GLV = true;
  static constexpr int GLV_KIND = 2;
  using Glv = Bn254G1Glv;
  using G = SwXyzz<Fp<FpBn254>>;
  using Fn = Fn_bn254;
  static constexpr bool COFACTOR_ONE = true;  // the endomorphism acts as lambda on the WHOLE group E(Fp)
  static constexpr int ID = 2;
};
struct CurveBn254G2 {
  static constexpr bool GLV = false;
  static constexpr int GLV_KIND = 0;
  using G = SwXyzz<Fp2<FpBn254>>;
  using Fn = Fn_bn254;
  static constexpr bool COFACTOR_ONE = false;  // the endomorphism acts as lambda on the WHOLE group E(Fp)
  static constexpr int ID = 3;
};
struct CurveBls381G1 {
  // terms are split as k = v1 + v2*lambda and accumulated against P and phi(P) = (beta*x, y): half as many
  // windows, buckets and Horner doublings for the same number of mixed additions (msm_body.cuh glv_split)
  static constexpr bool GLV = true;
  static constexpr int GLV_KIND = 1;  // r = lambda^2 + lambda + 1: one Barrett division, msm_body.cuh glv_split
  using Glv = Bls381G1Glv;
  using G = SwXyzz<Fp<FpBls381>>;
  using Fn = Fn_bls12_381;
  static constexpr bool COFACTOR_ONE = false;  // the endomorphism acts as lambda on the WHOLE group E(Fp)
  static constexpr int ID = 4;
};
// BLS12-381 G1 for ARBITRARY points of E(Fp) (cofactor h = 0x396c8c005555e1568c00aaab0000aaab): phi(P) = lambda * P only
// holds on the prime-order subgroup, so this id runs the plain signed-window schedule (16 windows instead of 8).
// The reference's pippenger is the group law and accepts any Point instance; NMSM_BLS12_381_G1 (GLV) matches it on
// every point that passes the reference's assertValidity / fromBytes (on curve AND torsion-free,
// weierstrass.ts:690-707), this id on every on-curve point.
struct CurveBls381G1Any {
  static constexpr bool GLV = false;
  static constexpr int GLV_KIND = 0;
  using G = SwXyzz<Fp<FpBls381>>;
  using Fn = Fn_bls12_381;
  static constexpr bool COFACTOR_ONE = false;
  static constexpr int ID = 6;
};
// BLS12-381 G2 for points of the prime-order subgroup: terms are split four ways along the untwist-Frobenius-twist
// endomorphism psi (psi(P) = [x]P there, bls12-381.ts:600), k = k0 + k1 z + k2 z^2 + k3 z^3 with 63-bit digits against
// P, -psi(P), psi^2(P), -psi^3(P): 4 windows of 16 bits instead of 16, a quarter of the bucket reduction and of the
// Horner doublings for the same number of mixed additions (msm_body.cuh gls_split).
struct CurveBls381G2 {
  static constexpr bool GLV = true;
  static constexpr int GLV_KIND = 3;  // psi-GLS, four sub-terms per term
  using Glv = Bls381G2Gls;
  using G = SwXyzz<Fp2<FpBls381>>;
  using Fn = Fn_bls12_381;
  static constexpr bool COFACTOR_ONE = false;  // psi acts as [x] only on the prime-order subgroup: multiply() stays generic
  static constexpr int ID = 5;
};
// BLS12-381 G2 for ARBITRARY points of the twist E'(Fp2) (e.g. before cofactor clearing): plain signed windows.
struct CurveBls381G2Any {
  static constexpr bool GLV = false;
  static constexpr int GLV_KIND = 0;
  using G = SwXyzz<Fp2<FpBls381>>;
  using Fn = Fn_bls12_381;
  static constexpr bool COFACTOR_ONE = false;
  static constexpr int ID = 7;
};

}  // namespace nmsm
