// Curve-equation check of canonical affine inputs: the device form of the equation test inside the reference's
// assertValidity (/root/reference/src/abstract/weierstrass.ts:617-624 `isValidXY` used at :766; edwards.ts:461-480).
// The reference's pippenger / constructor do NOT run it ("Does NOT validate", weierstrass.ts:695,711); callers that
// take points from untrusted bigints call assertValidity, and the host mirror's Point.assertValidity lands here.
#pragma once
#include "ec.cuh"

namespace nmsm {

template <class F>
NMSM_HD F field_from_small(uint32_t v) {
  uint32_t w[F::LIMBS];
  for (int k = 0; k < F::LIMBS; k++) w[k] = 0;
  w[0] = v;
  return F::from_canonical(w);
}

// curve constant b of y^2 = x^3 + a x + b (secp256k1.ts:48-56, bn254.ts:80-90,207-223, bls12-381.ts:134-148,321-345;
// P-256, P-384: SEC 2 §2.4.2, §2.5.1)
template <class Cv>
NMSM_HD typename Cv::G::Field curve_b() {
  using F = typename Cv::G::Field;
  if constexpr (Cv::ID == 0) return field_from_small<F>(7);
  else if constexpr (Cv::ID == 8) {
    F b;
    for (int k = 0; k < F::LIMBS; k++) b.v[k] = P256Consts::B_MONT(k);
    return b;
  }
  else if constexpr (Cv::ID == 9) {
    F b;
    for (int k = 0; k < F::LIMBS; k++) b.v[k] = P384Consts::B_MONT(k);
    return b;
  }
  else if constexpr (Cv::ID == 2) return field_from_small<F>(3);
  else if constexpr (Cv::ID == 4 || Cv::ID == 6) return field_from_small<F>(4);
  else if constexpr (Cv::ID == 5 || Cv::ID == 7) {  // 4 * (1 + u)
    using B = typename F::Base;
    return F{field_from_small<B>(4), field_from_small<B>(4)};
  } else {  // bn254 G2: 3 / (9 + u)
    static_assert(Cv::ID == 3, "curve_b: unknown curve");
    const uint32_t w[16] = {0x24a138e5u, 0x3267e6dcu, 0x59dbefa3u, 0xb5b4c5e5u, 0x1be06ac3u, 0x81be1899u, 0xceb8aaaeu, 0x2b149d40u,
                            0x85c315d2u, 0xe4a2bd06u, 0xe52d1852u, 0xa74fa084u, 0xeed8fdf4u, 0xcd2cafadu, 0x3af0fed4u, 0x009713b0u};
    return F::from_canonical(w);
  }
}

// x^3 + a x + b, the right-hand side of the short Weierstrass equation (a = 0, or a = -3 as (x^2 - 3) x)
template <class Cv>
NMSM_HD typename Cv::G::Field sw_rhs(const typename Cv::G::Field& x) {
  using F = typename Cv::G::Field;
  if constexpr (Cv::G::CURVE_A == 0) {
    return sqr(x) * x + curve_b<Cv>();
  } else {
    static_assert(Cv::G::CURVE_A == -3, "sw_rhs: a = 0 or a = -3");
    const F three = nmsm::dbl(F::one()) + F::one();
    return (sqr(x) - three) * x + curve_b<Cv>();
  }
}

// 1 = coordinates in range and on the curve (the affine identity encoding — (0,0) Weierstrass, weierstrass.ts:716;
// (0,1) Edwards — counts as on the curve), 0 otherwise.
template <class Cv>
NMSM_HD int point_on_curve(const uint32_t* xy) {
  using G = typename Cv::G;
  using F = typename G::Field;
  if (!G::input_in_range(xy)) return 0;
  const F x = F::from_canonical(xy), y = F::from_canonical(xy + F::LIMBS);
  if constexpr (G::IS_EDWARDS) {  // -x^2 + y^2 = 1 + d x^2 y^2
    F d;
    for (int k = 0; k < F::LIMBS; k++) d.v[k] = Ed25519Consts::D_MONT(k);
    const F x2 = sqr(x), y2 = sqr(y);
    return (y2 - x2) == (F::one() + d * x2 * y2) ? 1 : 0;
  } else {
    if (x.is_zero() && y.is_zero()) return 1;
    return sqr(y) == sw_rhs<Cv>(x) ? 1 : 0;
  }
}

}  // namespace nmsm
