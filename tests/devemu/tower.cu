// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// The two Fp12 towers and the two pairings on the device, one case per thread.  Op numbers and word layouts are those
// of tests/hostemu/pairing_emu.cpp and bn254_pairing_emu.cpp emu_fp12 / emu_pairing: Fp12 values as 12 canonical
// base-field values in the device's memory order, points as canonical affine words, (0, 0) for the identity.
#include "devemu.cuh"
#include "pairing.cuh"
#include "pairing_bn254.cuh"

using namespace nmsm;

namespace {

template <class T>
__device__ Fp12<T> from_canon(const uint32_t* w) {
  constexpr int N = T::C::N;
  Fp12<T> r;
  typename T::F* f = reinterpret_cast<typename T::F*>(&r);
  for (int k = 0; k < 12; k++) f[k] = T::F::from_canonical(w + N * k);
  return r;
}

template <class T>
__device__ void to_canon(const Fp12<T>& a, uint32_t* w) {
  constexpr int N = T::C::N;
  const typename T::F* f = reinterpret_cast<const typename T::F*>(&a);
  for (int k = 0; k < 12; k++) f[k].to_canonical(w + N * k);
}

template <class T>
__device__ Fp12<T> final_exp(const Fp12<T>& f) {
  if constexpr (T::C::N == 12) return bls_final_exp(f);
  else return bn_final_exp(f);
}

// op: 0 a*b, 1 a^2, 2 cyclotomic a^2, 3 a^-1, 4..6 a^(p^1..3), 7 conj(a), 8 a^x (cyclotomic; |x| for BLS12-381, u for
// bn254), 9 final exponentiation, 10 the sparse line product of the tower (BLS12-381: a * (l0 + l1 v + l4 v w) by
// fp12_mul_by_014, bn254: a * (l0 + l3 w + l4 v w) by fp12_mul_by_034) with the first three Fp2 coefficients of b
template <class T>
__global__ void k_fp12(int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  constexpr int W = 12 * T::C::N;
  const Fp12<T> x = from_canon<T>(a + (size_t)i * W), y = from_canon<T>(b + (size_t)i * W);
  Fp12<T> r;
  switch (op) {
    case 0: r = fp12_mul(x, y); break;
    case 1: r = fp12_sqr(x); break;
    case 2: r = fp12_cyclotomic_sqr(x); break;
    case 3: r = fp12_inv(x); break;
    case 4: r = fp12_frobenius<1>(x); break;
    case 5: r = fp12_frobenius<2>(x); break;
    case 6: r = fp12_frobenius<3>(x); break;
    case 7: r = fp12_conj(x); break;
    case 8: r = fp12_cyclotomic_exp_x(x); break;
    case 9: r = final_exp<T>(x); break;
    default:
      if constexpr (T::C::N == 12) r = fp12_mul_by_014(x, y.c0.c0, y.c0.c1, y.c0.c2);
      else r = fp12_mul_by_034(x, y.c0.c0, y.c0.c1, y.c0.c2);
      break;
  }
  to_canon<T>(r, out + (size_t)i * W);
}

// e(P_i, Q_i) of one pair per thread: Miller loop, then final exponentiation; 1 if either point is the identity
template <class T>
__global__ void k_pairing(uint32_t n, const uint32_t* g1, const uint32_t* g2, uint32_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  constexpr int N = T::C::N;
  const uint32_t* p = g1 + (size_t)i * 2 * N;
  const uint32_t* q = g2 + (size_t)i * 4 * N;
  Fp12<T> f = Fp12<T>::one();
  if (!words_zero(p, 2 * N) && !words_zero(q, 4 * N)) {
    if constexpr (N == 12) f = bls_miller_loop(p, q);
    else f = bn_miller_loop(p, q);
  }
  to_canon<T>(final_exp<T>(f), out + (size_t)i * 12 * N);
}

template <class T>
cudaError_t fp12_n(int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  if (n == 0) return cudaSuccess;
  const size_t w = (size_t)n * 12 * T::C::N;
  devemu::Buf A(a, w), B(b, w), O(nullptr, w);
  cudaError_t e = devemu::first_error(devemu::first_error(A.err, B.err), O.err);
  if (e != cudaSuccess) return e;
  k_fp12<T><<<devemu::blocks_for(n), devemu::THREADS>>>(op, n, A.p, B.p, O.p);
  return devemu::finish(out, O);
}

template <class T>
cudaError_t pairing_n(uint32_t n, const uint32_t* g1, const uint32_t* g2, uint32_t* out) {
  if (n == 0) return cudaSuccess;
  constexpr int N = T::C::N;
  devemu::Buf P(g1, (size_t)n * 2 * N), Q(g2, (size_t)n * 4 * N), O(nullptr, (size_t)n * 12 * N);
  cudaError_t e = devemu::first_error(devemu::first_error(P.err, Q.err), O.err);
  if (e != cudaSuccess) return e;
  k_pairing<T><<<devemu::blocks_for(n), devemu::THREADS>>>(n, P.p, Q.p, O.p);
  return devemu::finish(out, O);
}

}  // namespace

extern "C" {
// tower: 0 BLS12-381 (Bls381Tower), 1 bn254 (Bn254Tower)
int dev_fp12(int tower, int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  if (tower == 0) return fp12_n<Bls381Tower>(op, n, a, b, out);
  if (tower == 1) return fp12_n<Bn254Tower>(op, n, a, b, out);
  return -1;
}
int dev_pairing(int tower, uint32_t n, const uint32_t* g1, const uint32_t* g2, uint32_t* out) {
  if (tower == 0) return pairing_n<Bls381Tower>(n, g1, g2, out);
  if (tower == 1) return pairing_n<Bn254Tower>(n, g1, g2, out);
  return -1;
}
}
