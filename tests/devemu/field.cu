// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// The eight Montgomery fields, the double-width pieces of the lazy reduction and Fp2 on the device.  Built twice: with
// the product's -DNMSM_MUL_NOINLINE (multiplications through mul_call / sqr_call / fp2_mul_call, what the kernels run)
// and without it (the inlined mont_mul / mul_lazy of `make EXTRA=`); the second build's entry points end in _inl.
// Word layouts and op numbers are those of tests/hostemu/hostemu.cpp emu_field_n / emu_wide_n / emu_fp2_n.
#include "devemu.cuh"
#include "curve_consts.cuh"
#include "field.cuh"
#include "fp2.cuh"
#include "inv_divsteps.cuh"

#if defined(NMSM_MUL_NOINLINE)
#define DEVEMU_SYM(name) name
#else
#define DEVEMU_SYM(name) name##_inl
#endif

using namespace nmsm;

namespace {

// op: 0 a*b, 1 a+b, 2 a-b, 3 inv_xgcd, 4 from_canonical, 5 to_canonical, 6 sqr, 7 -a, 8 DivstepsInv::inverse,
// 9 DivstepsInv::inverse_words (plain integers, 0 if the walk did not finish), 10 inv, 11 canonical_in_range (word 0)
template <class P>
__global__ void k_field(int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  constexpr int N = P::N;
  const uint32_t* ai = a + (size_t)i * N;
  const uint32_t* bi = b + (size_t)i * N;
  Fp<P> x, y, z = Fp<P>::zero();
  for (int k = 0; k < N; k++) {
    x.v[k] = ai[k];
    y.v[k] = bi[k];
  }
  switch (op) {
    case 0: z = x * y; break;
    case 1: z = x + y; break;
    case 2: z = x - y; break;
    case 3: z = inv_xgcd(x); break;
    case 4: z = Fp<P>::from_canonical(ai); break;
    case 5: x.to_canonical(z.v); break;
    case 6: z = sqr(x); break;
    case 7: z = -x; break;
    case 8: z = DivstepsInv<P>::inverse(x); break;
    case 9: if (!DivstepsInv<P>::inverse_words(ai, z.v)) z = Fp<P>::zero(); break;
    case 10: z = inv(x); break;
    default: z.v[0] = Fp<P>::canonical_in_range(ai) ? 1u : 0u; break;
  }
  for (int k = 0; k < N; k++) r[(size_t)i * N + k] = z.v[k];
}

template <class P>
cudaError_t field_n(int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (n == 0) return cudaSuccess;
  const size_t w = (size_t)n * P::N;
  devemu::Buf A(a, w), B(b, w), Rr(nullptr, w);
  cudaError_t e = devemu::first_error(devemu::first_error(A.err, B.err), Rr.err);
  if (e != cudaSuccess) return e;
  k_field<P><<<devemu::blocks_for(n), devemu::THREADS>>>(op, n, A.p, B.p, Rr.p);
  return devemu::finish(r, Rr);
}

// op 0: T = a * b (any N-limb a, b; 2N output words); op 1: r = T / R mod p (2N-word T < p R / 2; N output words)
template <class P>
__global__ void k_wide(int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  constexpr int N = P::N;
  uint32_t T[2 * N], x[N], y[N];
  if (op == 0) {
    for (int k = 0; k < N; k++) {
      x[k] = a[(size_t)i * N + k];
      y[k] = b[(size_t)i * N + k];
    }
    mul_wide<P>(T, x, y);
    for (int k = 0; k < 2 * N; k++) r[(size_t)i * 2 * N + k] = T[k];
  } else {
    for (int k = 0; k < 2 * N; k++) T[k] = a[(size_t)i * 2 * N + k];
    mont_reduce_wide<P>(x, T);
    for (int k = 0; k < N; k++) r[(size_t)i * N + k] = x[k];
  }
}

template <class P>
cudaError_t wide_n(int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (n == 0) return cudaSuccess;
  const size_t wa = (size_t)n * P::N * (op == 0 ? 1 : 2), wr = (size_t)n * P::N * (op == 0 ? 2 : 1);
  devemu::Buf A(a, wa), B(op == 0 ? b : nullptr, op == 0 ? wa : 0), Rr(nullptr, wr);
  cudaError_t e = devemu::first_error(devemu::first_error(A.err, B.err), Rr.err);
  if (e != cudaSuccess) return e;
  k_wide<P><<<devemu::blocks_for(n), devemu::THREADS>>>(op, n, A.p, B.p, Rr.p);
  return devemu::finish(r, Rr);
}

// form: 0 three reduced base multiplications, 1 mul_lazy, 2 operator* (fp2_mul_call in the NMSM_MUL_NOINLINE build),
// 3 sqr, 4 inv.  Montgomery words, c0 limbs then c1 limbs.
template <class P>
__global__ void k_fp2(int form, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  constexpr int N = P::N;
  const uint32_t* ai = a + (size_t)i * 2 * N;
  const uint32_t* bi = b + (size_t)i * 2 * N;
  Fp2<P> x, y, z;
  for (int k = 0; k < N; k++) {
    x.c0.v[k] = ai[k];
    x.c1.v[k] = ai[N + k];
    y.c0.v[k] = bi[k];
    y.c1.v[k] = bi[N + k];
  }
  switch (form) {
    case 0: {
      Fp<P> t1 = x.c0 * y.c0, t2 = x.c1 * y.c1;
      z = Fp2<P>{t1 - t2, (x.c0 + x.c1) * (y.c0 + y.c1) - (t1 + t2)};
      break;
    }
    case 1: z = Fp2<P>::mul_lazy(x, y); break;
    case 2: z = x * y; break;
    case 3: z = sqr(x); break;
    default: z = inv(x); break;
  }
  for (int k = 0; k < N; k++) {
    r[(size_t)i * 2 * N + k] = z.c0.v[k];
    r[(size_t)i * 2 * N + N + k] = z.c1.v[k];
  }
}

template <class P>
cudaError_t fp2_n(int form, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (n == 0) return cudaSuccess;
  const size_t w = (size_t)n * 2 * P::N;
  devemu::Buf A(a, w), B(b, w), Rr(nullptr, w);
  cudaError_t e = devemu::first_error(devemu::first_error(A.err, B.err), Rr.err);
  if (e != cudaSuccess) return e;
  k_fp2<P><<<devemu::blocks_for(n), devemu::THREADS>>>(form, n, A.p, B.p, Rr.p);
  return devemu::finish(r, Rr);
}

}  // namespace

extern "C" {
// field: 0 secp256k1 p, 1 ed25519 p, 2 bn254 p, 3 BLS12-381 p, 4 secp256k1 n, 5 ed25519 l, 6 bn254 r, 7 BLS12-381 r
int DEVEMU_SYM(dev_field)(int field, int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  switch (field) {
    case 0: return field_n<FpSecp256k1>(op, n, a, b, r);
    case 1: return field_n<FpEd25519>(op, n, a, b, r);
    case 2: return field_n<FpBn254>(op, n, a, b, r);
    case 3: return field_n<FpBls381>(op, n, a, b, r);
    case 4: return field_n<FnSecp256k1Mod>(op, n, a, b, r);
    case 5: return field_n<FnEd25519Mod>(op, n, a, b, r);
    case 6: return field_n<FrBn254>(op, n, a, b, r);
    case 7: return field_n<FrBls381>(op, n, a, b, r);
  }
  return -1;
}
// field: 2 bn254 p, 3 BLS12-381 p
int DEVEMU_SYM(dev_wide)(int field, int op, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (field == 2) return wide_n<FpBn254>(op, n, a, b, r);
  if (field == 3) return wide_n<FpBls381>(op, n, a, b, r);
  return -1;
}
int DEVEMU_SYM(dev_fp2)(int field, int form, uint32_t n, const uint32_t* a, const uint32_t* b, uint32_t* r) {
  if (field == 2) return fp2_n<FpBn254>(form, n, a, b, r);
  if (field == 3) return fp2_n<FpBls381>(form, n, a, b, r);
  return -1;
}
}
