// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// The group law of ec.cuh (serial and lane-parallel) and msm.cuh's warp_batch_inverse on the device.
#include "devemu.cuh"
#include "context.h"  // msm.cuh's peer-fold kernel names its PeerPtrs, as in engine.cuh
#include "msm.cuh"

using namespace nmsm;

namespace {

template <class G>
__device__ typename G::Acc load_canon_acc(const uint32_t* w) {
  using F = typename G::Field;
  typename G::Acc a;
  F* c = reinterpret_cast<F*>(&a);
  for (int k = 0; k < 4; k++) c[k] = F::from_canonical(w + k * F::LIMBS);
  return a;
}

// One case per LANES lanes.  p, q: accumulators as four canonical coordinates (SwXyzz: X, Y, ZZ, ZZZ; EdExt: X, Y, Z,
// T), ACC_WORDS words each; for madd the first IN_WORDS words of q (and for dbl_affine those of p) are a canonical
// affine point.  op (LANES = 1): 0 add, 1 madd, 2 dbl, 3 dbl_affine (SwXyzz only); op (LANES = 4 or 32): 0 par_add,
// 1 par_dbl with FULLWARP = (LANES == 32).  Output: canonical affine x, y (to_affine_canonical) and the identity flag;
// a lane-parallel case whose lanes disagree on the result sets bit 1 of the flag.
template <class G, int LANES>
__global__ void k_group(int op, uint32_t n, const uint32_t* p, const uint32_t* q, uint32_t* xy, uint32_t* inf) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t i = t / LANES;
  if (i >= n) return;  // whole quads / warps leave together
  typename G::Acc a = load_canon_acc<G>(p + (size_t)i * G::ACC_WORDS);
  const typename G::Acc b = load_canon_acc<G>(q + (size_t)i * G::ACC_WORDS);
  if constexpr (LANES == 1) {
    switch (op) {
      case 0: G::add(a, b); break;
      case 1: G::madd(a, G::prepare(q + (size_t)i * G::ACC_WORDS)); break;
      case 2: G::dbl(a); break;
      default:
        if constexpr (!G::IS_EDWARDS) a = G::dbl_affine(G::prepare(p + (size_t)i * G::ACC_WORDS));
        break;
    }
  } else {
    if (op == 0) G::template par_add<LANES == 32>(a, b);
    else G::template par_dbl<LANES == 32>(a);
  }
  uint32_t r[G::IN_WORDS], f;
  G::to_affine_canonical(a, r, &f);
  if constexpr (LANES > 1) {
    const unsigned lane = threadIdx.x & 31u, base = lane & ~(unsigned)(LANES - 1);
    const unsigned mask = LANES == 32 ? 0xffffffffu : (0xFu << base);
    uint32_t diff = 0;
    for (int k = 0; k < G::IN_WORDS; k++) diff |= r[k] ^ __shfl_sync(mask, r[k], base);
    diff |= f ^ __shfl_sync(mask, f, base);
    diff = __any_sync(mask, diff != 0);
    if (lane != base) return;
    if (diff) f |= 2u;
  }
  for (int k = 0; k < G::IN_WORDS; k++) xy[(size_t)i * G::IN_WORDS + k] = r[k];
  inf[i] = f;
}

template <class G, int LANES>
cudaError_t group_n(int op, uint32_t n, const uint32_t* p, const uint32_t* q, uint32_t* xy, uint32_t* inf) {
  if (n == 0) return cudaSuccess;
  devemu::Buf P(p, (size_t)n * G::ACC_WORDS), Q(q, (size_t)n * G::ACC_WORDS), XY(nullptr, (size_t)n * G::IN_WORDS),
      I(nullptr, n);
  cudaError_t e = devemu::first_error(devemu::first_error(P.err, Q.err), devemu::first_error(XY.err, I.err));
  if (e != cudaSuccess) return e;
  k_group<G, LANES><<<devemu::blocks_for((size_t)n * LANES), devemu::THREADS>>>(op, n, P.p, Q.p, XY.p, I.p);
  e = devemu::finish(xy, XY);
  if (e == cudaSuccess) e = cudaMemcpy(inf, I.p, (size_t)n * 4, cudaMemcpyDeviceToHost);
  return e;
}

// op: 0 add, 1 madd, 2 dbl, 3 dbl_affine, 4 par_add per quad, 5 par_dbl per quad, 6 par_add per warp, 7 par_dbl per warp
template <class G>
int group_op(int op, uint32_t n, const uint32_t* p, const uint32_t* q, uint32_t* xy, uint32_t* inf) {
  if (op < 0 || op > 7 || (op == 3 && G::IS_EDWARDS)) return -1;
  if (op < 4) return group_n<G, 1>(op, n, p, q, xy, inf);
  if (op < 6) return group_n<G, 4>(op - 4, n, p, q, xy, inf);
  return group_n<G, 32>(op - 6, n, p, q, xy, inf);
}

// lanes at and past n feed 1, as the kernels do; inputs and outputs canonical, F::LIMBS words per value
template <class F>
__global__ void k_warp_inv(uint32_t n, const uint32_t* z, uint32_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const F x = i < n ? F::from_canonical(z + (size_t)i * F::LIMBS) : F::one();
  const F r = warp_batch_inverse(x);
  if (i < n) r.to_canonical(out + (size_t)i * F::LIMBS);
}

template <class F>
cudaError_t warp_inv_n(uint32_t n, const uint32_t* z, uint32_t* out) {
  if (n == 0) return cudaSuccess;
  devemu::Buf Z(z, (size_t)n * F::LIMBS), O(nullptr, (size_t)n * F::LIMBS);
  cudaError_t e = devemu::first_error(Z.err, O.err);
  if (e != cudaSuccess) return e;
  k_warp_inv<F><<<devemu::blocks_for(n), devemu::THREADS>>>(n, Z.p, O.p);
  return devemu::finish(out, O);
}

}  // namespace

extern "C" {
// curve: 0 secp256k1, 1 ed25519, 2 bn254 G1, 3 bn254 G2, 4 BLS12-381 G1, 5 BLS12-381 G2
int dev_group(int curve, int op, uint32_t n, const uint32_t* p, const uint32_t* q, uint32_t* xy, uint32_t* inf) {
  switch (curve) {
    case 0: return group_op<CurveSecp256k1::G>(op, n, p, q, xy, inf);
    case 1: return group_op<CurveEd25519::G>(op, n, p, q, xy, inf);
    case 2: return group_op<CurveBn254G1::G>(op, n, p, q, xy, inf);
    case 3: return group_op<CurveBn254G2::G>(op, n, p, q, xy, inf);
    case 4: return group_op<CurveBls381G1::G>(op, n, p, q, xy, inf);
    case 5: return group_op<CurveBls381G2::G>(op, n, p, q, xy, inf);
  }
  return -1;
}
// field: 0 secp256k1 Fp (also the Schnorr kernels' SchF), 1 ed25519 Fp, 2 bn254 Fp, 3 bn254 Fp2, 4 BLS12-381 Fp,
// 5 BLS12-381 Fp2, 6 secp256k1 Fn (the ECDSA kernels' EcS)
int dev_warp_inv(int field, uint32_t n, const uint32_t* z, uint32_t* out) {
  switch (field) {
    case 0: return warp_inv_n<Fp<FpSecp256k1>>(n, z, out);
    case 1: return warp_inv_n<Fp<FpEd25519>>(n, z, out);
    case 2: return warp_inv_n<Fp<FpBn254>>(n, z, out);
    case 3: return warp_inv_n<Fp2<FpBn254>>(n, z, out);
    case 4: return warp_inv_n<Fp<FpBls381>>(n, z, out);
    case 5: return warp_inv_n<Fp2<FpBls381>>(n, z, out);
    case 6: return warp_inv_n<Fp<FnSecp256k1Mod>>(n, z, out);
  }
  return -1;
}
}
