// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// tests/devemu runs the device arithmetic (field.cuh, fp2.cuh, fp12.cuh, the pairings, ec.cuh, msm.cuh's
// warp_batch_inverse) on the GPU, one case per thread (per quad or per warp where the operation is lane-parallel), so
// tests/test_gpu_arith.py can compare it bit for bit with Python integers, the oracles and tests/hostemu.  The sources
// include the product headers unchanged and are compiled with the product's flags.
//
// Every host wrapper is `extern "C"`, takes a batch of n cases as plain 32-bit words, copies them in, launches one
// kernel, synchronises, copies the result out and returns the cudaError_t (0 = success).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace devemu {

// a device copy of `words` 32-bit words (uninitialised if `src` is null); freed on scope exit
struct Buf {
  uint32_t* p = nullptr;
  cudaError_t err = cudaSuccess;
  size_t words = 0;
  Buf(const uint32_t* src, size_t w) : words(w) {
    err = cudaMalloc(&p, (w ? w : 1) * 4);
    if (err == cudaSuccess && src && w) err = cudaMemcpy(p, src, w * 4, cudaMemcpyHostToDevice);
  }
  ~Buf() {
    if (p) cudaFree(p);
  }
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
};

inline cudaError_t first_error(cudaError_t a, cudaError_t b) { return a != cudaSuccess ? a : b; }

// after a launch: launch error, then execution error, then the copy of `out` back to the host
inline cudaError_t finish(uint32_t* host_out, const Buf& out) {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess && out.words) e = cudaMemcpy(host_out, out.p, out.words * 4, cudaMemcpyDeviceToHost);
  return e;
}

constexpr int THREADS = 128;  // a multiple of 32: whole warps, whole quads
inline unsigned blocks_for(size_t threads) { return (unsigned)((threads + THREADS - 1) / THREADS); }

}  // namespace devemu
