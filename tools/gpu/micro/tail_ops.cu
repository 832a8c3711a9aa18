// Microbenchmark of the latency-bound primitives of the bucket-reduction / Horner tails (one warp, dependent chains).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 [-DNMSM_MUL_NOINLINE] -I noble-curves_b200/csrc
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdint.h>
#include "ec.cuh"
#include "field_lat.cuh"
#include "inv_divsteps.cuh"
using namespace nmsm;
using F = Fp<FpBls381>;
using G = SwXyzz<F>;

__device__ F mk(uint32_t s) {
  F x;
  // thread-dependent data: with warp-uniform operands ptxas moves the whole chain to the uniform datapath (UIMAD),
  // which is not the pipe the kernels use
  s += (threadIdx.x >> 2) * 7919u + blockIdx.x * 104729u;
  for (int k = 0; k < 12; k++) x.v[k] = FpBls381::R2(k) ^ (s * 2654435761u >> (k & 7));
  x.v[11] &= 0x0fffffffu;
  return x;
}
__device__ G::Acc mkp(uint32_t s) {
  // a real curve point is not needed for timing: formulas are branch-free except for the exceptional cases
  return G::Acc{mk(s), mk(s + 1), mk(s + 2), mk(s + 3)};
}

template <int OP>
__global__ void k(uint32_t* out, long long* cyc, int iters, uint32_t seed) {
  F a = mk(seed + (OP >= 100 ? 0 : 0)), b = mk(seed + 7);
  G::Acc p = mkp(seed + 11), q = mkp(seed + 23);
  unsigned long long g0;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(g0));
  long long t0 = clock64();
  for (int i = 0; i < iters; i++) {
    if (OP == 0) a = a * b;
    if (OP == 1) a = sqr(a);
    if (OP == 2) a = a + b;
    if (OP == 3) a = a - b;
    if (OP == 4) G::template par_dbl<true>(p);
    if (OP == 5) G::template par_add<true>(p, q);
    if (OP == 6) G::dbl(p);
    if (OP == 7) G::add(p, q);
    if (OP == 8) G::template par_dbl<false>(p);
    if (OP == 9) G::template par_add<false>(p, q);
    if (OP == 10) { F r; mont_mul<FpBls381>(r.v, a.v, b.v); a = r; }
    if (OP == 11) { F r; mont_mul_c64<FpBls381>(r.v, a.v, b.v); a = r; }
    if (OP == 12) { F r; mont_mul_sos<FpBls381>(r.v, a.v, b.v); a = r; }
    if (OP == 13) { F r; mont_mul_lat4<FpBls381>(r.v, a.v, b.v); a = r; }
    if (OP == 14) { a = inv(a) + b; }
    if (OP == 15) { a = DivstepsInv<FpBls381>::inverse(a) + b; }
  }
  long long t1 = clock64();
  unsigned long long g1;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(g1));
  uint32_t acc = 0;
  for (int k2 = 0; k2 < 12; k2++) acc ^= a.v[k2] ^ p.X.v[k2] ^ p.Y.v[k2] ^ p.ZZ.v[k2] ^ p.ZZZ.v[k2];
  if (threadIdx.x == 0 && blockIdx.x == 0) { cyc[0] = t1 - t0; cyc[1] = (long long)(g1 - g0); }
  if (acc == 0x1234567u) out[threadIdx.x] = acc;
}

template <int OP>
void run(const char* name, int threads, int blocks, int iters) {
  uint32_t* d; long long* c;
  cudaMalloc(&d, 4096 * 4); cudaMalloc(&c, 64);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e9; long long cy = 0, ns = 0;
  for (int r = 0; r < 3; r++) {
    cudaEventRecord(e0);
    k<OP><<<blocks, threads>>>(d, c, iters, 12345u + r);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
    cudaMemcpy(&cy, c, 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(&ns, c + 1, 8, cudaMemcpyDeviceToHost);
  }
  printf("{\"op\": \"%s\", \"threads\": %d, \"blocks\": %d, \"iters\": %d, \"us_per_op\": %.4f, \"cycles_per_op\": %.1f, \"sm_mhz\": %.0f, \"gmodmul_s\": %.2f, \"err\": \"%s\"}\n",
         name, threads, blocks, iters, best * 1e3 / iters, (double)cy / iters, ns ? (double)cy / ns * 1e3 : 0.0,
         (double)blocks * threads * iters / (best * 1e-3) / 1e9, cudaGetErrorString(cudaGetLastError()));
  cudaFree(d); cudaFree(c);
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  // burst vs sustained: the same saturating multiply chain for 0.5 ms .. 60 ms
  for (int it : {1024}) run<0>("mul_sat", 128, sms * 4, it);
  for (int it : {1024}) run<0>("mul_sat8", 128, sms * 8, it);
  for (int it : {256, 4096}) run<1>("sqr_sat", 128, sms * 4, it);
  run<11>("mul_c64_sat", 128, sms * 4, 1024);
  run<12>("mul_sos_sat", 128, sms * 4, 1024);
  run<13>("mul_lat4_sat", 128, sms * 4, 1024);
  const int IT = 512;
  for (int thr : {32}) {
    for (int blocks : {1, sms * 4}) {
      run<0>("mul", thr, blocks, IT);
      run<10>("mul_inline", thr, blocks, IT);
      run<11>("mul_c64", thr, blocks, IT);
      run<12>("mul_sos", thr, blocks, IT);
      run<13>("mul_lat4", thr, blocks, IT);
      run<14>("inv_xgcd", thr, blocks, 32);
      run<15>("inv_divsteps", thr, blocks, 32);
      run<1>("sqr", thr, blocks, IT);
      run<2>("fadd", thr, blocks, IT * 8);
      run<3>("fsub", thr, blocks, IT * 8);
      run<4>("par_dbl_fw", thr, blocks, IT);
      run<5>("par_add_fw", thr, blocks, IT);
      run<6>("dbl_serial", thr, blocks, IT);
      run<7>("add_serial", thr, blocks, IT);
      run<8>("par_dbl_quad", thr, blocks, IT);
      run<9>("par_add_quad", thr, blocks, IT);
    }
  }
  return 0;
}
