// Radix-2 NTT over the scalar field Fr of the pairing curves (SURVEY §8 f4: the MSM's companion in SNARK provers).
//
// Replaces FFT(rootsOfUnity(Fr, G), Fr).direct / .inverse, /root/reference/src/abstract/fft.ts:518-575 (loops
// :422-480, root tables :230-312).  The reference walks one butterfly at a time over bigint arrays; here a
// transform of N = 2^n elements is ceil(n / 10) passes over HBM: every block keeps a tile of 2048 elements in shared
// memory and runs up to 10 butterfly stages on it, twiddles gathered from an L2-resident table of the N roots.
// The table is in Montgomery form and the DATA stays canonical: mont_mul(x, w * R) = x * w, so the one multiplication
// of a butterfly needs no conversion of the data on the way in or out (additions and subtractions do not care).
// Field arithmetic is exact, so any correct schedule is bit-identical to the reference's DIT/DIF loops; the
// schedule per boundary layout:
//   natural in,  natural out : DIF passes, bit-reversal folded into the store          (fft.ts:551 `dit: true, brp: true`)
//   natural in,  brp out     : DIF passes                                               (fft.ts:550)
//   brp in,      natural out : DIT passes                                               (fft.ts:549)
//   brp in,      brp out     : permute, DIF passes                                      (fft.ts:544-548)
// Bound: the integer multiply pipe — one 256-bit Montgomery multiplication per butterfly against 64 bytes of tile traffic,
// most of it in shared memory (64 KB per block: two blocks fit in an H100 SM's 228 KB).
#include "context.h"
#include "field.cuh"
#include "inv_divsteps.cuh"
#include "curve_consts.cuh"

namespace nmsm {

static constexpr int NTT_TILE_LOG = 11;               // elements per block tile (2048 x 32 B = 64 KB shared memory)
static constexpr int NTT_MAX_STAGES = NTT_TILE_LOG - 1;  // stages per pass: leaves >= 2 adjacent columns per row
static constexpr int NTT_THREADS = 1 << (NTT_TILE_LOG - 2);  // 2 butterflies per thread per stage, 2 blocks per SM

struct NttPass {
  int log_n;
  int s_lo, s_hi;  // stages m = 2^s for s in [s_lo, s_hi]
  int cl;          // tile columns taken from the index bits below s_lo - 1 (contiguous in memory)
  int ca;          // tile columns taken from the index bits at and above s_hi
  int tile_log;    // cl + (s_hi - s_lo + 1) + ca
  int inverse;     // use roots[(N - k) mod N]
};

// tile-local index e = [a_part | rho | c]  ->  global index (see NttPass)
__device__ __forceinline__ uint32_t ntt_global_index(const NttPass& p, uint32_t tile, uint32_t e) {
  const int r = p.s_hi - p.s_lo + 1, L = p.s_lo - 1;
  const uint32_t c = e & ((1u << p.cl) - 1u);
  const uint32_t rho = (e >> p.cl) & ((1u << r) - 1u);
  const uint32_t ap = e >> (p.cl + r);
  const uint32_t low_hi = tile & ((1u << (L - p.cl)) - 1u);
  const uint32_t a_hi = tile >> (L - p.cl);
  return (a_hi << (p.s_hi + p.ca)) | (ap << p.s_hi) | (rho << L) | (low_hi << p.cl) | c;
}

template <class F>
__device__ __forceinline__ F ntt_load(const uint32_t* p) {
  F r;
  const uint4* s = reinterpret_cast<const uint4*>(p);
  const uint4 a = s[0], b = s[1];
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
template <class F>
__device__ __forceinline__ void ntt_store(uint32_t* p, const F& x) {
  uint4* d = reinterpret_cast<uint4*>(p);
  d[0] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
  d[1] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
}

// One pass: stages s_hi..s_lo (DIF, descending) or s_lo..s_hi (DIT, ascending) on a shared-memory tile.
template <class P, bool DIT>
__global__ void __launch_bounds__(NTT_THREADS, 2)
k_ntt_pass(uint32_t* __restrict__ data, const uint32_t* __restrict__ roots, NttPass p) {
  using F = Fp<P>;
  extern __shared__ uint4 ntt_smem4[];
  uint32_t* tile = reinterpret_cast<uint32_t*>(ntt_smem4);
  const uint32_t E = 1u << p.tile_log, half = E >> 1;
  const uint32_t N = 1u << p.log_n;
  for (uint32_t e = threadIdx.x; e < E; e += blockDim.x)
    ntt_store<F>(tile + (size_t)e * 8, ntt_load<F>(data + (size_t)ntt_global_index(p, blockIdx.x, e) * 8));
  __syncthreads();
  const int r = p.s_hi - p.s_lo + 1;
  for (int t = 0; t < r; t++) {
    const int s = DIT ? p.s_lo + t : p.s_hi - t;
    const int pb = p.cl + (s - p.s_lo);  // bit of the tile-local index that separates the two butterfly inputs
    for (uint32_t q = threadIdx.x; q < half; q += blockDim.x) {
      const uint32_t e0 = ((q >> pb) << (pb + 1)) | (q & ((1u << pb) - 1u)), e1 = e0 | (1u << pb);
      const uint32_t i0 = ntt_global_index(p, blockIdx.x, e0);
      uint32_t k = (i0 & ((1u << (s - 1)) - 1u)) << (p.log_n - s);  // j * stride, fft.ts:456
      if (p.inverse) k = (N - k) & (N - 1u);                        // inverse table = reversed roots, fft.ts:296-303
      const F w = ntt_load<F>(roots + (size_t)k * 8);
      F a = ntt_load<F>(tile + (size_t)e0 * 8), b = ntt_load<F>(tile + (size_t)e1 * 8);
      if (DIT) {  // fft.ts:463-466
        const F tw = b * w;
        b = a - tw;
        a = a + tw;
      } else {    // fft.ts:470-472
        const F d = a - b;
        a = a + b;
        b = d * w;
      }
      ntt_store<F>(tile + (size_t)e0 * 8, a);
      ntt_store<F>(tile + (size_t)e1 * 8, b);
    }
    __syncthreads();
  }
  for (uint32_t e = threadIdx.x; e < E; e += blockDim.x)
    ntt_store<F>(data + (size_t)ntt_global_index(p, blockIdx.x, e) * 8, ntt_load<F>(tile + (size_t)e * 8));
}

// aux layout (words): [0,8) omega  [8,16) 1/N (Montgomery)  [16, 16 + 8*32) omega^(2^k)
template <class P>
__global__ void k_ntt_setup(uint64_t generator, int log_n, uint32_t* __restrict__ aux) {
  using F = Fp<P>;
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint32_t g[8] = {(uint32_t)generator, (uint32_t)(generator >> 32), 0, 0, 0, 0, 0, 0};
  const F G = F::from_canonical(g);
  // omega = G^((r - 1) >> log_n)  (= G^(oddFactor * 2^(powerOfTwo - bits)), fft.ts:243-245)
  uint32_t ex[8];
  for (int i = 0; i < 8; i++) ex[i] = P::P(i);
  ex[0] -= 1u;  // r is odd
  F w = F::one();
  for (int bit = 255; bit >= log_n; bit--) {
    w = sqr(w);
    if ((ex[bit >> 5] >> (bit & 31)) & 1u) w = w * G;
  }
  for (int i = 0; i < 8; i++) aux[i] = w.v[i];
  uint32_t nn[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  nn[log_n >> 5] = 1u << (log_n & 31);
  const F ninv = inv(F::from_canonical(nn));
  for (int i = 0; i < 8; i++) aux[8 + i] = ninv.v[i];
  F pw = w;
  for (int k = 0; k < 32; k++) {
    for (int i = 0; i < 8; i++) aux[16 + 8 * k + i] = pw.v[i];
    pw = sqr(pw);
  }
}

// roots[i] = omega^i, natural order (fft.ts:258-262), from the omega^(2^k) ladder
template <class P>
__global__ void __launch_bounds__(256)
k_ntt_roots(const uint32_t* __restrict__ aux, uint32_t n, uint32_t* __restrict__ roots) {
  using F = Fp<P>;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  F acc = F::one();
  for (int k = 0; (i >> k) != 0; k++)
    if ((i >> k) & 1u) acc = acc * ntt_load<F>(aux + 16 + 8 * k);
  ntt_store<F>(roots + (size_t)i * 8, acc);
}

// copy into the work buffer with the range check (element >= r: first bad index to err); `reverse` folds the
// bit-reversal permutation of a brp-ordered input into the copy (fft.ts:544-548)
template <class P>
__global__ void __launch_bounds__(256)
k_ntt_ingest(const uint32_t* __restrict__ in, uint32_t* __restrict__ work, int log_n, int reverse, unsigned int* err) {
  using F = Fp<P>;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << log_n)) return;
  const F raw = ntt_load<F>(in + (size_t)i * 8);
  if (!F::canonical_in_range(raw.v)) {
    atomicMin(err, i);
    return;
  }
  const uint32_t j = reverse ? (log_n ? (__brev(i) >> (32 - log_n)) : 0u) : i;
  ntt_store<F>(work + (size_t)j * 8, raw);
}

// copy out with the optional 1/N scaling (fft.ts:566-568; 1/N is held in Montgomery form, so the product is
// canonical again) and the optional bit-reversed destination
template <class P>
__global__ void __launch_bounds__(256)
k_ntt_emit(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, int log_n, const uint32_t* __restrict__ aux,
           int scale, int reverse) {
  using F = Fp<P>;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << log_n)) return;
  F x = ntt_load<F>(src + (size_t)i * 8);
  if (scale) x = x * ntt_load<F>(aux + 8);
  const uint32_t j = reverse ? (log_n ? (__brev(i) >> (32 - log_n)) : 0u) : i;
  ntt_store<F>(dst + (size_t)j * 8, x);
}

template <class P>
static int ntt_run(int field_key, int two_adicity, uint64_t default_gen, void* values, bool on_device, int log_n,
                   uint64_t generator, int inverse, int brp_input, int brp_output) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  if (log_n < 0 || log_n > 31 || log_n > two_adicity)
    return fail(NMSM_ERR_ARG, "rootsOfUnity: wrong bits " + std::to_string(log_n) + " powerOfTwo=" + std::to_string(two_adicity));
  if (log_n > 27) return fail(NMSM_ERR_ARG, "nmsm_ntt: transforms above 2^27 elements are not supported");
  if (generator == 0) generator = default_gen;
  const uint32_t n = 1u << log_n;
  const size_t bytes = (size_t)n * 32;
  cudaStream_t st = C.stream;
  CK(X.ntt_aux.ensure((16 + 8 * 32) * 4 + 16));
  // growing the root buffer discards its contents: forget the cached key first, so that a call failing between here and
  // the table's rebuild (an allocation below) cannot leave a stale key naming a garbage table
  if (bytes > X.ntt_roots.cap) X.ntt_key_bits = -1;
  CK(X.ntt_roots.ensure(bytes));
  CK(X.ntt_work.ensure(bytes));
  CK(X.ntt_tmp.ensure(bytes));
  const uint32_t* d_in = (const uint32_t*)values;
  if (!on_device) {
    CK(X.ntt_data.ensure(bytes));
    CK(cudaMemcpyAsync(X.ntt_data.p, values, bytes, cudaMemcpyHostToDevice, st));
    d_in = (const uint32_t*)X.ntt_data.p;
  }
  uint32_t* aux = (uint32_t*)X.ntt_aux.p;
  uint32_t* roots = (uint32_t*)X.ntt_roots.p;
  uint32_t* tmp = (uint32_t*)X.ntt_tmp.p;
  unsigned int* d_err = (unsigned int*)(aux + 16 + 8 * 32);
  if (X.profiling) cudaEventRecord(C.ev[0], st);
  // root table: cached per (field, generator, size)
  if (X.ntt_key_field != field_key || X.ntt_key_gen != generator || X.ntt_key_bits != log_n) {
    k_ntt_setup<P><<<1, 1, 0, st>>>(generator, log_n, aux);
    k_ntt_roots<P><<<(n + 255) / 256, 256, 0, st>>>(aux, n, roots);
    X.ntt_key_field = field_key;
    X.ntt_key_gen = generator;
    X.ntt_key_bits = log_n;
  }
  if (X.profiling) cudaEventRecord(C.ev[1], st);
  CK(cudaMemsetAsync(d_err, 0xff, 4, st));
  uint32_t* cur = (uint32_t*)X.ntt_work.p;
  k_ntt_ingest<P><<<(n + 255) / 256, 256, 0, st>>>(d_in, cur, log_n, (brp_input && brp_output) ? 1 : 0, d_err);
  const bool dit = brp_input && !brp_output;
  // split the log_n stages into ceil(log_n / NTT_MAX_STAGES) passes of (nearly) equal depth
  const int npass = log_n ? (log_n + NTT_MAX_STAGES - 1) / NTT_MAX_STAGES : 0;
  // the 64 KB opt-in is a property of the current device's context, not of the process: set it on every call (a few
  // microseconds) so that a context re-bound to another device by nmsm_shutdown / nmsm_init has it too
  CK(cudaFuncSetAttribute(k_ntt_pass<P, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (1 << NTT_TILE_LOG) * 32));
  CK(cudaFuncSetAttribute(k_ntt_pass<P, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (1 << NTT_TILE_LOG) * 32));
  for (int k = 0; k < npass; k++) {
    // DIF consumes stages from the top, DIT from the bottom; pass k covers stages (lo, hi]
    const int a = (int)((long long)log_n * k / npass), b = (int)((long long)log_n * (k + 1) / npass);
    NttPass p;
    p.log_n = log_n;
    if (dit) { p.s_lo = a + 1; p.s_hi = b; } else { p.s_lo = log_n - b + 1; p.s_hi = log_n - a; }
    const int r = p.s_hi - p.s_lo + 1;
    const int tile_log = log_n < NTT_TILE_LOG ? log_n : NTT_TILE_LOG;
    const int x = tile_log - r, L = p.s_lo - 1;
    p.cl = L < x ? L : x;
    p.ca = x - p.cl;
    p.tile_log = tile_log;
    p.inverse = inverse ? 1 : 0;
    const unsigned int tiles = n >> tile_log;
    const int threads = tile_log >= 2 ? (1 << (tile_log - 2)) : 1;
    const size_t smem = (size_t)(1u << tile_log) * 32;
    if (dit) k_ntt_pass<P, true><<<tiles, threads, smem, st>>>(cur, roots, p);
    else k_ntt_pass<P, false><<<tiles, threads, smem, st>>>(cur, roots, p);
  }
  const int reverse = (!brp_input && !brp_output) ? 1 : 0;  // DIF leaves bit-reversed order
  k_ntt_emit<P><<<(n + 255) / 256, 256, 0, st>>>(cur, tmp, log_n, aux, inverse ? 1 : 0, reverse);
  CK(cudaGetLastError());
  if (X.profiling) cudaEventRecord(C.ev[2], st);
  unsigned int err = 0xffffffffu;
  CK(cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (err == 0xffffffffu) {  // the caller's buffer is only written when every element was a valid field element
    CK(cudaMemcpyAsync(values, tmp, bytes, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  if (X.profiling) {
    memset(C.last_ms, 0, sizeof(C.last_ms));
    cudaEventElapsedTime(&C.last_ms[NMSM_T_PREPARE], C.ev[0], C.ev[1]);   // root table (0 when cached)
    cudaEventElapsedTime(&C.last_ms[NMSM_T_TOTAL], C.ev[1], C.ev[2]);     // transform, device time
    memcpy(X.last_ms, C.last_ms, sizeof(C.last_ms));
  }
  if (err != 0xffffffffu) {
    return fail(NMSM_ERR_SCALAR, "invalid field element at index " + std::to_string(err), err);
  }
  return NMSM_OK;
}

int ntt_impl(int curve, void* values, int on_device, int log_n, uint64_t generator, int inverse, int brp_input,
             int brp_output) {
  switch (curve) {
    case NMSM_BN254_G1:
    case NMSM_BN254_G2:
      return ntt_run<FrBn254>(0, 28, 5, values, on_device != 0, log_n, generator, inverse, brp_input, brp_output);
    case NMSM_BLS12_381_G1:
    case NMSM_BLS12_381_G2:
      return ntt_run<FrBls381>(1, 32, 5, values, on_device != 0, log_n, generator, inverse, brp_input, brp_output);
    default:
      return fail(NMSM_ERR_ARG, "nmsm_ntt: scalar fields of bn254 and BLS12-381 only");
  }
}

}  // namespace nmsm
