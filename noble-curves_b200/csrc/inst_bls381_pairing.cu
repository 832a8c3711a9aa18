// BLS12-381 pairing checks and BLS signature verification (SURVEY §8 row f7, pairing.cuh): the kernels and the two
// C-ABI implementations.
//
// Work is split by pairs, not by checks, so that one check's pairs run in parallel:
//   k_bls_verify_prepare  (verify only) one thread per signature: decode, subgroup checks, the two pairs
//   k_bls_miller          one thread per pair: validation and f_i = f_{|x|,Q_i}(P_i) into the workspace
//   k_bls_final           one thread per check: the product of its f_i, the final exponentiation, the verdict
// The Miller values of at most BLS_CHUNK pairs are alive at once (BLS_CHUNK x 576 B = 37.7 MB); a check that spans a
// chunk boundary carries its partial product to the next chunk in one of two alternating carry slots.
#include <algorithm>

#include "engine.cuh"
#include "pairing.cuh"

namespace nmsm {

static constexpr uint64_t BLS_CHUNK = 1ull << 16;  // pairs per Miller-loop chunk
static constexpr int BLS_BLOCK = 64;               // small blocks spread few, long threads over all SMs

__global__ void __launch_bounds__(BLS_BLOCK)
k_bls_miller(uint64_t q0, uint32_t cnt, const uint32_t* __restrict__ g1, const uint32_t* __restrict__ g2,
             uint32_t* __restrict__ W, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) bls_miller_body(q0 + i, g1, g2, W + (size_t)i * BLS_F12_WORDS, err);
}

__global__ void __launch_bounds__(BLS_BLOCK)
k_bls_final(uint64_t j0, uint32_t cnt, const uint64_t* __restrict__ off, uint64_t q0, uint64_t q1,
            const uint32_t* __restrict__ W, const uint32_t* carry_in, uint32_t* carry_out,
            const uint8_t* __restrict__ pre_ok, uint8_t* __restrict__ out_ok) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) bls_final_body(j0 + i, off, q0, q1, W, carry_in, carry_out, pre_ok, out_ok);
}

__global__ void __launch_bounds__(BLS_BLOCK)
k_bls_verify_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                     const uint32_t* __restrict__ msg_pts, uint32_t* __restrict__ g1, uint32_t* __restrict__ g2,
                     uint8_t* __restrict__ pre_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) bls_verify_prepare_body(i, sigs, pks, msg_pts, g1, g2, pre_ok, err);
}

namespace {
// Runs one launch; with profiling on, times it with events 0-1 of slot 0 and adds the time to last_ms[slot] and to
// NMSM_T_TOTAL (synchronising after every launch, which only profiling pays for).
template <class L>
int bls_launch(Context& X, Slot& C, int slot, L launch) {
  if (X.profiling) cudaEventRecord(C.ev[0], C.stream);
  launch();
  CK(cudaGetLastError());
  if (X.profiling) {
    cudaEventRecord(C.ev[1], C.stream);
    CK(cudaEventSynchronize(C.ev[1]));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, C.ev[0], C.ev[1]);
    X.last_ms[slot] += ms;
    X.last_ms[NMSM_T_TOTAL] += ms;
  }
  return NMSM_OK;
}

// Miller loops and final exponentiations of n_checks checks over pairs already on the device (d_g1, d_g2).  off: host
// offsets (nullptr: two pairs per check); d_off: their device copy.  slot0: timing slot of k_bls_miller.
int bls_checks_run(Context& X, Slot& C, uint64_t n_checks, const uint64_t* off, const uint64_t* d_off,
                   const uint32_t* d_g1, const uint32_t* d_g2, const uint8_t* d_pre, uint32_t* W, uint8_t* d_ok,
                   unsigned int* d_err, int slot0) {
  cudaStream_t st = C.stream;
  const uint64_t total = off ? off[n_checks] : 2 * n_checks;
  uint64_t c = 0;
  for (uint64_t q0 = 0; q0 < total; q0 += BLS_CHUNK, c++) {
    const uint64_t q1 = std::min(q0 + BLS_CHUNK, total);
    const uint32_t cnt = (uint32_t)(q1 - q0);
    if (int r = bls_launch(X, C, slot0, [&] {
          k_bls_miller<<<cdiv(cnt, BLS_BLOCK), BLS_BLOCK, 0, st>>>(q0, cnt, d_g1, d_g2, W, d_err);
        }))
      return r;
    // checks with a pair in [q0, q1): off[j + 1] > q0 and off[j] < q1
    uint64_t ja, jb;
    if (off) {
      ja = (uint64_t)(std::upper_bound(off + 1, off + n_checks + 1, q0) - (off + 1));
      jb = (uint64_t)(std::lower_bound(off, off + n_checks, q1) - off);
    } else {
      ja = q0 / 2;
      jb = (q1 + 1) / 2;
    }
    const uint32_t* carry_in = W + (BLS_CHUNK + ((c + 1) & 1)) * BLS_F12_WORDS;
    uint32_t* carry_out = W + (BLS_CHUNK + (c & 1)) * BLS_F12_WORDS;
    const uint32_t m = (uint32_t)(jb - ja);
    if (m)
      if (int r = bls_launch(X, C, slot0 + 1, [&] {
            k_bls_final<<<cdiv(m, BLS_BLOCK), BLS_BLOCK, 0, st>>>(ja, m, d_off, q0, q1, W, carry_in, carry_out, d_pre,
                                                                 d_ok);
          }))
        return r;
  }
  return NMSM_OK;
}

uint64_t al256(uint64_t x) { return (x + 255) & ~255ull; }
}  // namespace

int bls12_381_pairing_check_batch_impl(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                       uint64_t n_checks, uint8_t* out_ok) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  if (n_checks == 0) return NMSM_OK;
  if (n_checks >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n_checks must be < 2^31");
  if (pair_off[0] != 0) return fail(NMSM_ERR_ARG, "pair_off[0] must be 0");
  for (uint64_t j = 0; j < n_checks; j++)
    if (pair_off[j + 1] < pair_off[j])
      return fail(NMSM_ERR_ARG, "pair_off must be non-decreasing (index " + std::to_string(j + 1) + ")",
                  (long long)(j + 1));
  const uint64_t total = pair_off[n_checks];
  if (total >= (1ull << 31)) return fail(NMSM_ERR_ARG, "the number of pairs must be < 2^31");
  if (total && (!g1_xy || !g2_xy)) return fail(NMSM_ERR_ARG, "null pointer");
  if (X.profiling) memset(X.last_ms, 0, sizeof(X.last_ms));
  const uint64_t o_g1 = 0, o_g2 = o_g1 + al256(96 * total), o_off = o_g2 + al256(192 * total),
                 o_w = o_off + al256(8 * (n_checks + 1)), o_ok = o_w + al256((BLS_CHUNK + 2) * BLS_F12_WORDS * 4),
                 o_misc = o_ok + al256(n_checks), bytes = o_misc + 256;
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  if (total) {
    if (int r = h2d_any(base + o_g1, g1_xy, 96 * total, st)) return r;
    if (int r = h2d_any(base + o_g2, g2_xy, 192 * total, st)) return r;
  }
  if (int r = h2d_any(base + o_off, pair_off, 8 * (n_checks + 1), st)) return r;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  uint8_t* d_ok = base + o_ok;
  CK(cudaMemsetAsync(d_err, 0xff, 8, st));
  CK(cudaMemsetAsync(d_ok, 1, n_checks, st));  // empty checks: the empty product is 1
  if (int r = bls_checks_run(X, C, n_checks, pair_off, (const uint64_t*)(base + o_off), (const uint32_t*)(base + o_g1),
                             (const uint32_t*)(base + o_g2), nullptr, (uint32_t*)(base + o_w), d_ok, d_err, 0))
    return r;
  unsigned int err[2];
  CK(cudaMemcpyAsync(err, d_err, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (err[0] != 0xffffffffu)
    return fail(NMSM_ERR_POINT, "G1 point of pair " + std::to_string(err[0]) + " is out of range or not on the curve",
                err[0]);
  if (err[1] != 0xffffffffu)
    return fail(NMSM_ERR_POINT, "G2 point of pair " + std::to_string(err[1]) + " is out of range or not on the curve",
                err[1]);
  CK(cudaMemcpy(out_ok, d_ok, n_checks, cudaMemcpyDeviceToHost));
  return NMSM_OK;
}

int bls12_381_verify_batch_impl(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msg_pts, uint64_t n,
                                uint8_t* out_ok) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");
  if (X.profiling) memset(X.last_ms, 0, sizeof(X.last_ms));
  const uint64_t o_sig = 0, o_pk = o_sig + al256(96 * n), o_h = o_pk + al256(48 * n), o_g1 = o_h + al256(192 * n),
                 o_g2 = o_g1 + al256(192 * n), o_pre = o_g2 + al256(384 * n),
                 o_w = o_pre + al256(n), o_ok = o_w + al256((BLS_CHUNK + 2) * BLS_F12_WORDS * 4),
                 o_misc = o_ok + al256(n), bytes = o_misc + 256;
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  if (int r = h2d_any(base + o_sig, sigs96, 96 * n, st)) return r;
  if (int r = h2d_any(base + o_pk, pks48, 48 * n, st)) return r;
  if (int r = h2d_any(base + o_h, msg_pts, 192 * n, st)) return r;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  uint32_t *d_g1 = (uint32_t*)(base + o_g1), *d_g2 = (uint32_t*)(base + o_g2);
  uint8_t *d_pre = base + o_pre, *d_ok = base + o_ok;
  CK(cudaMemsetAsync(d_err, 0xff, 16, st));
  if (int r = bls_launch(X, C, 0, [&] {
        k_bls_verify_prepare<<<cdiv(n, BLS_BLOCK), BLS_BLOCK, 0, st>>>(
            (uint32_t)n, base + o_sig, base + o_pk, (const uint32_t*)(base + o_h), d_g1, d_g2, d_pre, d_err);
      }))
    return r;
  if (int r = bls_checks_run(X, C, n, nullptr, nullptr, d_g1, d_g2, d_pre, (uint32_t*)(base + o_w), d_ok, d_err + 2, 1))
    return r;
  unsigned int err[4];
  CK(cudaMemcpyAsync(err, d_err, 16, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (err[0] != 0xffffffffu)
    return fail(NMSM_ERR_POINT,
                "message point " + std::to_string(err[0]) + " is out of range or not on the twist", err[0]);
  if (err[2] != 0xffffffffu || err[3] != 0xffffffffu)  // prepare only emits valid or identity pairs
    return fail(NMSM_ERR_CUDA, "internal error: a prepared pair failed validation");
  CK(cudaMemcpy(out_ok, d_ok, n, cudaMemcpyDeviceToHost));
  return NMSM_OK;
}

}  // namespace nmsm
