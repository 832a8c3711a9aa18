// Host side of the batch pairing checks for any pairing curve (inst_bls381_pairing.cu, inst_bn254_pairing.cu): the
// chunked launch sequence of a curve's Miller and final kernels, and the C-ABI check entry point's argument checks,
// workspace layout and error reporting.  P is a pairing policy of pairing_check.cuh.
//
// Work is split by pairs, not by checks, so that one check's pairs run in parallel:
//   miller kernel  one thread per pair: validation and f_i into the workspace
//   final kernel   one thread per check: the product of its f_i, the final exponentiation, the verdict
// The Miller values of at most PAIRING_CHUNK pairs are alive at once; a check that spans a chunk boundary carries its
// partial product to the next chunk in one of two alternating carry slots.
#pragma once
#include <algorithm>

#include "engine.cuh"
#include "pairing_check.cuh"

namespace nmsm {

static constexpr uint64_t PAIRING_CHUNK = 1ull << 16;  // pairs per Miller-loop chunk
static constexpr int PAIRING_BLOCK = 64;               // small blocks spread few, long threads over all SMs

// the kernels of one curve: pairing_miller_body / pairing_final_body<P> over a chunk
struct PairingKernels {
  void (*miller)(uint64_t q0, uint32_t cnt, const uint32_t* g1, const uint32_t* g2, uint32_t* W, unsigned int* err);
  void (*final)(uint64_t j0, uint32_t cnt, const uint64_t* off, uint64_t q0, uint64_t q1, const uint32_t* W,
                const uint32_t* carry_in, uint32_t* carry_out, const uint8_t* pre_ok, uint8_t* out_ok);
};
// BLS12-381's (inst_bls381_pairing.cu), also run by the KZG proof checks of inst_kzg.cu
extern const PairingKernels BLS_KERNELS;

namespace {
// Runs one launch; with profiling on, times it with events 0-1 of slot 0 and adds the time to last_ms[slot] and to
// NMSM_T_TOTAL (synchronising after every launch, which only profiling pays for).
template <class L>
int pairing_launch(Context& X, Slot& C, int slot, L launch) {
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
// offsets (nullptr: two pairs per check); d_off: their device copy.  slot0: timing slot of the Miller kernel.
template <class P>
int pairing_checks_run(Context& X, Slot& C, const PairingKernels& K, uint64_t n_checks, const uint64_t* off,
                       const uint64_t* d_off, const uint32_t* d_g1, const uint32_t* d_g2, const uint8_t* d_pre,
                       uint32_t* W, uint8_t* d_ok, unsigned int* d_err, int slot0) {
  constexpr int WORDS = P::F12::WORDS;
  cudaStream_t st = C.stream;
  const uint64_t total = off ? off[n_checks] : 2 * n_checks;
  uint64_t c = 0;
  for (uint64_t q0 = 0; q0 < total; q0 += PAIRING_CHUNK, c++) {
    const uint64_t q1 = std::min(q0 + PAIRING_CHUNK, total);
    const uint32_t cnt = (uint32_t)(q1 - q0);
    if (int r = pairing_launch(X, C, slot0, [&] {
          K.miller<<<cdiv(cnt, PAIRING_BLOCK), PAIRING_BLOCK, 0, st>>>(q0, cnt, d_g1, d_g2, W, d_err);
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
    const uint32_t* carry_in = W + (PAIRING_CHUNK + ((c + 1) & 1)) * WORDS;
    uint32_t* carry_out = W + (PAIRING_CHUNK + (c & 1)) * WORDS;
    const uint32_t m = (uint32_t)(jb - ja);
    if (m)
      if (int r = pairing_launch(X, C, slot0 + 1, [&] {
            K.final<<<cdiv(m, PAIRING_BLOCK), PAIRING_BLOCK, 0, st>>>(ja, m, d_off, q0, q1, W, carry_in, carry_out,
                                                                      d_pre, d_ok);
          }))
        return r;
  }
  return NMSM_OK;
}

uint64_t al256(uint64_t x) { return (x + 255) & ~255ull; }

// bytes of the Miller workspace: PAIRING_CHUNK values and the two carry slots
template <class P>
constexpr uint64_t pairing_workspace_bytes() {
  return (PAIRING_CHUNK + 2) * P::F12::WORDS * 4;
}

// the C-ABI pairing check (include/nmsm.h nmsm_*_pairing_check_batch) on host arrays; pair_off and out_ok are non-null
template <class P>
int pairing_check_batch_impl(const PairingKernels& K, const uint8_t* g1_xy, const uint8_t* g2_xy,
                             const uint64_t* pair_off, uint64_t n_checks, uint8_t* out_ok) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  constexpr uint64_t G1B = 4 * P::G1_WORDS, G2B = 4 * P::G2_WORDS;
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
  const uint64_t o_g1 = 0, o_g2 = o_g1 + al256(G1B * total), o_off = o_g2 + al256(G2B * total),
                 o_w = o_off + al256(8 * (n_checks + 1)), o_ok = o_w + al256(pairing_workspace_bytes<P>()),
                 o_misc = o_ok + al256(n_checks), bytes = o_misc + 256;
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  if (total) {
    if (int r = h2d_any(base + o_g1, g1_xy, G1B * total, st)) return r;
    if (int r = h2d_any(base + o_g2, g2_xy, G2B * total, st)) return r;
  }
  if (int r = h2d_any(base + o_off, pair_off, 8 * (n_checks + 1), st)) return r;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  uint8_t* d_ok = base + o_ok;
  CK(cudaMemsetAsync(d_err, 0xff, 8, st));
  CK(cudaMemsetAsync(d_ok, 1, n_checks, st));  // empty checks: the empty product is 1
  if (int r = pairing_checks_run<P>(X, C, K, n_checks, pair_off, (const uint64_t*)(base + o_off),
                                    (const uint32_t*)(base + o_g1), (const uint32_t*)(base + o_g2), nullptr,
                                    (uint32_t*)(base + o_w), d_ok, d_err, 0))
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
}  // namespace

}  // namespace nmsm
