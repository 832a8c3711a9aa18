// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the BLS12-381 aggregate-verification bodies (bls_aggregate.cuh) with g++ and the emulated PTX carry
// flag, in the manner of pairing_emu.cpp: k_bls_hash_to_g2's serial statement over the groups' messages, then
// bls_agg_serial with a chosen tile size, tile cap and Miller chunk, so `pytest -m "not gpu"` can hit tile and chunk
// boundaries at small sizes and compare the verdicts with oracle/bls_aggregate_ref.py.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "bls_aggregate.cuh"
#include "hash_to_curve.cuh"

using namespace nmsm;

extern "C" {
// the C ABI's arguments (keys as 24 canonical words each); err3: smallest bad key index, then the pair validation's
// smallest bad G1 / G2 pair index (0xffffffff: none)
int emu_bls_aggregate(const uint8_t* sigs96, const uint64_t* group_off, uint64_t n_checks, const uint8_t* msgs,
                      const uint64_t* msg_off, const uint32_t* keys, const uint64_t* key_off, const uint8_t* dst,
                      uint32_t dlen, uint64_t tile, uint64_t cap, uint64_t chunk, uint8_t* out_ok, uint32_t* err3) {
  const uint64_t n_groups = group_off[n_checks];
  std::vector<uint32_t> h(n_groups * 48 + 1), W((size_t)(chunk + 2) * BLS_F12_WORDS);
  h2c_hash_serial((uint32_t)n_groups, msgs, msg_off, dst, dlen, h.data());
  unsigned int err[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu};
  bls_agg_serial(n_checks, sigs96, group_off, keys, key_off, h.data(), tile, cap, chunk, W.data(), out_ok, err);
  for (int k = 0; k < 3; k++) err3[k] = err[k];
  return 0;
}
}
