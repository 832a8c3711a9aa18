// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the EIP-4844 KZG bodies (kzg.cuh) with g++ and the emulated PTX carry flag, in the manner of
// h2g1_emu.cpp: the challenge, the blob evaluation (kzg_eval_serial), Fr inversion, the prepare body's pairs and the
// serial statement of the whole check, so `pytest -m "not gpu"` can compare them with oracle/kzg_ref.py.  Field
// elements cross the boundary as 32-byte big-endian values, points in the library's packings.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "inv_divsteps.cuh"
#include "kzg.cuh"

using namespace nmsm;

static std::vector<uint32_t> roots_table() {
  std::vector<uint32_t> t(8 * KZG_N);
  for (uint32_t i = 0; i < KZG_N; i++) memcpy(&t[8 * i], kzg_root(i).v, 32);
  return t;
}

extern "C" {
int emu_kzg_challenge(const uint8_t* blobs, const uint8_t* commitments48, uint32_t n, uint8_t* zs32) {
  for (uint32_t i = 0; i < n; i++) kzg_challenge_body(i, blobs, commitments48, zs32);
  return 0;
}
// the domain as k_kzg_roots writes it, converted to canonical little-endian words
int emu_kzg_roots(uint32_t* out) {
  for (uint32_t i = 0; i < KZG_N; i++) kzg_root(i).to_canonical(out + 8 * i);
  return 0;
}
int emu_kzg_eval(const uint8_t* blobs, const uint8_t* zs32, uint32_t n, uint8_t* ys32, uint8_t* item_ok) {
  const std::vector<uint32_t> roots = roots_table();
  for (uint32_t i = 0; i < n; i++) kzg_eval_serial(i, blobs, zs32, roots.data(), ys32, item_ok);
  return 0;
}
// canonical little-endian words in and out
int emu_fr_inv(const uint32_t* a, uint32_t* out) {
  inv(KzgFr::from_canonical(a)).to_canonical(out);
  return 0;
}
// the setup check, then k_kzg_prepare's pairs (g1: n x 48 words, g2: n x 96 words) and pre_ok; -1: setup rejected
int emu_kzg_prepare(const uint8_t* commitments48, const uint8_t* zs32, const uint8_t* ys32, const uint8_t* proofs48,
                    const uint8_t* vhs32, const uint8_t* item_ok, uint32_t n, const uint8_t* setup96, uint32_t* g1,
                    uint32_t* g2, uint8_t* pre_ok) {
  uint32_t sxy[48];
  if (!kzg_setup_body(setup96, sxy)) return -1;
  kzg_prepare_serial(n, commitments48, zs32, ys32, proofs48, vhs32, item_ok, sxy, g1, g2, pre_ok);
  return 0;
}
// the whole proof check: prepare and the serial pairing checks; -1: setup rejected, -3: a pair failed validation
int emu_kzg_verify(const uint8_t* commitments48, const uint8_t* zs32, const uint8_t* ys32, const uint8_t* proofs48,
                   const uint8_t* vhs32, uint32_t n, const uint8_t* setup96, uint8_t* out_ok) {
  std::vector<uint32_t> g1((size_t)n * 48), g2((size_t)n * 96), W((size_t)(64 + 2) * BLS_F12_WORDS);
  std::vector<uint8_t> pre(n);
  if (emu_kzg_prepare(commitments48, zs32, ys32, proofs48, vhs32, nullptr, n, setup96, g1.data(), g2.data(),
                      pre.data()))
    return -1;
  unsigned int perr[2] = {0xffffffffu, 0xffffffffu};
  bls_check_serial(n, nullptr, g1.data(), g2.data(), pre.data(), 64, W.data(), out_ok, perr);
  return perr[0] == 0xffffffffu && perr[1] == 0xffffffffu ? 0 : -3;
}
}
