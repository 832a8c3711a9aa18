// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the secp256k1 public-key recovery bodies (recover.cuh) with g++ and the emulated PTX carry flag, in
// the manner of schnorr_emu.cpp: Keccak-256 of 64 bytes, and the serial statements of k_recover_prepare and
// k_recover_check (both input layouts) over a small fixed-point table of G, so `pytest -m "not gpu"` can compare them
// with the oracle.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "recover.cuh"
#include "inv_divsteps.cuh"

using namespace nmsm;

constexpr int TB = 8;  // table digits: 8 bits (the library's table uses 16-bit digits), as schnorr_emu.cpp

// d * 2^(8 j) * G in table_mul_body's layout, built once per process with the library's table bodies
static const uint32_t* g_table8() {
  using Cv = CurveSecp256k1;
  using G = Cv::G;
  constexpr int LV = point_table_levels<Cv, TB>();
  constexpr uint32_t HALF = 1u << (TB - 1);
  static std::vector<uint32_t> tbl;
  if (tbl.empty()) {
    const uint32_t g_xy[16] = {0x16f81798u, 0x59f2815bu, 0x2dce28d9u, 0x029bfcdbu, 0xce870b07u, 0x55a06295u,
                               0xf9dcbbacu, 0x79be667eu, 0xfb10d4b8u, 0x9c47d08fu, 0xa6855419u, 0xfd17b448u,
                               0x0e1108a8u, 0x5da4fbfcu, 0x26a3c465u, 0x483ada77u};
    unsigned int err[2] = {0xffffffffu, 0xffffffffu};
    std::vector<uint32_t> aff((size_t)split_of<Cv>() * G::AFF_WORDS);
    prepare_body<Cv>(0, 1, g_xy, aff.data(), err);
    const size_t level_words = (size_t)HALF * G::AFF_WORDS;
    tbl.assign(level_words * LV, 0);
    for (uint32_t i = 0; i < HALF; i++) table_base_body<Cv, TB>(i, aff.data(), tbl.data());
    for (int j = 1; j < LV; j++)
      for (uint32_t i = 0; i < HALF; i++)
        table_level_body<Cv>(i, tbl.data() + (size_t)(j - 1) * level_words, tbl.data() + (size_t)j * level_words, TB);
  }
  return tbl.data();
}

template <int LAYOUT>
static int emu_recover(const uint8_t* in, const uint8_t* msgs, const uint64_t* msg_off, uint32_t n, int flags,
                       uint8_t* out, uint8_t* out_ok) {
  constexpr int OUT_WORDS = LAYOUT == RECOVER_SIG65 ? 16 : 8;
  std::vector<uint32_t> rpts((size_t)n * 16), u1s((size_t)n * 8), u2s((size_t)n * 8), words((size_t)n * OUT_WORDS);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  recover_prepare_serial<LAYOUT>(n, in, msgs, msg_off, flags, rpts.data(), u1s.data(), u2s.data(), out_ok);
  recover_check_serial<LAYOUT, TB>(n, g_table8(), rpts.data(), u1s.data(), u2s.data(), out_ok, words.data(), err);
  memcpy(out, words.data(), words.size() * 4);  // little-endian host: the device's byte layout
  return err[1] == 0xffffffffu ? 0 : -2;
}

extern "C" {
int emu_keccak256_64(const uint8_t* in, uint8_t* digest) {
  keccak256_64(in, digest);
  return 0;
}
int emu_recover_batch(const uint8_t* sigs65, const uint8_t* msgs, const uint64_t* msg_off, uint32_t n, int flags,
                      uint8_t* out_xy, uint8_t* out_ok) {
  return emu_recover<RECOVER_SIG65>(sigs65, msgs, msg_off, n, flags, out_xy, out_ok);
}
int emu_ecrecover_batch(const uint8_t* inputs128, uint32_t n, uint8_t* out32, uint8_t* out_ok) {
  return emu_recover<RECOVER_ECREC>(inputs128, nullptr, nullptr, n, 0, out32, out_ok);
}
}
