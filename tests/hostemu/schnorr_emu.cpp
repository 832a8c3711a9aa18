// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the secp256k1 BIP340 Schnorr verification bodies (schnorr_verify.cuh) with g++ and the emulated PTX
// carry flag, in the manner of ecdsa_emu.cpp: the challenge hash, and the serial statements of k_schnorr_prepare and
// k_schnorr_check over a small fixed-point table of G, so `pytest -m "not gpu"` can compare them with the oracle.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "schnorr_verify.cuh"
#include "inv_divsteps.cuh"

using namespace nmsm;

constexpr int TB = 8;  // table digits: 8 bits (the library's table uses 16-bit digits), as ecdsa_emu.cpp

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

extern "C" {
int emu_bip340_challenge(const uint8_t* r32, const uint8_t* pk32, const uint8_t* msg, uint64_t len, uint8_t* digest) {
  bip340_challenge(r32, pk32, msg, len, digest);
  return 0;
}
int emu_schnorr_verify_batch(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs, const uint64_t* msg_off,
                             uint32_t n, uint8_t* out_ok) {
  std::vector<uint32_t> ps((size_t)n * 16), ss((size_t)n * 8), us((size_t)n * 8), rs((size_t)n * 8);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  schnorr_prepare_serial(n, sigs, pks, msgs, msg_off, ps.data(), ss.data(), us.data(), rs.data(), out_ok);
  schnorr_check_serial<TB>(n, g_table8(), ps.data(), ss.data(), us.data(), rs.data(), out_ok, err);
  return err[1] == 0xffffffffu ? 0 : -2;
}
}
