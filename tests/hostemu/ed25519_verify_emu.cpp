// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the ed25519 per-signature verification bodies (ed25519_verify.cuh) with g++ and the emulated PTX carry
// flag, in the manner of ecdsa_emu.cpp: the serial statements of k_ed_verify_prepare and k_ed_verify_check over a
// small fixed-point table of B, so `pytest -m "not gpu"` can compare them with the oracle.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "ed25519_verify.cuh"
#include "inv_divsteps.cuh"

using namespace nmsm;

// the serial statements over a fixed-point table of B with 8-bit digits (the library's table uses 16-bit digits)
static int emu_ed25519_verify(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs, const uint64_t* msg_off,
                              uint32_t n, int flags, uint8_t* out_ok) {
  using Cv = CurveEd25519;
  using G = Cv::G;
  constexpr int TB = 8;
  constexpr int LV = point_table_levels<Cv, TB>();
  constexpr uint32_t HALF = 1u << (TB - 1);
  static std::vector<uint32_t> tbl;  // built once per process
  if (tbl.empty()) {
    uint32_t b_xy[16];
    for (int k = 0; k < 8; k++) {
      b_xy[k] = Ed25519Consts::GX(k);
      b_xy[8 + k] = Ed25519Consts::GY(k);
    }
    unsigned int err[2] = {0xffffffffu, 0xffffffffu};
    std::vector<uint32_t> aff((size_t)split_of<Cv>() * G::AFF_WORDS);
    prepare_body<Cv>(0, 1, b_xy, aff.data(), err);
    const size_t level_words = (size_t)HALF * G::AFF_WORDS;
    tbl.assign(level_words * LV, 0);
    for (uint32_t i = 0; i < HALF; i++) table_base_body<Cv, TB>(i, aff.data(), tbl.data());
    for (int j = 1; j < LV; j++)
      for (uint32_t i = 0; i < HALF; i++)
        table_level_body<Cv>(i, tbl.data() + (size_t)(j - 1) * level_words, tbl.data() + (size_t)j * level_words, TB);
  }
  std::vector<uint32_t> as((size_t)n * 16), rs((size_t)n * 16), ss((size_t)n * 8), ks((size_t)n * 8);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  ed_verify_prepare_serial(n, sigs, pks, msgs, msg_off, flags, as.data(), rs.data(), ss.data(), ks.data(), out_ok);
  ed_verify_check_serial<TB>(n, tbl.data(), as.data(), rs.data(), ss.data(), ks.data(), out_ok, err);
  return err[1] == 0xffffffffu ? 0 : -2;
}

extern "C" {
int emu_ed25519_verify_each(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs, const uint64_t* msg_off,
                            uint32_t n, int flags, uint8_t* out_ok) {
  return emu_ed25519_verify(sigs, pks, msgs, msg_off, n, flags, out_ok);
}
}
