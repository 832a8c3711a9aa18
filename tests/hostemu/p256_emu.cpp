// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the P-256 ECDSA verification bodies (ecdsa_verify.cuh on CurveP256) with g++ and the emulated PTX
// carry flag, in the manner of ecdsa_emu.cpp: the SEC1 decoders, the a = -3 group law (dbl, dbl_affine, madd, add),
// the windowed scalar multiplication, and the serial statements of k_p256_ecdsa_prepare and k_p256_ecdsa_check over a
// small fixed-point table of G, so `pytest -m "not gpu"` can compare them with the oracle.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "ecdsa_verify.cuh"
#include "inv_divsteps.cuh"

using namespace nmsm;
using Cv = CurveP256;
using G = Cv::G;
using F = G::Field;

// the serial statements over a fixed-point table of G with 8-bit digits (the library's table uses 16-bit digits)
static int emu_verify(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                      const uint64_t* msg_off, uint32_t n, int flags, uint8_t* out_ok) {
  constexpr int TB = 8;
  constexpr int LV = point_table_levels<Cv, TB>();
  constexpr uint32_t HALF = 1u << (TB - 1);
  static std::vector<uint32_t> tbl;  // built once per process
  if (tbl.empty()) {
    uint32_t g_xy[16];
    for (int k = 0; k < 8; k++) {
      g_xy[k] = P256Consts::GX(k);
      g_xy[8 + k] = P256Consts::GY(k);
    }
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
  std::vector<uint32_t> qs((size_t)n * 16), u1s((size_t)n * 8), u2s((size_t)n * 8), rs((size_t)n * 8);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  ecdsa_prepare_serial<Cv>(n, sigs, pks, pk_off, msgs, msg_off, flags, qs.data(), u1s.data(), u2s.data(), rs.data(),
                           out_ok);
  ecdsa_check_serial<TB, Cv>(n, tbl.data(), qs.data(), u1s.data(), u2s.data(), rs.data(), out_ok, err);
  return err[1] == 0xffffffffu ? 0 : -2;
}

// canonical affine (x, y) -> accumulator with projective factor lam (lam = 0 means 1): (x l^2, y l^3, l^2, l^3)
static G::Acc acc_from(const uint32_t* xy, const uint32_t* lam) {
  const G::Affine a = G::prepare(xy);
  G::Acc p = G::from_affine(a);
  uint32_t any = 0;
  for (int k = 0; k < 8; k++) any |= lam[k];
  if (!any || G::is_identity(p)) return p;
  const F l = F::from_canonical(lam), l2 = sqr(l), l3 = l2 * l;
  return G::Acc{p.X * l2, p.Y * l3, l2, l3};
}

extern "C" {
int emu_p256_verify_batch(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                          const uint64_t* msg_off, uint32_t n, int flags, uint8_t* out_ok) {
  return emu_verify(sigs, pks, pk_off, msgs, msg_off, n, flags, out_ok);
}
// 33-byte or 65-byte SEC1 key -> status (0 invalid, 1 point written)
int emu_p256_decode(const uint8_t* enc, uint64_t len, uint32_t* out_xy) {
  if (len == 33) return sec1_decode_compressed<Cv>(enc, out_xy);
  if (len == 65) return sec1_decode_uncompressed<Cv>(enc, out_xy);
  return 0;
}
// op 0: p + q (add), 1: p + q (madd, q affine), 2: 2p (dbl), 3: 2p (dbl_affine, p affine).  p, q: canonical affine,
// (0, 0) = O; lam_p, lam_q: projective factors of the accumulators.  out: canonical affine, returns 1 for O.
int emu_p256_group_op(int op, const uint32_t* p, const uint32_t* lam_p, const uint32_t* q, const uint32_t* lam_q,
                      uint32_t* out_xy) {
  G::Acc a = acc_from(p, lam_p);
  if (op == 0) G::add(a, acc_from(q, lam_q));
  else if (op == 1) G::madd(a, G::prepare(q));
  else if (op == 2) G::dbl(a);
  else a = G::dbl_affine(G::prepare(p));
  uint32_t inf = 0;
  G::to_affine_canonical(a, out_xy, &inf);
  return (int)inf;
}
// s * P through scalar_mul_acc (4-bit windows, no GLV); s: 8 little-endian words, any 256-bit value
int emu_p256_mul(const uint32_t* p, const uint32_t* s, uint32_t* out_xy) {
  const G::Acc a = scalar_mul_acc<Cv>(G::prepare(p), s);
  uint32_t inf = 0;
  G::to_affine_canonical(a, out_xy, &inf);
  return (int)inf;
}
}
