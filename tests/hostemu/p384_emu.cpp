// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the P-384 ECDSA verification bodies (ecdsa_verify.cuh on CurveP384) with g++ and the emulated PTX
// carry flag, in the manner of p256_emu.cpp: SHA-384, the 49- and 97-byte SEC1 decoders, the a = -3 group law at 12
// limbs, the windowed scalar multiplication and the fixed-point table walk with 12-word scalars, and the serial
// statements of k_p384_ecdsa_prepare and k_p384_ecdsa_check over a small fixed-point table of G, so
// `pytest -m "not gpu"` can compare them with the oracle.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "ecdsa_verify.cuh"
#include "inv_divsteps.cuh"

using namespace nmsm;
using Cv = CurveP384;
using G = Cv::G;
using F = G::Field;
static constexpr int W = F::LIMBS;  // 12
static constexpr int TB = 8;        // digit bits of the test table (the library's table uses 16-bit digits)

// the fixed-point table of G with 8-bit digits, built once per process
static const std::vector<uint32_t>& g_table() {
  constexpr int LV = point_table_levels<Cv, TB>();
  constexpr uint32_t HALF = 1u << (TB - 1);
  static std::vector<uint32_t> tbl;
  if (tbl.empty()) {
    uint32_t g_xy[2 * W];
    for (int k = 0; k < W; k++) {
      g_xy[k] = P384Consts::GX(k);
      g_xy[W + k] = P384Consts::GY(k);
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
  return tbl;
}

// canonical affine (x, y) -> accumulator with projective factor lam (lam = 0 means 1): (x l^2, y l^3, l^2, l^3)
static G::Acc acc_from(const uint32_t* xy, const uint32_t* lam) {
  const G::Affine a = G::prepare(xy);
  G::Acc p = G::from_affine(a);
  uint32_t any = 0;
  for (int k = 0; k < W; k++) any |= lam[k];
  if (!any || G::is_identity(p)) return p;
  const F l = F::from_canonical(lam), l2 = sqr(l), l3 = l2 * l;
  return G::Acc{p.X * l2, p.Y * l3, l2, l3};
}

extern "C" {
// the serial statements of the two kernels over the 8-bit table; returns -2 if table_mul_body rejected a u1
int emu_p384_verify_batch(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                          const uint64_t* msg_off, uint32_t n, int flags, uint8_t* out_ok) {
  const std::vector<uint32_t>& tbl = g_table();
  std::vector<uint32_t> qs((size_t)n * 2 * W), u1s((size_t)n * W), u2s((size_t)n * W), rs((size_t)n * W);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  ecdsa_prepare_serial<Cv>(n, sigs, pks, pk_off, msgs, msg_off, flags, qs.data(), u1s.data(), u2s.data(), rs.data(),
                           out_ok);
  ecdsa_check_serial<TB, Cv>(n, tbl.data(), qs.data(), u1s.data(), u2s.data(), rs.data(), out_ok, err);
  return err[1] == 0xffffffffu ? 0 : -2;
}
// SHA-384(msg[0..len)) -> out[48]
void emu_sha384(const uint8_t* msg, uint64_t len, uint8_t* out) { sha384(msg, len, out); }
// 49-byte or 97-byte SEC1 key -> status (0 invalid, 1 point written)
int emu_p384_decode(const uint8_t* enc, uint64_t len, uint32_t* out_xy) {
  if (len == 1 + 4 * W) return sec1_decode_compressed<Cv>(enc, out_xy);
  if (len == 1 + 8 * W) return sec1_decode_uncompressed<Cv>(enc, out_xy);
  return 0;
}
// op 0: p + q (add), 1: p + q (madd, q affine), 2: 2p (dbl), 3: 2p (dbl_affine, p affine).  p, q: canonical affine,
// (0, 0) = O; lam_p, lam_q: projective factors of the accumulators.  out: canonical affine, returns 1 for O.
int emu_p384_group_op(int op, const uint32_t* p, const uint32_t* lam_p, const uint32_t* q, const uint32_t* lam_q,
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
// s * P through scalar_mul_acc (4-bit windows, no GLV); s: 12 little-endian words, any 384-bit value
int emu_p384_mul(const uint32_t* p, const uint32_t* s, uint32_t* out_xy) {
  const G::Acc a = scalar_mul_acc<Cv>(G::prepare(p), s);
  uint32_t inf = 0;
  G::to_affine_canonical(a, out_xy, &inf);
  return (int)inf;
}
// s * G through table_mul_body over the 8-bit table; s: 12 words.  Returns 1 for O, 0 for a point, -1 if s >= n.
int emu_p384_table_mul(const uint32_t* s, uint32_t* out_xy) {
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  G::Acc a;
  if (!table_mul_body<Cv, TB>(0, g_table().data(), s, 1, a, err)) return -1;
  uint32_t inf = 0;
  G::to_affine_canonical(a, out_xy, &inf);
  return (int)inf;
}
}
