// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the EIP-4844 prover bodies (kzg.cuh) with g++ and the emulated PTX carry flag, in the manner of
// kzg_emu.cpp: the quotient (kzg_quotient_serial), the G1 compression and the comb lincomb over a small table, so
// `pytest -m "not gpu"` can compare them with oracle/kzg_ref.py.  Field elements cross the boundary as 32-byte
// big-endian values, points as canonical little-endian words or 48-byte compressed encodings.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "inv_divsteps.cuh"
#include "kzg.cuh"

using namespace nmsm;

static constexpr int EMU_BITS = 4;         // a small table: 64 levels x 8 entries per point
static constexpr uint32_t EMU_POINTS = 5;  // points of the small setup

extern "C" {
// k_kzg_quotient for each blob, in place; item_ok in/out (the range vote of the evaluation, cleared for z >= r)
int emu_kzg_quotient(uint8_t* blobs, const uint8_t* zs32, const uint8_t* ys32, uint32_t n, uint8_t* item_ok) {
  std::vector<uint32_t> roots(8 * KZG_N);
  for (uint32_t i = 0; i < KZG_N; i++) memcpy(&roots[8 * i], kzg_root(i).v, 32);
  for (uint32_t i = 0; i < n; i++) kzg_quotient_serial(i, blobs, zs32, ys32, roots.data(), item_ok);
  return 0;
}
// kzg_g1_compress of n canonical affine points (24 words each) with their identity flags
int emu_g1_compress(const uint32_t* xy, const uint8_t* inf, uint32_t n, uint8_t* out48) {
  for (uint32_t i = 0; i < n; i++) kzg_g1_compress(xy + 24 * (size_t)i, inf[i] != 0, out48 + 48 * (size_t)i);
  return 0;
}
// the comb over EMU_POINTS compressed points (table order, each a point of G1 other than the identity) with
// EMU_BITS-bit digits, S lanes: out48[i] = sum_p s_ip P_p for n scalar rows of EMU_POINTS big-endian elements; -1: a
// point is rejected, -2: npts != EMU_POINTS
int emu_kzg_lincomb(const uint8_t* points48, uint32_t npts, const uint8_t* scalars_be, uint32_t n, uint32_t S,
                    uint8_t* out48, uint8_t* item_ok) {
  constexpr uint32_t HALF = 1u << (EMU_BITS - 1);
  if (npts != EMU_POINTS) return -2;
  std::vector<uint32_t> aff((size_t)npts * KzgG::AFF_WORDS);
  for (uint32_t p = 0; p < npts; p++) {
    uint32_t xy[24];
    if (kzg_decode_g1(points48 + 48 * (size_t)p, xy) != 1) return -1;
    const KzgG::Affine a = KzgG::prepare(xy);
    memcpy(&aff[(size_t)p * KzgG::AFF_WORDS], &a, sizeof(a));
  }
  const size_t level = (size_t)npts * HALF * KzgG::AFF_WORDS;
  std::vector<uint32_t> tbl(kzg_table_bytes<EMU_BITS>(npts) / 4);
  for (uint32_t t = 0; t < npts * HALF; t++) kzg_table_base_body<EMU_BITS>(t, aff.data(), tbl.data());
  for (int j = 1; j < point_table_levels<KzgCv, EMU_BITS>(); j++)
    for (uint32_t t = 0; t < npts * HALF; t++)
      table_level_body<KzgCv>(t, tbl.data() + (j - 1) * level, tbl.data() + j * level, EMU_BITS);
  for (uint32_t i = 0; i < n; i++) {
    item_ok[i] = 1;
    kzg_lincomb_serial<EMU_BITS, EMU_POINTS>(i, S, scalars_be, tbl.data(), out48, item_ok);
  }
  return 0;
}
}
