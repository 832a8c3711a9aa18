// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the hash-to-G1 bodies (hash_to_curve.cuh) and the short-signature prepare body (pairing.cuh) with g++
// and the emulated PTX carry flag, in the manner of h2c_emu.cpp: the serial statement of k_bls_hash_to_g1, its steps
// one at a time (hash_to_field, the SWU map, the isogeny, clear_cofactor), and the short-signature verification
// kernels' work, so `pytest -m "not gpu"` can compare them with oracle/hash_to_g1_ref.py.  Points cross the boundary in
// the G1 packing (24 canonical words; the identity is all zero).
#include <stdint.h>
#include <string.h>

#include <vector>

#include "hash_to_curve.cuh"
#include "inv_divsteps.cuh"
#include "pairing.cuh"

using namespace nmsm;

static void acc_to_affine(const H2cG1::Acc& q, uint32_t* out_xy) {
  uint32_t inf;
  H2cG1::to_affine_canonical(q, out_xy, &inf);
}

extern "C" {
int emu_h2g1_hash(const uint8_t* msgs, const uint64_t* msg_off, uint32_t n, const uint8_t* dst, uint32_t dlen,
                  uint32_t* out_xy) {
  h2c_hash_serial_g1(n, msgs, msg_off, dst, dlen, out_xy);
  return 0;
}
// out: u0, u1 canonical (24 words)
int emu_h2g1_hash_to_field(const uint8_t* msg, uint64_t mlen, const uint8_t* dst, uint32_t dlen, uint32_t* out) {
  H2cF u[2];
  h2c_expand_to_fp<2>(msg, mlen, dst, dlen, u);
  u[0].to_canonical(out);
  u[1].to_canonical(out + 12);
  return 0;
}
// the SWU point of E1' for the canonical u (12 words)
int emu_h2g1_sswu(const uint32_t* u, uint32_t* out_xy) {
  H2cF x, y;
  h2c_sswu_g1(H2cF::from_canonical(u), x, y);
  x.to_canonical(out_xy);
  y.to_canonical(out_xy + 12);
  return 0;
}
// iso_map of the E1' point xy
int emu_h2g1_iso_map(const uint32_t* xy, uint32_t* out_xy) {
  acc_to_affine(h2c_iso_map_g1(H2cF::from_canonical(xy), H2cF::from_canonical(xy + 12)), out_xy);
  return 0;
}
// clear_cofactor of the E1 point xy (the identity encoded as all zero)
int emu_h2g1_clear_cofactor(const uint32_t* xy, uint32_t* out_xy) {
  H2cG1::Acc p = H2cG1::identity();
  if (!words_zero(xy, 24)) p = H2cG1::from_affine(H2cG1::prepare(xy));
  acc_to_affine(h2c_clear_cofactor_g1(p), out_xy);
  return 0;
}
// the short-signature verification kernels' work; *err: smallest index whose message point is out of range or off
// the curve
int emu_short_verify(const uint8_t* sigs48, const uint8_t* pks96, const uint32_t* msg_pts, uint32_t n, uint64_t chunk,
                     uint8_t* out_ok, uint32_t* err_out) {
  std::vector<uint32_t> g1((size_t)n * 48), g2((size_t)n * 96), W((size_t)(chunk + 2) * BLS_F12_WORDS);
  std::vector<uint8_t> pre(n);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu}, perr[2] = {0xffffffffu, 0xffffffffu};
  for (uint32_t i = 0; i < n; i++)
    bls_short_verify_prepare_body(i, sigs48, pks96, msg_pts, g1.data(), g2.data(), pre.data(), err);
  bls_check_serial(n, nullptr, g1.data(), g2.data(), pre.data(), chunk, W.data(), out_ok, perr);
  *err_out = err[0];
  return perr[0] == 0xffffffffu && perr[1] == 0xffffffffu ? 0 : -3;
}
}
