// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the hash-to-G2 bodies (hash_to_curve.cuh) with g++ and the emulated PTX carry flag, in the manner of
// pairing_emu.cpp: the serial statement of k_bls_hash_to_g2, and its steps one at a time (the 512-bit reduction,
// hash_to_field, the SWU map, the isogeny, clear_cofactor) so `pytest -m "not gpu"` can compare them with the oracle
// on chosen inputs.  Points cross the boundary in the G2 packing (48 canonical words; the identity is all zero).
#include <stdint.h>
#include <string.h>

#include "hash_to_curve.cuh"
#include "inv_divsteps.cuh"

using namespace nmsm;

static void acc_to_affine(const H2cG::Acc& q, uint32_t* out_xy) {
  uint32_t inf;
  H2cG::to_affine_canonical(q, out_xy, &inf);
}

extern "C" {
int emu_h2c_hash(const uint8_t* msgs, const uint64_t* msg_off, uint32_t n, const uint8_t* dst, uint32_t dlen,
                 uint32_t* out_xy) {
  h2c_hash_serial(n, msgs, msg_off, dst, dlen, out_xy);
  return 0;
}
// w: 16 little-endian words of a 512-bit integer; out: its residue mod p, canonical
int emu_h2c_reduce512(const uint32_t* w, uint32_t* out) {
  h2c_reduce512(w).to_canonical(out);
  return 0;
}
// out: u0, u1 canonical (48 words)
int emu_h2c_hash_to_field(const uint8_t* msg, uint64_t mlen, const uint8_t* dst, uint32_t dlen, uint32_t* out) {
  H2cF2 u0, u1;
  h2c_hash_to_field(msg, mlen, dst, dlen, u0, u1);
  u0.to_canonical(out);
  u1.to_canonical(out + 24);
  return 0;
}
// the SWU point of E2' for the canonical u (24 words)
int emu_h2c_sswu(const uint32_t* u, uint32_t* out_xy) {
  H2cF2 x, y;
  h2c_sswu(H2cF2::from_canonical(u), x, y);
  x.to_canonical(out_xy);
  y.to_canonical(out_xy + 24);
  return 0;
}
// iso_map of the E2' point xy
int emu_h2c_iso_map(const uint32_t* xy, uint32_t* out_xy) {
  acc_to_affine(h2c_iso_map(H2cF2::from_canonical(xy), H2cF2::from_canonical(xy + 24)), out_xy);
  return 0;
}
// clear_cofactor of the E2 point xy (the identity encoded as all zero)
int emu_h2c_clear_cofactor(const uint32_t* xy, uint32_t* out_xy) {
  H2cG::Acc p = H2cG::identity();
  uint32_t any = 0;
  for (int k = 0; k < 48; k++) any |= xy[k];
  if (any) p = H2cG::from_affine(H2cG::prepare(xy));
  acc_to_affine(h2c_clear_cofactor(p), out_xy);
  return 0;
}
}
