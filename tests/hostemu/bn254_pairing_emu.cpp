// TEST INFRASTRUCTURE ONLY — never linked into libnmsm.so.
//
// Host build of the bn254 pairing bodies (fp12.cuh, pairing_bn254.cuh, pairing_check.cuh) with g++ and the emulated
// PTX carry flag, in the manner of pairing_emu.cpp: single Fp12 operations, the full pairing value, and the serial
// statement of the pairing-check kernels, so `pytest -m "not gpu"` can compare them with oracle/bn254_pairing_ref.py.
// Fp12 values cross this interface as 96 canonical little-endian words in the device's memory order.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "pairing_bn254.cuh"

using namespace nmsm;

static BnF12 from_canon(const uint32_t* w) {
  BnF12 r;
  BnF* f = reinterpret_cast<BnF*>(&r);
  for (int k = 0; k < 12; k++) f[k] = BnF::from_canonical(w + 8 * k);
  return r;
}

static void to_canon(const BnF12& a, uint32_t* w) {
  const BnF* f = reinterpret_cast<const BnF*>(&a);
  for (int k = 0; k < 12; k++) f[k].to_canonical(w + 8 * k);
}

extern "C" {
// op: 0 a*b, 1 a^2, 2 cyclotomic a^2, 3 a^-1, 4..6 a^(p^1..3), 7 conj(a), 8 a^u (cyclotomic), 9 final exponentiation,
// 10 a * (l0 + l3 w + l4 v w) with (l0, l3, l4) the first three Fp2 coefficients of b
int emu_fp12(int op, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  const BnF12 x = from_canon(a), y = from_canon(b);
  BnF12 r;
  switch (op) {
    case 0: r = fp12_mul(x, y); break;
    case 1: r = fp12_sqr(x); break;
    case 2: r = fp12_cyclotomic_sqr(x); break;
    case 3: r = fp12_inv(x); break;
    case 4: r = fp12_frobenius<1>(x); break;
    case 5: r = fp12_frobenius<2>(x); break;
    case 6: r = fp12_frobenius<3>(x); break;
    case 7: r = fp12_conj(x); break;
    case 8: r = fp12_cyclotomic_exp_x(x); break;
    case 9: r = bn_final_exp(x); break;
    case 10: r = fp12_mul_by_034(x, y.c0.c0, y.c0.c1, y.c0.c2); break;
    default: return -1;
  }
  to_canon(r, out);
  return 0;
}

// prod e(P_i, Q_i)^M over n pairs (identity pairs contribute 1), canonical
int emu_pairing(const uint32_t* g1, const uint32_t* g2, uint32_t n, uint32_t* out) {
  BnF12 f = BnF12::one();
  for (uint32_t i = 0; i < n; i++)
    if (!words_zero(g1 + 16 * i, 16) && !words_zero(g2 + 32 * i, 32))
      f = fp12_mul(f, bn_miller_loop(g1 + 16 * i, g2 + 32 * i));
  to_canon(bn_final_exp(f), out);
  return 0;
}

// the pairing-check kernels' work with a workspace of `chunk` pairs; err2: smallest bad G1 / G2 pair index
int emu_pairing_check(const uint32_t* g1, const uint32_t* g2, const uint64_t* pair_off, uint64_t n_checks,
                      uint64_t chunk, uint8_t* out_ok, uint32_t* err2) {
  std::vector<uint32_t> W((size_t)(chunk + 2) * BN_F12_WORDS);
  unsigned int err[2] = {0xffffffffu, 0xffffffffu};
  pairing_check_serial<Bn254Pairing>(n_checks, pair_off, g1, g2, nullptr, chunk, W.data(), out_ok, err);
  err2[0] = err[0];
  err2[1] = err[1];
  return 0;
}
}
