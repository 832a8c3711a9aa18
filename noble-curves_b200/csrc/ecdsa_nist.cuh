// The host driver of ECDSA batch verification on the NIST curves (a = -3, no endomorphism): P-256 (inst_p256.cu) and
// P-384 (inst_p384.cu) instantiate it with their own two kernels and table slot.  Widths come from the curve
// (ecdsa_verify.cuh ecdsa_sw / ecdsa_fw): 8 SW-byte signatures, 2 FW-word keys, SW-word scalars.
#pragma once
#include "engine.cuh"
#include "ecdsa_verify.cuh"

namespace nmsm {

using EcdsaPrepareKernel = void (*)(uint32_t, const uint8_t*, const uint8_t*, const uint64_t*, const uint8_t*,
                                    const uint64_t*, int, uint32_t*, uint32_t*, uint32_t*, uint32_t*, uint8_t*);
using EcdsaCheckKernel = void (*)(uint32_t, const uint32_t*, const uint32_t*, const uint32_t*, const uint32_t*,
                                  const uint32_t*, uint8_t*, unsigned int*);

// The fixed-point table of G in *slot: d * 2^(16 j) * G, point_table_levels<Cv>() levels of 2^15 prepared points.
// Built by the first verify after nmsm_init, freed by nmsm_shutdown.  GConsts: the curve's GX / GY words.
template <class Cv, class GConsts>
int ensure_nist_g_table(uint32_t** slot) {
  if (*slot) return NMSM_OK;
  constexpr int FW = ecdsa_fw<Cv>();
  uint32_t g_xy[2 * FW];
  for (int k = 0; k < FW; k++) {
    g_xy[k] = GConsts::GX(k);
    g_xy[FW + k] = GConsts::GY(k);
  }
  int levels = 0;
  return Engine<Cv>::build_point_table((const uint8_t*)g_xy, slot, &levels);
}

// The batch: arguments as nmsm_p256_verify_batch, already checked for flags and null pointers.  Scratch in
// ed_scratch, slot 0's stream and events, the error slot of the check kernel, record_verify_timing.
template <class Cv, class GConsts>
int nist_ecdsa_verify_batch(EcdsaPrepareKernel prepare, EcdsaCheckKernel check, uint32_t** g_table,
                            const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                            const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok) {
  constexpr uint64_t SB = 4 * ecdsa_sw<Cv>(), FB = 4 * ecdsa_fw<Cv>();  // bytes of a scalar / a field element
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  if (int r = check_offsets(pk_off, "pk_off", n)) return r;
  if (int r = check_offsets(msg_off, "msg_off", n)) return r;
  if (int r = ensure_nist_g_table<Cv, GConsts>(g_table)) return r;
  const uint64_t pk_bytes = pk_off[n], msg_bytes = msg_off[n];
  auto al = [](uint64_t x) { return (x + 255) & ~255ull; };
  const uint64_t o_sig = 0, o_pk = o_sig + al(2 * SB * n), o_pko = o_pk + al(pk_bytes + 16),
                 o_msg = o_pko + al(8 * (n + 1)), o_mo = o_msg + al(msg_bytes + 16), o_q = o_mo + al(8 * (n + 1)),
                 o_u1 = o_q + al(2 * FB * n), o_u2 = o_u1 + al(SB * n), o_r = o_u2 + al(SB * n),
                 o_ok = o_r + al(SB * n), o_misc = o_ok + al(n), total = o_misc + 256;
  CK(X.ed_scratch.ensure(total));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  if (int r = h2d_any(base + o_sig, sigs, 2 * SB * n, st)) return r;
  if (pk_bytes)
    if (int r = h2d_any(base + o_pk, pks, pk_bytes, st)) return r;
  if (int r = h2d_any(base + o_pko, pk_off, 8 * (n + 1), st)) return r;
  if (msg_bytes)
    if (int r = h2d_any(base + o_msg, msgs, msg_bytes, st)) return r;
  if (int r = h2d_any(base + o_mo, msg_off, 8 * (n + 1), st)) return r;
  uint32_t *d_q = (uint32_t*)(base + o_q), *d_u1 = (uint32_t*)(base + o_u1), *d_u2 = (uint32_t*)(base + o_u2),
           *d_r = (uint32_t*)(base + o_r);
  uint8_t* d_ok = base + o_ok;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  CK(cudaMemsetAsync(d_err, 0xff, 8, st));
  EV(0);
  prepare<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, base + o_sig, base + o_pk, (const uint64_t*)(base + o_pko),
                                        base + o_msg, (const uint64_t*)(base + o_mo), flags, d_q, d_u1, d_u2, d_r,
                                        d_ok);
  EV(1);
  check<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, *g_table, d_q, d_u1, d_u2, d_r, d_ok, d_err);
  EV(2);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out_ok, d_ok, n, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  record_verify_timing(X, C);
  return NMSM_OK;
}

}  // namespace nmsm
