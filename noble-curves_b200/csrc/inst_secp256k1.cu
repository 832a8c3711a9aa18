// Instantiation of the MSM / scalar-multiplication engine for secp256k1, plus ECDSA batch verification
// (SURVEY §8 f5, ecdsa_verify.cuh).
#include "engine.cuh"
#include "ecdsa_verify.cuh"

namespace nmsm {
NMSM_DEFINE_ENGINE(engine_secp256k1, CurveSecp256k1)

// decode + SHA-256 + range checks, then u1 = h/s, u2 = r/s with one inversion per warp.  Every lane of a warp reaches
// warp_batch_inverse: lanes past n and invalid signatures feed 1, so one bad signature cannot touch its neighbours.
__global__ void __launch_bounds__(128)
k_ecdsa_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                const uint64_t* __restrict__ pk_off, const uint8_t* __restrict__ msgs,
                const uint64_t* __restrict__ msg_off, int flags, uint32_t* __restrict__ qs, uint32_t* __restrict__ u1s,
                uint32_t* __restrict__ u2s, uint32_t* __restrict__ rs, uint8_t* __restrict__ ok_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t q[16], r[8], s[8], h[8];
  const bool ok = i < n && ecdsa_prepare_body(i, sigs, pks, pk_off, msgs, msg_off, flags, q, r, s, h);
  const EcS w = warp_batch_inverse(ok ? EcS::from_canonical(s) : EcS::one());
  if (i < n) ecdsa_store(i, ok, q, r, h, w, qs, u1s, u2s, rs, ok_out);
}

// R = u1 G + u2 Q and the x comparison
__global__ void __launch_bounds__(128)
k_ecdsa_check(uint32_t n, const uint32_t* __restrict__ g_tbl, const uint32_t* __restrict__ qs,
              const uint32_t* __restrict__ u1s, const uint32_t* __restrict__ u2s, const uint32_t* __restrict__ rs,
              uint8_t* __restrict__ out_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ecdsa_check_body(i, g_tbl, qs, u1s, u2s, rs, out_ok, err);
}

int secp256k1_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                                const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  // the offsets drive device reads of `pks` / `msgs`: they must start at 0 and never decrease
  for (const uint64_t* off : {pk_off, msg_off}) {
    const char* name = off == pk_off ? "pk_off" : "msg_off";
    if (off[0] != 0) return fail(NMSM_ERR_ARG, std::string(name) + "[0] must be 0");
    for (uint64_t i = 0; i < n; i++)
      if (off[i + 1] < off[i])
        return fail(NMSM_ERR_ARG, std::string(name) + " must be non-decreasing (index " + std::to_string(i + 1) + ")",
                    (long long)(i + 1));
  }
  if (!X.ecdsa_g_table) {  // once per nmsm_init: d * 2^(16 j) * G, the table table_mul_body walks
    static const uint32_t g_xy[16] = {0x16f81798u, 0x59f2815bu, 0x2dce28d9u, 0x029bfcdbu, 0xce870b07u, 0x55a06295u,
                                      0xf9dcbbacu, 0x79be667eu, 0xfb10d4b8u, 0x9c47d08fu, 0xa6855419u, 0xfd17b448u,
                                      0x0e1108a8u, 0x5da4fbfcu, 0x26a3c465u, 0x483ada77u};
    int levels = 0;
    if (int r = Engine<CurveSecp256k1>::build_point_table((const uint8_t*)g_xy, &X.ecdsa_g_table, &levels)) return r;
  }
  const uint64_t pk_bytes = pk_off[n], msg_bytes = msg_off[n];
  auto al = [](uint64_t x) { return (x + 255) & ~255ull; };
  const uint64_t o_sig = 0, o_pk = o_sig + al(64 * n), o_pko = o_pk + al(pk_bytes + 16), o_msg = o_pko + al(8 * (n + 1)),
                 o_mo = o_msg + al(msg_bytes + 16), o_q = o_mo + al(8 * (n + 1)), o_u1 = o_q + al(64 * n),
                 o_u2 = o_u1 + al(32 * n), o_r = o_u2 + al(32 * n), o_ok = o_r + al(32 * n), o_misc = o_ok + al(n),
                 total = o_misc + 256;
  CK(X.ed_scratch.ensure(total));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  if (int r = h2d_any(base + o_sig, sigs, 64 * n, st)) return r;
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
  k_ecdsa_prepare<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, base + o_sig, base + o_pk, (const uint64_t*)(base + o_pko),
                                                base + o_msg, (const uint64_t*)(base + o_mo), flags, d_q, d_u1, d_u2, d_r,
                                                d_ok);
  EV(1);
  k_ecdsa_check<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, X.ecdsa_g_table, d_q, d_u1, d_u2, d_r, d_ok, d_err);
  EV(2);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out_ok, d_ok, n, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (X.profiling) {
    memset(X.last_ms, 0, sizeof(X.last_ms));
    cudaEventElapsedTime(&X.last_ms[0], C.ev[0], C.ev[1]);
    cudaEventElapsedTime(&X.last_ms[1], C.ev[1], C.ev[2]);
    cudaEventElapsedTime(&X.last_ms[NMSM_T_TOTAL], C.ev[0], C.ev[2]);
    (void)cudaGetLastError();
  }
  return NMSM_OK;
}

}  // namespace nmsm
