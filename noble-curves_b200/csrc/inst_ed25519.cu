// Instantiation of the MSM / scalar-multiplication engine for ed25519, plus the batch-verification
// front/back end that feeds it (SURVEY §8 f1) and per-signature verification (ed25519_verify.cuh).
#include "engine.cuh"
#include "ed25519_verify.cuh"

namespace nmsm {
NMSM_DEFINE_ENGINE(engine_ed25519, CurveEd25519)

__global__ void __launch_bounds__(128)
k_ed_terms(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
           const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ msg_off, const uint8_t* __restrict__ z16,
           uint32_t* __restrict__ pts, uint32_t* __restrict__ scalars, uint32_t* __restrict__ zs_mont,
           unsigned int* bad) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ed_terms_body(i, n, sigs, pks, msgs, msg_off, z16, pts, scalars, zs_mont, bad);
}

// one block: c = -(sum zs_i) mod l, appended with the base point as term 2n
__global__ void __launch_bounds__(256)
k_ed_finish(uint32_t n, const uint32_t* __restrict__ zs_mont, uint32_t* __restrict__ pts,
            uint32_t* __restrict__ scalars) {
  __shared__ uint32_t sh[256 * 8];
  EdS acc = EdS::zero();
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    EdS t;
    for (int k = 0; k < 8; k++) t.v[k] = zs_mont[(size_t)i * 8 + k];
    acc = acc + t;
  }
  for (int k = 0; k < 8; k++) sh[threadIdx.x * 8 + k] = acc.v[k];
  __syncthreads();
  for (uint32_t d = blockDim.x / 2; d >= 1; d >>= 1) {
    if (threadIdx.x < d) {
      EdS a, b;
      for (int k = 0; k < 8; k++) {
        a.v[k] = sh[threadIdx.x * 8 + k];
        b.v[k] = sh[(threadIdx.x + d) * 8 + k];
      }
      a = a + b;
      for (int k = 0; k < 8; k++) sh[threadIdx.x * 8 + k] = a.v[k];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    EdS tot;
    for (int k = 0; k < 8; k++) tot.v[k] = sh[k];
    tot = -tot;
    uint32_t c[8];
    tot.to_canonical(c);
    for (int k = 0; k < 8; k++) {
      scalars[(size_t)(2 * n) * 8 + k] = c[k];
      pts[(size_t)(2 * n) * 16 + k] = Ed25519Consts::GX(k);
      pts[(size_t)(2 * n) * 16 + 8 + k] = Ed25519Consts::GY(k);
    }
  }
}

// [8]*acc == O ?  (clearCofactor, edwards.ts:611-618, then is0)
__global__ void __launch_bounds__(32) k_ed_check(const uint32_t* __restrict__ acc_words, uint32_t* flag) {
  using G = CurveEd25519::G;
  G::Acc acc = load_acc<G>(acc_words);
  for (int j = 0; j < 3; j++) G::par_dbl<true>(acc);
  if (threadIdx.x == 0) *flag = G::is_identity(acc) ? 1u : 0u;
}

int ed25519_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs, const uint64_t* msg_off,
                              uint64_t n, const uint8_t* z16, int* out_ok, long long* out_bad_index) {
  using G = CurveEd25519::G;
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  *out_ok = 0;
  *out_bad_index = -1;
  if (n == 0) {
    *out_ok = 1;
    return NMSM_OK;
  }
  if (2 * n + 1 >= (1ull << 31)) return fail(NMSM_ERR_ARG, "batch too large");
  if (int r = check_offsets(msg_off, "msg_off", n)) return r;
  const uint64_t msg_bytes = msg_off[n];
  const uint64_t terms = 2 * n + 1;
  // scratch layout in one buffer
  const uint64_t o_sig = 0, o_pk = o_sig + al256(64 * n), o_msg = o_pk + al256(32 * n),
                 o_off = o_msg + al256(msg_bytes + 16), o_z = o_off + al256(8 * (n + 1)), o_pts = o_z + al256(16 * n),
                 o_sc = o_pts + al256(64 * terms), o_zs = o_sc + al256(32 * terms), o_misc = o_zs + al256(32 * n),
                 total = o_misc + 1024;
  CK(X.ed_scratch.ensure(total));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  CK(cudaMemcpyAsync(base + o_sig, sigs, 64 * n, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(base + o_pk, pks, 32 * n, cudaMemcpyHostToDevice, st));
  if (msg_bytes) CK(cudaMemcpyAsync(base + o_msg, msgs, msg_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(base + o_off, msg_off, 8 * (n + 1), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(base + o_z, z16, 16 * n, cudaMemcpyHostToDevice, st));
  unsigned int* d_bad = (unsigned int*)(base + o_misc);
  uint32_t* d_flag = (uint32_t*)(base + o_misc + 16);
  uint32_t* d_acc = (uint32_t*)(base + o_misc + 256);
  CK(cudaMemsetAsync(d_bad, 0xff, 4, st));
  uint32_t* d_pts = (uint32_t*)(base + o_pts);
  uint32_t* d_sc = (uint32_t*)(base + o_sc);
  uint32_t* d_zs = (uint32_t*)(base + o_zs);
  k_ed_terms<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, base + o_sig, base + o_pk, base + o_msg,
                                           (const uint64_t*)(base + o_off), base + o_z, d_pts, d_sc, d_zs, d_bad);
  k_ed_finish<<<1, 256, 0, st>>>((uint32_t)n, d_zs, d_pts, d_sc);
  CK(cudaGetLastError());
  if (int r = Engine<CurveEd25519>::run_msm(d_pts, d_sc, terms, d_acc, nullptr, nullptr)) return r;
  k_ed_check<<<1, 32, 0, st>>>(d_acc, d_flag);
  CK(cudaGetLastError());
  uint32_t host[8] = {0};
  CK(cudaMemcpyAsync(host, d_bad, 32, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint32_t bad = host[0], flag = host[4];
  if (bad != 0xffffffffu) {
    *out_bad_index = bad;
    *out_ok = 0;
  } else {
    *out_ok = flag ? 1 : 0;
  }
  (void)G::ACC_WORDS;
  return NMSM_OK;
}

// Per-signature verification: decode, s < l, strict small-order test, SHA-512 and k mod l
__global__ void __launch_bounds__(128)
k_ed_verify_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                    const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ msg_off, int flags,
                    uint32_t* __restrict__ as, uint32_t* __restrict__ rs, uint32_t* __restrict__ ss,
                    uint32_t* __restrict__ ks, uint8_t* __restrict__ ok_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ed_verify_prepare_body(i, sigs, pks, msgs, msg_off, flags, as, rs, ss, ks, ok_out);
}

// [8](s B - k A - R) == O
__global__ void __launch_bounds__(128)
k_ed_verify_check(uint32_t n, const uint32_t* __restrict__ b_tbl, const uint32_t* __restrict__ as,
                  const uint32_t* __restrict__ rs, const uint32_t* __restrict__ ss, const uint32_t* __restrict__ ks,
                  uint8_t* __restrict__ out_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ed_verify_check_body(i, b_tbl, as, rs, ss, ks, out_ok, err);
}

// The check kernel walks the fixed-point table of B in Context::ed25519_b_table (16 levels x 2^15 points x 96 B,
// 48 MiB).
int ed25519_verify_each_impl(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs, const uint64_t* msg_off,
                             uint64_t n, int flags, uint8_t* out_ok) {
  Context& X = g_ctx;
  if (int r = check_offsets(msg_off, "msg_off", n)) return r;
  if (int r = ensure_g_table<CurveEd25519, Ed25519Consts>(&X.ed25519_b_table)) return r;
  const uint64_t msg_bytes = msg_off[n];
  const uint64_t o_sig = 0, o_pk = o_sig + al256(64 * n), o_msg = o_pk + al256(32 * n),
                 o_mo = o_msg + al256(msg_bytes + 16), o_a = o_mo + al256(8 * (n + 1)), o_r = o_a + al256(64 * n),
                 o_s = o_r + al256(64 * n), o_k = o_s + al256(32 * n), o_ok = o_k + al256(32 * n),
                 o_misc = o_ok + al256(n), total = o_misc + 256;
  CK(X.ed_scratch.ensure(total));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = X.slot[0].stream;
  if (int r = h2d_any(base + o_sig, sigs, 64 * n, st)) return r;
  if (int r = h2d_any(base + o_pk, pks, 32 * n, st)) return r;
  if (int r = h2d_any(base + o_msg, msgs, msg_bytes, st)) return r;
  if (int r = h2d_any(base + o_mo, msg_off, 8 * (n + 1), st)) return r;
  uint32_t *d_a = (uint32_t*)(base + o_a), *d_r = (uint32_t*)(base + o_r), *d_s = (uint32_t*)(base + o_s),
           *d_k = (uint32_t*)(base + o_k);
  uint8_t* d_ok = base + o_ok;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  return verify_launch(
      d_err,
      [&] {
        k_ed_verify_prepare<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, base + o_sig, base + o_pk, base + o_msg,
                                                          (const uint64_t*)(base + o_mo), flags, d_a, d_r, d_s, d_k,
                                                          d_ok);
      },
      [&] {
        k_ed_verify_check<<<cdiv(n, 128), 128, 0, st>>>((uint32_t)n, X.ed25519_b_table, d_a, d_r, d_s, d_k, d_ok,
                                                        d_err);
      },
      d_ok, out_ok, n);
}

}  // namespace nmsm
