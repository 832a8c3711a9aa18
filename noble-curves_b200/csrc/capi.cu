// libnmsm.so — C ABI (include/nmsm.h) over the sm_90a kernels in msm.cuh.
// The per-curve engines are instantiated in inst_*.cu (compiled in parallel); this file holds the
// process-wide context, the Montgomery-multiplication microbenchmark and the extern "C" surface.
// There is deliberately no CPU path: every entry point needs a CUDA device.
#include <dlfcn.h>
#include <thread>
#include <nccl.h>  // types only: the entry points are resolved with dlsym (no link-time dependency)

#include "context.h"
#include "curve_consts.cuh"
#include "field.cuh"

namespace nmsm {

Context g_ctx;
std::mutex g_mu;
DistState g_dist;

// ---------------------------------------------------------------------------------------------
// NCCL, resolved at run time
// ---------------------------------------------------------------------------------------------
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  int (*GetVersion)(int*) = nullptr;
};
static NcclApi g_nccl;

static int nccl_load() {
  if (g_nccl.handle) return NMSM_OK;
  void* h = nullptr;
  for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
    h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) return fail(NMSM_ERR_CUDA, std::string("NCCL is not available: ") + (dlerror() ? dlerror() : "dlopen failed"));
#define NCCL_SYM(field, sym)                                                            \
  *(void**)(&g_nccl.field) = dlsym(h, sym);                                             \
  if (!g_nccl.field) return fail(NMSM_ERR_CUDA, std::string("NCCL symbol missing: ") + sym)
  NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
  NCCL_SYM(CommInitRank, "ncclCommInitRank");
  NCCL_SYM(CommDestroy, "ncclCommDestroy");
  NCCL_SYM(Send, "ncclSend");
  NCCL_SYM(Recv, "ncclRecv");
  NCCL_SYM(AllGather, "ncclAllGather");
  NCCL_SYM(GroupStart, "ncclGroupStart");
  NCCL_SYM(GroupEnd, "ncclGroupEnd");
  NCCL_SYM(GetErrorString, "ncclGetErrorString");
  NCCL_SYM(GetVersion, "ncclGetVersion");
#undef NCCL_SYM
  g_nccl.handle = h;
  return NMSM_OK;
}
static int nccl_check(ncclResult_t r, const char* what) {
  if (r == ncclSuccess) return NMSM_OK;
  return fail(NMSM_ERR_CUDA, std::string("NCCL error in ") + what + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"));
}
int nccl_send(const void* buf, size_t bytes, int peer, cudaStream_t st) {
  return nccl_check(g_nccl.Send(buf, bytes, ncclUint8, peer, (ncclComm_t)g_dist.comm, st), "ncclSend");
}
int nccl_recv(void* buf, size_t bytes, int peer, cudaStream_t st) {
  return nccl_check(g_nccl.Recv(buf, bytes, ncclUint8, peer, (ncclComm_t)g_dist.comm, st), "ncclRecv");
}
int nccl_group_start() { return nccl_check(g_nccl.GroupStart(), "ncclGroupStart"); }
int nccl_group_end() { return nccl_check(g_nccl.GroupEnd(), "ncclGroupEnd"); }
int nccl_all_gather(const void* send, void* recv, size_t bytes_per_rank, cudaStream_t st) {
  return nccl_check(g_nccl.AllGather(send, recv, bytes_per_rank, ncclUint8, (ncclComm_t)g_dist.comm, st), "ncclAllGather");
}

// ---------------------------------------------------------------------------------------------
// staged upload of pageable host memory (context.h h2d_any)
// ---------------------------------------------------------------------------------------------
namespace {
constexpr int STAGE_THREADS_MAX = 8;
constexpr int STAGE_SLOTS_PER_THREAD = 2;
constexpr size_t STAGE_CHUNK = 4u << 20;      // bytes per staging buffer
constexpr size_t STAGE_MIN_BYTES = 16u << 20;  // below this the plain copy is as fast (worker start-up ~0.1 ms)
struct StageState {
  bool ready = false;
  int threads = 0;
  uint8_t* buf[STAGE_THREADS_MAX][STAGE_SLOTS_PER_THREAD] = {};
  cudaEvent_t ev[STAGE_THREADS_MAX][STAGE_SLOTS_PER_THREAD] = {};
  cudaStream_t st[STAGE_THREADS_MAX] = {};
  cudaEvent_t done[STAGE_THREADS_MAX] = {};
};
StageState g_stage;

bool stage_init() {
  StageState& S = g_stage;
  if (S.ready) return S.threads > 0;
  S.ready = true;
  int want = 4;  // worker threads (at most half the host's)
  if (const char* e = getenv("NMSM_STAGE_THREADS")) want = atoi(e);  // 0 disables the staged path
  const int hw = (int)std::thread::hardware_concurrency();
  if (hw > 0 && want > hw / 2) want = hw / 2;
  if (want > STAGE_THREADS_MAX) want = STAGE_THREADS_MAX;
  if (want < 1) return false;
  for (int t = 0; t < want; t++) {
    bool ok = cudaStreamCreateWithFlags(&S.st[t], cudaStreamNonBlocking) == cudaSuccess &&
              cudaEventCreateWithFlags(&S.done[t], cudaEventDisableTiming) == cudaSuccess;
    for (int k = 0; ok && k < STAGE_SLOTS_PER_THREAD; k++)
      ok = cudaHostAlloc((void**)&S.buf[t][k], STAGE_CHUNK, cudaHostAllocDefault) == cudaSuccess &&
           cudaEventCreateWithFlags(&S.ev[t][k], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {  // keep what was fully set up
      (void)cudaGetLastError();
      break;
    }
    S.threads = t + 1;
  }
  return S.threads > 0;
}
}  // namespace

void h2d_release() {
  StageState& S = g_stage;
  for (int t = 0; t < STAGE_THREADS_MAX; t++) {
    for (int k = 0; k < STAGE_SLOTS_PER_THREAD; k++) {
      if (S.buf[t][k]) cudaFreeHost(S.buf[t][k]);
      if (S.ev[t][k]) cudaEventDestroy(S.ev[t][k]);
    }
    if (S.st[t]) cudaStreamDestroy(S.st[t]);
    if (S.done[t]) cudaEventDestroy(S.done[t]);
  }
  S = StageState();
}

int h2d_any(void* dst, const void* src, size_t bytes, cudaStream_t stream) {
  if (bytes == 0) return NMSM_OK;
  bool pageable = false;
  if (bytes >= STAGE_MIN_BYTES) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, src) == cudaSuccess) pageable = at.type == cudaMemoryTypeUnregistered;
    else (void)cudaGetLastError();
  }
  if (!pageable || !stage_init()) {
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
    return NMSM_OK;
  }
  StageState& S = g_stage;
  const size_t nchunks = (bytes + STAGE_CHUNK - 1) / STAGE_CHUNK;
  const int T = (size_t)S.threads < nchunks ? S.threads : (int)nchunks;
  const int device = g_ctx.device;
  cudaError_t errs[STAGE_THREADS_MAX];
  auto work = [&](int t) {
    cudaError_t e = cudaSetDevice(device);
    int k = 0;
    for (size_t c = (size_t)t; e == cudaSuccess && c < nchunks; c += (size_t)T, k ^= 1) {
      const size_t off = c * STAGE_CHUNK, len = bytes - off < STAGE_CHUNK ? bytes - off : STAGE_CHUNK;
      e = cudaEventSynchronize(S.ev[t][k]);  // the DMA that last read this staging buffer (no-op the first time)
      if (e != cudaSuccess) break;
      memcpy(S.buf[t][k], (const uint8_t*)src + off, len);
      e = cudaMemcpyAsync((uint8_t*)dst + off, S.buf[t][k], len, cudaMemcpyHostToDevice, S.st[t]);
      if (e == cudaSuccess) e = cudaEventRecord(S.ev[t][k], S.st[t]);
    }
    if (e == cudaSuccess) e = cudaEventRecord(S.done[t], S.st[t]);
    errs[t] = e;
  };
  std::thread th[STAGE_THREADS_MAX];
  for (int t = 1; t < T; t++) th[t] = std::thread(work, t);
  work(0);
  for (int t = 1; t < T; t++) th[t].join();
  for (int t = 0; t < T; t++) CK(errs[t]);
  for (int t = 0; t < T; t++) CK(cudaStreamWaitEvent(stream, S.done[t], 0));
  return NMSM_OK;
}

static const EngineVTable* engine_for(int curve) {
  switch (curve) {
    case NMSM_SECP256K1: return engine_secp256k1();
    case NMSM_ED25519: return engine_ed25519();
    case NMSM_BN254_G1: return engine_bn254g1();
    case NMSM_BN254_G2: return engine_bn254g2();
    case NMSM_BLS12_381_G1: return engine_bls381g1();
    case NMSM_BLS12_381_G2: return engine_bls381g2();
    case NMSM_BLS12_381_G1_ANY: return engine_bls381g1_any();
    case NMSM_BLS12_381_G2_ANY: return engine_bls381g2_any();
    default: return nullptr;
  }
}

// ---------------------------------------------------------------------------------------------
// Montgomery-multiplication throughput microbenchmark (roofline denominator)
// ---------------------------------------------------------------------------------------------
template <class P, int ILP>
__global__ void k_modmul_bench(uint32_t* io, int iters) {
  Fp<P> x[ILP], y;
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
  for (int k = 0; k < P::N; k++) {
    y.v[k] = P::R2(k) ^ (t * 2654435761u >> 7 & 0xffff);
#pragma unroll
    for (int q = 0; q < ILP; q++) x[q].v[k] = P::R1(k) + q + (k == 0 ? t : 0);
  }
  // make operands < p so the reduced-input invariant holds
  y.v[P::N - 1] &= 0x0fffffffu;
#pragma unroll
  for (int q = 0; q < ILP; q++) x[q].v[P::N - 1] &= 0x0fffffffu;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int q = 0; q < ILP; q++) x[q] = x[q] * y;
  }
  uint32_t acc = 0;
#pragma unroll
  for (int q = 0; q < ILP; q++)
#pragma unroll
    for (int k = 0; k < P::N; k++) acc ^= x[q].v[k];
  if (acc == 0x12345678u) io[t] = acc;  // keep the chain alive without measurable traffic
}

template <class P>
static double bench_modmul(int blocks_per_sm, int threads, int iters, int ilp) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  uint32_t* d = nullptr;
  int blocks = blocks_per_sm * X.sm_count;
  if (cudaMalloc(&d, (size_t)blocks * threads * 4) != cudaSuccess) return -1;
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  float best = 1e30f;
  for (int rep = 0; rep < 4; rep++) {
    cudaEventRecord(a, C.stream);
    if (ilp == 1) k_modmul_bench<P, 1><<<blocks, threads, 0, C.stream>>>(d, iters);
    else if (ilp == 2) k_modmul_bench<P, 2><<<blocks, threads, 0, C.stream>>>(d, iters);
    else k_modmul_bench<P, 4><<<blocks, threads, 0, C.stream>>>(d, iters);
    cudaEventRecord(b, C.stream);
    if (cudaEventSynchronize(b) != cudaSuccess) { best = -1; break; }
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    if (rep > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  cudaFree(d);
  if (best <= 0) return -1;
  int eff_ilp = ilp == 1 ? 1 : (ilp == 2 ? 2 : 4);
  return (double)blocks * threads * (double)iters * eff_ilp / (best * 1e-3);
}

// Collective (every rank calls it for the same MSM, because the bucket workspace grows at the same call on every rank: its
// size depends only on the plan of the whole MSM): publish this rank's bucket array through CUDA IPC and map every peer's.
int dist_map_peer_buckets(int slot, void* local_base, cudaStream_t st) {
  DistState& D = g_dist;
  if (D.world == 1 || !D.p2p) return NMSM_OK;
  if (D.mapped_local[slot] == local_base) return NMSM_OK;
  for (int r = 0; r < D.world; r++)
    if (D.mapped[slot][r]) {
      cudaIpcCloseMemHandle(D.mapped[slot][r]);
      D.mapped[slot][r] = nullptr;
    }
  cudaIpcMemHandle_t mine;
  CK(cudaIpcGetMemHandle(&mine, local_base));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t* d_h = nullptr;
  CK(cudaMalloc((void**)&d_h, sizeof(mine) * (D.world + 1)));
  CK(cudaMemcpyAsync(d_h + D.world, &mine, sizeof(mine), cudaMemcpyHostToDevice, st));
  if (int r = nccl_all_gather(d_h + D.world, d_h, sizeof(mine), st)) { cudaFree(d_h); return r; }
  std::vector<cudaIpcMemHandle_t> all(D.world);
  CK(cudaMemcpyAsync(all.data(), d_h, sizeof(mine) * D.world, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  cudaFree(d_h);
  // map every peer; if ANY rank cannot map ANY peer, every rank drops to the copy form together (the owner's fold and the
  // non-owners' sends must agree on the form): a second tiny all-gather carries the verdicts
  uint32_t ok = 1;
  for (int r = 0; r < D.world; r++) {
    if (r == D.rank) continue;
    cudaError_t e = cudaIpcOpenMemHandle(&D.mapped[slot][r], all[r], cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      D.mapped[slot][r] = nullptr;
      ok = 0;
    }
  }
  uint32_t* d_ok = nullptr;
  CK(cudaMalloc((void**)&d_ok, 4 * (D.world + 1)));
  CK(cudaMemcpyAsync(d_ok + D.world, &ok, 4, cudaMemcpyHostToDevice, st));
  if (int r = nccl_all_gather(d_ok + D.world, d_ok, 4, st)) { cudaFree(d_ok); return r; }
  std::vector<uint32_t> oks(D.world);
  CK(cudaMemcpyAsync(oks.data(), d_ok, 4 * D.world, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  cudaFree(d_ok);
  for (uint32_t v : oks) ok &= v;
  if (!ok) {
    for (int r = 0; r < D.world; r++)
      if (D.mapped[slot][r]) {
        cudaIpcCloseMemHandle(D.mapped[slot][r]);
        D.mapped[slot][r] = nullptr;
      }
    D.p2p = false;  // for the rest of the process: ncclSend / ncclRecv copies of the dense windows
    return NMSM_OK;
  }
  D.mapped_local[slot] = local_base;
  return NMSM_OK;
}

}  // namespace nmsm

using namespace nmsm;

// ---------------------------------------------------------------------------------------------
// extern "C"
// ---------------------------------------------------------------------------------------------
#define ENGINE(curve)                                      \
  const EngineVTable* E = engine_for(curve);               \
  if (!E) return fail(NMSM_ERR_ARG, "unknown curve id")
// The synchronous entry points run on slot 0's stream, workspace and pinned staging: refuse while an MSM submitted on
// slot 0 has not been collected (its result would be overwritten) instead of silently sharing them.
#define SLOT0_FREE()                                                                                         \
  if (g_ctx.slot[0].pend.active)                                                                             \
  return fail(NMSM_ERR_ARG, "slot 0 holds an MSM that has not been collected: collect it before a synchronous call")

extern "C" {

int nmsm_init(int device) {
  std::lock_guard<std::mutex> lk(g_mu);
  Context& C = g_ctx;
  if (C.ready && C.device == device) return NMSM_OK;
  if (C.ready) return fail(NMSM_ERR_ARG, "nmsm_init: context already bound to another device");
  // The MSM pipeline overlaps kernels on several streams per slot; with the default of 8 hardware work queues unrelated
  // streams share a queue and serialise.  Only effective if this process has not created its CUDA context yet (the
  // Python mirror and bench.py also set it before importing torch); never overrides the user's choice.
  setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail(NMSM_ERR_CUDA, std::string("no CUDA device available (there is no CPU fallback): ") +
                                   cudaGetErrorString(e));
  if (device < 0 || device >= count) return fail(NMSM_ERR_ARG, "nmsm_init: bad device ordinal");
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  C.sm_count = prop.multiProcessorCount;
  int prio_lo = 0, prio_hi = 0;  // numerically lower = more urgent
  CK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  for (Slot& S : C.slot) {
    CK(cudaStreamCreateWithFlags(&S.stream, cudaStreamNonBlocking));
    for (auto& st : S.acc_stream) CK(cudaStreamCreateWithPriority(&st, cudaStreamNonBlocking, prio_lo));
    for (auto& st : S.tail_stream) CK(cudaStreamCreateWithPriority(&st, cudaStreamNonBlocking, prio_hi));
    CK(cudaStreamCreateWithPriority(&S.horner_stream, cudaStreamNonBlocking, prio_hi));
    CK(cudaStreamCreateWithFlags(&S.prep_stream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&S.ev_start, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&S.ev_prep, cudaEventDisableTiming));
    CK(cudaMallocHost((void**)&S.h_result, 1024));
    for (auto& ev : S.ev) CK(cudaEventCreate(&ev));
    CK(cudaEventCreateWithFlags(&S.done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&S.ev_fork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&S.ev_horner, cudaEventDisableTiming));
    for (auto& ev : S.ev_acc) CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    for (auto& ev : S.ev_tail) CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    CK(cudaEventCreate(&S.ev_t0));
    CK(cudaEventCreate(&S.ev_t1));
    if (getenv("NMSM_TRACE")) {
      C.trace = true;
      CK(cudaEventCreate(&S.tr_fork));
      for (auto& ev : S.tr_acc) CK(cudaEventCreate(&ev));
      for (auto& ev : S.tr_tail) CK(cudaEventCreate(&ev));
      for (auto& ev : S.tr_h) CK(cudaEventCreate(&ev));
    }
    CK(cudaStreamCreateWithPriority(&S.comm_stream, cudaStreamNonBlocking, prio_hi));
    CK(cudaEventCreateWithFlags(&S.ev_gather, cudaEventDisableTiming));
    for (auto& ev : S.ev_fin) CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    for (auto& ev : S.ev_xchg) CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    CK(cudaMallocHost((void**)&S.h_gather, 64 * 1024));
  }
  C.device = device;
  C.ready = true;
  return NMSM_OK;
}

void nmsm_shutdown(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  Context& C = g_ctx;
  if (!C.ready) return;
  if (g_dist.ready) {
    for (Slot& S : C.slot) cudaStreamSynchronize(S.comm_stream);
    for (int sl = 0; sl < NUM_SLOTS; sl++)
      for (int r = 0; r < MAX_PEERS; r++)
        if (g_dist.mapped[sl][r]) cudaIpcCloseMemHandle(g_dist.mapped[sl][r]);
    g_nccl.CommDestroy((ncclComm_t)g_dist.comm);
    g_dist = DistState();
  }
  for (Slot& S : C.slot) {
    cudaStreamSynchronize(S.stream);
    cudaStreamSynchronize(S.comm_stream);
    for (auto st : S.acc_stream) cudaStreamSynchronize(st);
    for (auto st : S.tail_stream) cudaStreamSynchronize(st);
    cudaStreamSynchronize(S.horner_stream);
    cudaStreamSynchronize(S.prep_stream);
    for (Buf* b : {&S.in_pts, &S.in_scalars, &S.aff, &S.counts, &S.offsets, &S.cursor, &S.sorted, &S.buckets, &S.heads,
                   &S.tails, &S.chunk_out, &S.window_out, &S.tile_sums, &S.blk, &S.tiles, &S.result, &S.mul_out, &S.hacc,
                   &S.recv, &S.gsend, &S.grecv})
      b->release();
    for (auto& ev : S.ev_fin) cudaEventDestroy(ev);
    for (auto& ev : S.ev_xchg) cudaEventDestroy(ev);
    cudaEventDestroy(S.ev_gather);
    cudaFreeHost(S.h_gather);
    cudaStreamDestroy(S.comm_stream);
    for (auto& ev : S.ev) cudaEventDestroy(ev);
    for (auto& ev : S.ev_acc) cudaEventDestroy(ev);
    for (auto& ev : S.ev_tail) cudaEventDestroy(ev);
    for (cudaEvent_t ev : {S.done, S.ev_fork, S.ev_horner, S.ev_t0, S.ev_t1}) cudaEventDestroy(ev);
    cudaFreeHost(S.h_result);
    for (auto st : S.acc_stream) cudaStreamDestroy(st);
    for (auto st : S.tail_stream) cudaStreamDestroy(st);
    cudaStreamDestroy(S.horner_stream);
    cudaStreamDestroy(S.prep_stream);
    cudaEventDestroy(S.ev_start);
    cudaEventDestroy(S.ev_prep);
    cudaStreamDestroy(S.stream);
    S.pend = Pending();
  }
  h2d_release();
  C.ed_scratch.release();
  cudaFree(C.secp256k1_g_table);
  C.secp256k1_g_table = nullptr;
  cudaFree(C.p256_g_table);
  C.p256_g_table = nullptr;
  cudaFree(C.p384_g_table);
  C.p384_g_table = nullptr;
  cudaFree(C.kzg_roots);
  C.kzg_roots = nullptr;
  kzg_release_setups();
  cudaFree(C.ed25519_b_table);
  C.ed25519_b_table = nullptr;
  for (Buf* b : {&C.ntt_data, &C.ntt_work, &C.ntt_tmp, &C.ntt_roots, &C.ntt_aux}) b->release();
  C.ntt_key_field = -1;
  C.ntt_key_bits = -1;
  C.ready = false;
  C.device = -1;
}

const char* nmsm_last_error(void) {
  static thread_local std::string copy;  // the caller's pointer stays valid while other threads keep calling in
  std::lock_guard<std::mutex> lk(g_mu);
  copy = g_ctx.last_error;
  return copy.c_str();
}
long long nmsm_last_error_index(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  return g_ctx.last_error_index;
}

int nmsm_point_bytes(int curve) {
  ENGINE(curve);
  return E->point_bytes;
}
int nmsm_acc_bytes(int curve) {
  ENGINE(curve);
  return E->acc_bytes;
}

int nmsm_msm(int curve, const uint8_t* pts, const uint8_t* scalars, uint64_t n, uint8_t* out_xy, int* out_is_inf) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!out_xy || !out_is_inf || (n && (!pts || !scalars))) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  return E->msm_host(pts, scalars, n, out_xy, out_is_inf);
}

int nmsm_msm_device(int curve, const void* d_pts, const void* d_scalars, uint64_t n, uint8_t* out_xy,
                    int* out_is_inf) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!out_xy || !out_is_inf || (n && (!d_pts || !d_scalars))) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  return E->msm_device((const uint32_t*)d_pts, (const uint32_t*)d_scalars, n, nullptr, out_xy, out_is_inf);
}

int nmsm_msm_partial_device(int curve, const void* d_pts, const void* d_scalars, uint64_t n, void* d_out_acc) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!d_out_acc || (n && (!d_pts || !d_scalars))) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  return E->msm_device((const uint32_t*)d_pts, (const uint32_t*)d_scalars, n, (uint32_t*)d_out_acc, nullptr, nullptr);
}

int nmsm_fold_partials_device(int curve, const void* d_accs, int count, uint8_t* out_xy, int* out_is_inf) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!d_accs || count < 0 || !out_xy || !out_is_inf) return fail(NMSM_ERR_ARG, "bad argument");
  ENGINE(curve);
  return E->fold((const uint32_t*)d_accs, count, out_xy, out_is_inf);
}

int nmsm_accs_normalize(int curve, const void* accs, int on_device, uint64_t n, uint8_t* out_xy, uint8_t* out_is_inf) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n && (!accs || !out_xy || !out_is_inf)) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  return E->normalize(accs, on_device, n, out_xy, out_is_inf);
}

int nmsm_mul_batch(int curve, const uint8_t* pts, const uint8_t* scalars, uint64_t n, int allow_zero,
                   uint8_t* out_xy, uint8_t* out_is_inf) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n && (!pts || !scalars || !out_xy || !out_is_inf)) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  return E->mul_batch(pts, scalars, n, allow_zero, out_xy, out_is_inf);
}

int nmsm_points_torsion_free(int curve, const uint8_t* pts, uint64_t n, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n && (!pts || !out_ok)) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  return E->torsion_free(pts, n, out_ok);
}

// ---- device-resident point sets (fixed-base reuse) ---------------------------------------------
struct PointSet {
  int curve;
  uint64_t n;
  uint32_t* d_prepared;
  int table_c;       // 0: level 0 only; else window bits of the fixed-base table in d_prepared
  int table_levels;
};

int nmsm_points_upload(int curve, const uint8_t* pts, uint64_t n, uint64_t* out_handle) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!pts || !out_handle) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  uint32_t* d = nullptr;
  if (int r = E->prepare_points(pts, n, &d)) return r;
  PointSet* ps = new PointSet{curve, n, d, 0, 1};
  *out_handle = (uint64_t)(uintptr_t)ps;
  return NMSM_OK;
}

int nmsm_points_free(uint64_t handle) {
  std::lock_guard<std::mutex> lk(g_mu);
  PointSet* ps = (PointSet*)(uintptr_t)handle;
  if (!ps) return fail(NMSM_ERR_ARG, "null handle");
  cudaFree(ps->d_prepared);
  delete ps;
  return NMSM_OK;
}

int nmsm_msm_points(uint64_t handle, const uint8_t* scalars, uint64_t n, uint8_t* out_xy, int* out_is_inf) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  PointSet* ps = (PointSet*)(uintptr_t)handle;
  if (!ps || !out_xy || !out_is_inf || (n && !scalars)) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(ps->curve);
  return E->msm_prepared(ps->d_prepared, ps->n, ps->table_c, scalars, n, out_xy, out_is_inf);
}

int nmsm_msm_points_submit(uint64_t handle, const void* scalars, uint64_t n, int scalars_on_device, int slot) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  if (slot < 0 || slot >= NUM_SLOTS) return fail(NMSM_ERR_ARG, "slot out of range (0..3)");
  PointSet* ps = (PointSet*)(uintptr_t)handle;
  if (!ps || (n && !scalars)) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(ps->curve);
  g_ctx.cur = slot;
  return E->submit_prepared(ps->d_prepared, ps->n, ps->table_c, scalars, n, scalars_on_device);
}

int nmsm_points_precompute(uint64_t handle, int window_bits, int* out_window_bits, int* out_levels) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  PointSet* ps = (PointSet*)(uintptr_t)handle;
  if (!ps) return fail(NMSM_ERR_ARG, "null handle");
  if (ps->table_c) return fail(NMSM_ERR_ARG, "point set already carries a table");
  ENGINE(ps->curve);
  int c = 0, levels = 0;
  if (int r = E->precompute_table(&ps->d_prepared, ps->n, window_bits, &c, &levels)) return r;
  ps->table_c = c;
  ps->table_levels = levels;
  if (out_window_bits) *out_window_bits = c;
  if (out_levels) *out_levels = levels;
  return NMSM_OK;
}

// ---- fixed-point multiplication tables -----------------------------------------------------------
struct PointTable {
  int curve;
  uint32_t* d_tbl;
  int levels;
};

int nmsm_point_table_create(int curve, const uint8_t* point_xy, uint64_t* out_handle) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!point_xy || !out_handle) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  uint32_t* d = nullptr;
  int levels = 0;
  if (int r = E->build_point_table(point_xy, &d, &levels)) return r;
  *out_handle = (uint64_t)(uintptr_t) new PointTable{curve, d, levels};
  return NMSM_OK;
}

int nmsm_point_table_free(uint64_t handle) {
  std::lock_guard<std::mutex> lk(g_mu);
  PointTable* pt = (PointTable*)(uintptr_t)handle;
  if (!pt) return fail(NMSM_ERR_ARG, "null handle");
  cudaFree(pt->d_tbl);
  delete pt;
  return NMSM_OK;
}

int nmsm_point_table_mul_batch(uint64_t handle, const uint8_t* scalars, uint64_t n, int allow_zero, uint8_t* out_xy,
                               uint8_t* out_is_inf) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  PointTable* pt = (PointTable*)(uintptr_t)handle;
  if (!pt || (n && (!scalars || !out_xy || !out_is_inf))) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(pt->curve);
  return E->table_mul_batch(pt->d_tbl, scalars, n, allow_zero, out_xy, out_is_inf);
}

int nmsm_msm_submit(int curve, const void* pts, const void* scalars, uint64_t n, int inputs_on_device, int slot) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  if (slot < 0 || slot >= NUM_SLOTS) return fail(NMSM_ERR_ARG, "slot out of range (0..3)");
  if (n && (!pts || !scalars)) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  g_ctx.cur = slot;
  return E->submit(pts, scalars, n, inputs_on_device, nullptr, nullptr);
}

int nmsm_msm_submit_partial(int curve, const void* d_pts, const void* d_scalars, uint64_t n, void* d_out_acc, int slot) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  if (slot < 0 || slot >= NUM_SLOTS) return fail(NMSM_ERR_ARG, "slot out of range (0..3)");
  if (!d_out_acc || (n && (!d_pts || !d_scalars))) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  g_ctx.cur = slot;
  return E->submit(d_pts, d_scalars, n, 1, d_out_acc, nullptr);
}

// ---- multi-GPU: one process per GPU, NCCL communicator owned by the library ------------------------------------
int nmsm_dist_unique_id(uint8_t* out128) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!out128) return fail(NMSM_ERR_ARG, "null pointer");
  if (int r = nccl_load()) return r;
  ncclUniqueId id;
  if (int r = nccl_check(g_nccl.GetUniqueId(&id), "ncclGetUniqueId")) return r;
  static_assert(sizeof(id) == NMSM_DIST_ID_BYTES, "NCCL unique id size");
  memcpy(out128, &id, sizeof(id));
  return NMSM_OK;
}

int nmsm_dist_init(int rank, int world, const uint8_t* id128) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  if (g_dist.ready) {
    if (g_dist.rank == rank && g_dist.world == world) return NMSM_OK;
    return fail(NMSM_ERR_ARG, "nmsm_dist_init: already initialised with another rank / world size");
  }
  if (!id128 || world < 1 || rank < 0 || rank >= world) return fail(NMSM_ERR_ARG, "nmsm_dist_init: bad argument");
  if (int r = nccl_load()) return r;
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  ncclComm_t comm = nullptr;
  if (int r = nccl_check(g_nccl.CommInitRank(&comm, world, id, rank), "ncclCommInitRank")) return r;
  g_dist.comm = (NcclComm*)comm;
  g_dist.rank = rank;
  g_dist.world = world;
  g_dist.ready = true;
  // direct peer access for the bucket exchange: one process per GPU of one NVLink domain.  NMSM_DIST_P2P=0 falls back to
  // ncclSend / ncclRecv copies (also taken when a peer cannot be mapped).
  const char* e = getenv("NMSM_DIST_P2P");
  g_dist.p2p = world > 1 && world <= MAX_PEERS && !(e && atoi(e) == 0);
  if (g_dist.p2p) {
    int ndev = 0;
    cudaGetDeviceCount(&ndev);
    if (ndev >= world) {  // every rank's device is visible here: check the links
      for (int d = 0; d < ndev && g_dist.p2p; d++) {
        if (d == g_ctx.device) continue;
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, g_ctx.device, d) != cudaSuccess || !can) g_dist.p2p = false;
      }
    }
    (void)cudaGetLastError();
  }
  return NMSM_OK;
}

int nmsm_dist_info(int* out_rank, int* out_world, int* out_nccl_version) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_dist.ready) return fail(NMSM_ERR_ARG, "nmsm_dist_init has not been called");
  if (out_rank) *out_rank = g_dist.rank;
  if (out_world) *out_world = g_dist.world;
  if (out_nccl_version) g_nccl.GetVersion(out_nccl_version);
  return NMSM_OK;
}

int nmsm_dist_exchange_mode(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_dist.ready) return 0;
  return g_dist.p2p ? 2 : 1;
}

int nmsm_msm_sharded_submit(int curve, const void* pts, const void* scalars, uint64_t n_local, uint64_t n_total,
                            uint64_t shard_offset, int inputs_on_device, int slot) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  if (slot < 0 || slot >= NUM_SLOTS) return fail(NMSM_ERR_ARG, "slot out of range (0..3)");
  if (n_local && (!pts || !scalars)) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  g_ctx.cur = slot;
  ShardArgs sa{n_total, shard_offset};
  return E->submit(pts, scalars, n_local, inputs_on_device, nullptr, &sa);
}

int nmsm_msm_sharded(int curve, const void* pts, const void* scalars, uint64_t n_local, uint64_t n_total,
                     uint64_t shard_offset, int inputs_on_device, uint8_t* out_xy, int* out_is_inf) {
  if (!out_xy || !out_is_inf) return fail(NMSM_ERR_ARG, "null pointer");
  if (int r = nmsm_msm_sharded_submit(curve, pts, scalars, n_local, n_total, shard_offset, inputs_on_device, 0)) return r;
  return nmsm_msm_collect(0, out_xy, out_is_inf);
}

int nmsm_msm_collect(int slot, uint8_t* out_xy, int* out_is_inf) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  if (slot < 0 || slot >= NUM_SLOTS) return fail(NMSM_ERR_ARG, "slot out of range (0..3)");
  if (!g_ctx.slot[slot].pend.active) return fail(NMSM_ERR_ARG, "nothing submitted on this slot");
  if (!g_ctx.slot[slot].pend.partial && (!out_xy || !out_is_inf)) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(g_ctx.slot[slot].pend.curve);
  g_ctx.cur = slot;
  return E->collect(out_xy, out_is_inf);
}

int nmsm_ed25519_verify_batch(const uint8_t* sigs, const uint8_t* pubkeys, const uint8_t* msgs,
                              const uint64_t* msg_off, uint64_t n, const uint8_t* z16, int* out_ok,
                              long long* out_bad_index) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!out_ok || !out_bad_index || (n && (!sigs || !pubkeys || !msg_off || !z16)))
    return fail(NMSM_ERR_ARG, "null pointer");
  if (n && msg_off[n] && !msgs) return fail(NMSM_ERR_ARG, "null pointer");
  return ed25519_verify_batch_impl(sigs, pubkeys, msgs, msg_off, n, z16, out_ok, out_bad_index);
}

int nmsm_ed25519_verify_each(const uint8_t* sigs, const uint8_t* pubkeys, const uint8_t* msgs, const uint64_t* msg_off,
                             uint64_t n, int flags, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (flags & ~NMSM_ED25519_VERIFY_STRICT) return fail(NMSM_ERR_ARG, "nmsm_ed25519_verify_each: unknown flag");
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");  // before msg_off[n] is read
  if (!sigs || !pubkeys || !msg_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  if (msg_off[n] && !msgs) return fail(NMSM_ERR_ARG, "null pointer");
  return ed25519_verify_each_impl(sigs, pubkeys, msgs, msg_off, n, flags, out_ok);
}

int nmsm_secp256k1_verify_batch(const uint8_t* sigs, const uint8_t* pubkeys, const uint64_t* pk_off, const uint8_t* msgs,
                                const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (flags & ~(NMSM_ECDSA_PREHASH | NMSM_ECDSA_LOW_S)) return fail(NMSM_ERR_ARG, "nmsm_secp256k1_verify_batch: unknown flag");
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");  // before pk_off[n] / msg_off[n] are read
  if (!sigs || !pk_off || !msg_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  if ((pk_off[n] && !pubkeys) || (msg_off[n] && !msgs)) return fail(NMSM_ERR_ARG, "null pointer");
  return secp256k1_verify_batch_impl(sigs, pubkeys, pk_off, msgs, msg_off, n, flags, out_ok);
}

int nmsm_p256_verify_batch(const uint8_t* sigs, const uint8_t* pubkeys, const uint64_t* pk_off, const uint8_t* msgs,
                           const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (flags & ~(NMSM_ECDSA_PREHASH | NMSM_ECDSA_LOW_S)) return fail(NMSM_ERR_ARG, "nmsm_p256_verify_batch: unknown flag");
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");  // before pk_off[n] / msg_off[n] are read
  if (!sigs || !pk_off || !msg_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  if ((pk_off[n] && !pubkeys) || (msg_off[n] && !msgs)) return fail(NMSM_ERR_ARG, "null pointer");
  return p256_verify_batch_impl(sigs, pubkeys, pk_off, msgs, msg_off, n, flags, out_ok);
}

int nmsm_p384_verify_batch(const uint8_t* sigs, const uint8_t* pubkeys, const uint64_t* pk_off, const uint8_t* msgs,
                           const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (flags & ~(NMSM_ECDSA_PREHASH | NMSM_ECDSA_LOW_S)) return fail(NMSM_ERR_ARG, "nmsm_p384_verify_batch: unknown flag");
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");  // before pk_off[n] / msg_off[n] are read
  if (!sigs || !pk_off || !msg_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  if ((pk_off[n] && !pubkeys) || (msg_off[n] && !msgs)) return fail(NMSM_ERR_ARG, "null pointer");
  return p384_verify_batch_impl(sigs, pubkeys, pk_off, msgs, msg_off, n, flags, out_ok);
}

int nmsm_secp256k1_schnorr_verify_batch(const uint8_t* sigs, const uint8_t* pubkeys, const uint8_t* msgs,
                                        const uint64_t* msg_off, uint64_t n, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");  // before msg_off[n] is read
  if (!sigs || !pubkeys || !msg_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  if (msg_off[n] && !msgs) return fail(NMSM_ERR_ARG, "null pointer");
  return secp256k1_schnorr_verify_batch_impl(sigs, pubkeys, msgs, msg_off, n, out_ok);
}

int nmsm_secp256k1_recover_batch(const uint8_t* sigs65, const uint8_t* msgs, const uint64_t* msg_off, uint64_t n,
                                 int flags, uint8_t* out_xy, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (flags & ~NMSM_ECDSA_PREHASH) return fail(NMSM_ERR_ARG, "nmsm_secp256k1_recover_batch: unknown flag");
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");  // before msg_off[n] is read
  if (!sigs65 || !msg_off || !out_xy || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  if (msg_off[n] && !msgs) return fail(NMSM_ERR_ARG, "null pointer");
  return secp256k1_recover_batch_impl(sigs65, msgs, msg_off, n, flags, out_xy, out_ok);
}

int nmsm_secp256k1_ecrecover_batch(const uint8_t* inputs128, uint64_t n, uint8_t* out32, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 31)) return fail(NMSM_ERR_ARG, "n must be < 2^31");
  if (!inputs128 || !out32 || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  return secp256k1_ecrecover_batch_impl(inputs128, n, out32, out_ok);
}

int nmsm_bls12_381_pairing_check_batch(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                       uint64_t n_checks, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n_checks == 0) return NMSM_OK;
  if (!pair_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_pairing_check_batch_impl(g1_xy, g2_xy, pair_off, n_checks, out_ok);
}

int nmsm_bn254_pairing_check_batch(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                   uint64_t n_checks, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n_checks == 0) return NMSM_OK;
  if (!pair_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  return bn254_pairing_check_batch_impl(g1_xy, g2_xy, pair_off, n_checks, out_ok);
}

int nmsm_bls12_381_verify_batch(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msg_pts, uint64_t n,
                                uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n == 0) return NMSM_OK;
  if (!sigs96 || !pks48 || !msg_pts || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_verify_batch_impl(sigs96, pks48, msg_pts, n, out_ok);
}

int nmsm_bls12_381_hash_to_g2_batch(const uint8_t* msgs, const uint64_t* msg_off, uint64_t n, const uint8_t* dst,
                                    uint64_t dst_len, uint8_t* out_xy) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!dst) return fail(NMSM_ERR_ARG, "null pointer");
  if (dst_len == 0) return fail(NMSM_ERR_ARG, "dst must not be empty");
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");  // before msg_off[n] is read
  if (!msg_off || !out_xy) return fail(NMSM_ERR_ARG, "null pointer");
  if (msg_off[n] && !msgs) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_hash_to_g2_batch_impl(msgs, msg_off, n, dst, dst_len, out_xy);
}

int nmsm_bls12_381_verify_msg_batch(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msgs,
                                    const uint64_t* msg_off, uint64_t n, const uint8_t* dst, uint64_t dst_len,
                                    uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!dst) return fail(NMSM_ERR_ARG, "null pointer");
  if (dst_len == 0) return fail(NMSM_ERR_ARG, "dst must not be empty");
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");  // before msg_off[n] is read
  if (!sigs96 || !pks48 || !msg_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  if (msg_off[n] && !msgs) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_verify_msg_batch_impl(sigs96, pks48, msgs, msg_off, n, dst, dst_len, out_ok);
}

int nmsm_bls12_381_hash_to_g1_batch(const uint8_t* msgs, const uint64_t* msg_off, uint64_t n, const uint8_t* dst,
                                    uint64_t dst_len, uint8_t* out_xy) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!dst) return fail(NMSM_ERR_ARG, "null pointer");
  if (dst_len == 0) return fail(NMSM_ERR_ARG, "dst must not be empty");
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");  // before msg_off[n] is read
  if (!msg_off || !out_xy) return fail(NMSM_ERR_ARG, "null pointer");
  if (msg_off[n] && !msgs) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_hash_to_g1_batch_impl(msgs, msg_off, n, dst, dst_len, out_xy);
}

int nmsm_bls12_381_short_verify_batch(const uint8_t* sigs48, const uint8_t* pks96, const uint8_t* msg_pts, uint64_t n,
                                      uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n == 0) return NMSM_OK;
  if (!sigs48 || !pks96 || !msg_pts || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_short_verify_batch_impl(sigs48, pks96, msg_pts, n, out_ok);
}

int nmsm_bls12_381_short_verify_msg_batch(const uint8_t* sigs48, const uint8_t* pks96, const uint8_t* msgs,
                                          const uint64_t* msg_off, uint64_t n, const uint8_t* dst, uint64_t dst_len,
                                          uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!dst) return fail(NMSM_ERR_ARG, "null pointer");
  if (dst_len == 0) return fail(NMSM_ERR_ARG, "dst must not be empty");
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");  // before msg_off[n] is read
  if (!sigs48 || !pks96 || !msg_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  if (msg_off[n] && !msgs) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_short_verify_msg_batch_impl(sigs48, pks96, msgs, msg_off, n, dst, dst_len, out_ok);
}

int nmsm_bls12_381_aggregate_verify_batch(const uint8_t* sigs96, const uint64_t* group_off, uint64_t n_checks,
                                          const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* keys_xy,
                                          const uint64_t* key_off, const uint8_t* dst, uint64_t dst_len,
                                          uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!dst) return fail(NMSM_ERR_ARG, "null pointer");
  if (dst_len == 0) return fail(NMSM_ERR_ARG, "dst must not be empty");
  if (n_checks == 0) return NMSM_OK;
  if (!sigs96 || !group_off || !msg_off || !key_off || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_aggregate_verify_batch_impl(sigs96, group_off, n_checks, msgs, msg_off, keys_xy, key_off, dst,
                                               dst_len, out_ok);
}

int nmsm_bls12_381_kzg_verify_proof_batch(const uint8_t* commitments48, const uint8_t* zs32, const uint8_t* ys32,
                                          const uint8_t* proofs48, const uint8_t* versioned_hashes32, uint64_t n,
                                          const uint8_t* setup_g2_96, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");
  if (!commitments48 || !zs32 || !ys32 || !proofs48 || !setup_g2_96 || !out_ok)
    return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_kzg_verify_proof_batch_impl(commitments48, zs32, ys32, proofs48, versioned_hashes32, n, setup_g2_96,
                                               out_ok);
}

int nmsm_bls12_381_kzg_verify_blob_batch(const uint8_t* blobs, const uint8_t* commitments48, const uint8_t* proofs48,
                                         uint64_t n, const uint8_t* setup_g2_96, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");
  if (!blobs || !commitments48 || !proofs48 || !setup_g2_96 || !out_ok) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_kzg_verify_blob_batch_impl(blobs, commitments48, proofs48, n, setup_g2_96, out_ok);
}

int nmsm_bls12_381_kzg_setup_create(const uint8_t* g1_lagrange48, uint64_t* out_handle) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!g1_lagrange48 || !out_handle) return fail(NMSM_ERR_ARG, "null pointer");
  return bls12_381_kzg_setup_create_impl(g1_lagrange48, out_handle);
}

int nmsm_bls12_381_kzg_setup_free(uint64_t handle) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!handle) return fail(NMSM_ERR_ARG, "null handle");
  return bls12_381_kzg_setup_free_impl(handle);
}

// the argument checks the three provers share
static int kzg_prove_args(uint64_t setup, const uint8_t* blobs, uint64_t n, const void* in2, const uint8_t* out48,
                          const uint8_t* out_ok) {
  if (!setup) return fail(NMSM_ERR_ARG, "null handle");
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");
  if (n && (!blobs || !in2 || !out48 || !out_ok)) return fail(NMSM_ERR_ARG, "null pointer");
  return NMSM_OK;
}

int nmsm_bls12_381_kzg_commit_batch(uint64_t setup, const uint8_t* blobs, uint64_t n, uint8_t* out_commitments48,
                                    uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (int r = kzg_prove_args(setup, blobs, n, blobs, out_commitments48, out_ok)) return r;
  if (n == 0) return NMSM_OK;
  return bls12_381_kzg_commit_batch_impl(setup, blobs, n, out_commitments48, out_ok);
}

int nmsm_bls12_381_kzg_compute_proof_batch(uint64_t setup, const uint8_t* blobs, const uint8_t* zs32, uint64_t n,
                                           uint8_t* out_proofs48, uint8_t* out_ys32, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (int r = kzg_prove_args(setup, blobs, n, zs32, out_proofs48, out_ok)) return r;
  if (n && !out_ys32) return fail(NMSM_ERR_ARG, "null pointer");
  if (n == 0) return NMSM_OK;
  return bls12_381_kzg_compute_proof_batch_impl(setup, blobs, zs32, n, out_proofs48, out_ys32, out_ok);
}

int nmsm_bls12_381_kzg_compute_blob_proof_batch(uint64_t setup, const uint8_t* blobs, const uint8_t* commitments48,
                                                uint64_t n, uint8_t* out_proofs48, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (int r = kzg_prove_args(setup, blobs, n, commitments48, out_proofs48, out_ok)) return r;
  if (n == 0) return NMSM_OK;
  return bls12_381_kzg_compute_blob_proof_batch_impl(setup, blobs, commitments48, n, out_proofs48, out_ok);
}

int nmsm_points_decode_ex(int curve, const uint8_t* enc, uint64_t n, int flags, uint8_t* out_xy, uint8_t* out_status) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n && (!enc || !out_xy || !out_status)) return fail(NMSM_ERR_ARG, "null pointer");
  if (flags & ~NMSM_DECODE_ZIP215) return fail(NMSM_ERR_ARG, "nmsm_points_decode_ex: unknown flag");
  return decode_points_impl(curve, enc, n, flags, out_xy, out_status);
}

int nmsm_points_decode(int curve, const uint8_t* enc, uint64_t n, uint8_t* out_xy, uint8_t* out_status) {
  return nmsm_points_decode_ex(curve, enc, n, 0, out_xy, out_status);
}

int nmsm_points_on_curve(int curve, const uint8_t* pts, uint64_t n, uint8_t* out_ok) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (n && (!pts || !out_ok)) return fail(NMSM_ERR_ARG, "null pointer");
  ENGINE(curve);
  return E->on_curve(pts, n, out_ok);
}

int nmsm_set_window_bits(int c) {
  std::lock_guard<std::mutex> lk(g_mu);
  int prev = g_ctx.forced_c;
  g_ctx.forced_c = (c >= 1 && c <= 16) ? c : 0;
  return prev;
}

int nmsm_set_window_groups(int groups) {
  std::lock_guard<std::mutex> lk(g_mu);
  int prev = g_ctx.forced_groups;
  g_ctx.forced_groups = (groups >= 1 && groups <= MAX_GROUPS) ? groups : 0;
  return prev;
}

int nmsm_set_profiling(int enabled) {
  std::lock_guard<std::mutex> lk(g_mu);
  int prev = g_ctx.profiling ? 1 : 0;
  g_ctx.profiling = enabled != 0;
  return prev;
}

int nmsm_ntt(int curve, uint8_t* values, int log_n, uint64_t generator, int inverse, int brp_input, int brp_output) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!values) return fail(NMSM_ERR_ARG, "null pointer");
  return ntt_impl(curve, values, 0, log_n, generator, inverse, brp_input, brp_output);
}

int nmsm_ntt_device(int curve, void* d_values, int log_n, uint64_t generator, int inverse, int brp_input, int brp_output) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (int r = ensure_init()) return r;
  g_ctx.cur = 0;
  SLOT0_FREE();
  if (!d_values) return fail(NMSM_ERR_ARG, "null pointer");
  return ntt_impl(curve, d_values, 1, log_n, generator, inverse, brp_input, brp_output);
}

int nmsm_last_timing(float* ms, nmsm_plan_info* info) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (ms) memcpy(ms, g_ctx.last_ms, sizeof(g_ctx.last_ms));
  if (info) *info = g_ctx.last_info;
  return NMSM_OK;
}

double nmsm_bench_modmul(int field, int blocks_per_sm, int threads, int iters, int ilp) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (ensure_init()) return -1;
  if (blocks_per_sm < 1 || threads < 32 || threads > 1024 || iters < 1) return -1;
  if (field == 0) return bench_modmul<FpBn254>(blocks_per_sm, threads, iters, ilp);
  if (field == 1) return bench_modmul<FpBls381>(blocks_per_sm, threads, iters, ilp);
  return -1;
}

void* nmsm_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
  return p;
}
void nmsm_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

}  // extern "C"
