// Process-wide context, error mapping and the per-curve dispatch table shared by capi.cu and the
// per-curve translation units (inst_*.cu).  No kernels are visible from here, so capi.cu does not
// re-instantiate the curve templates.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "../../include/nmsm.h"

namespace nmsm {
struct MsmPlanLite {  // mirror of MsmPlan (msm_body.cuh) so this header stays free of device code
  int c, W, B, G, L, K, chunks, D;
  uint32_t TPW;
};
}  // namespace nmsm

namespace nmsm {

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
struct Buf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

// Everything one in-flight MSM needs.  NMSM_SLOTS slots let the caller keep several MSMs in flight (nmsm_msm_submit /
// nmsm_msm_collect): the latency-bound tail of one (second-level reduction, Horner, inversion — a handful of
// SMs) overlaps the H2D copy and the wide kernels of the next on the other stream.
struct Pending {
  bool active = false;
  int curve = -1;
  MsmPlanLite plan = {};
  uint64_t n = 0;
  bool partial = false;   // raw accumulator requested instead of an affine result
  bool empty = false;     // n == 0
  bool sharded = false;   // multi-GPU bucket-exchange MSM: errors of every rank arrive in h_gather
  int gather_words = 0;   // words per rank in h_gather
  bool profiled = false;  // per-kernel events were recorded at submit (nmsm_set_profiling was on then)
  int groups = 1;         // window groups the pipeline was split into
  int launches = 0;       // kernels launched for this MSM
};
static constexpr int MAX_GROUPS = 8;       // window groups per single-GPU MSM (engine.cuh submit_msm)
static constexpr int MAX_WINDOWS = 34;     // sharded MSMs run one group per window: 16-bit windows over <= 256+1 bits, c >= 8
static constexpr int ACC_STREAMS = 8, TAIL_STREAMS = 4;  // 8 accumulate streams: a sharded MSM launches one (small) accumulate kernel per window, all must be able to run at once
struct Slot {
  cudaStream_t stream = nullptr;
  // Window-group pipelining: the per-group accumulate launches alternate between two low-priority streams (the
  // next group's blocks fill the SMs as the previous group's drain), every finished group's bucket reduction runs
  // on a high-priority tail stream, and the Horner steps on their own high-priority stream.
  cudaStream_t acc_stream[ACC_STREAMS] = {}, tail_stream[TAIL_STREAMS] = {}, horner_stream = nullptr;
  cudaStream_t prep_stream = nullptr;  // k_prepare (multiplier-bound) runs beside the digit count / scan / scatter (atomics-bound)
  cudaEvent_t ev_start = nullptr, ev_prep = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_acc[MAX_WINDOWS] = {}, ev_tail[MAX_WINDOWS] = {}, ev_horner = nullptr;
  // multi-GPU bucket exchange (nmsm_msm_sharded_*): NCCL calls are issued on comm_stream
  cudaStream_t comm_stream = nullptr;
  cudaEvent_t ev_fin[MAX_WINDOWS] = {}, ev_xchg[MAX_WINDOWS] = {}, ev_gather = nullptr;
  uint32_t* h_gather = nullptr;  // pinned copy of the gathered window results + error words
  Buf recv, gsend, grecv;
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;  // whole-MSM device time, always recorded
  // NMSM_TRACE=1 (debugging aid): timing events at the end of every group's accumulate / reduction / Horner step
  cudaEvent_t tr_fork = nullptr, tr_acc[MAX_WINDOWS] = {}, tr_tail[MAX_WINDOWS] = {}, tr_h[MAX_WINDOWS] = {};
  Buf in_pts, in_scalars, aff, counts, offsets, cursor, sorted, buckets, heads, tails, chunk_out, window_out, tile_sums,
      blk, tiles, result, mul_out, hacc;
  uint32_t* h_result = nullptr;  // pinned staging for (xy | inf | err0 | err1 | entries)
  cudaEvent_t ev[NMSM_TIMING_SLOTS + 2] = {};
  cudaEvent_t done = nullptr;
  float last_ms[NMSM_TIMING_SLOTS] = {};
  nmsm_plan_info last_info = {};
  Pending pend;
};
static constexpr int NUM_SLOTS = NMSM_SLOTS;  // include/nmsm.h

struct Context {
  bool ready = false;
  int device = -1;
  int sm_count = 132;  // H100 SXM; nmsm_init reads the device's count
  Slot slot[NUM_SLOTS];
  int cur = 0;  // slot used by the call in progress (set by the C-ABI wrapper under the mutex)
  Buf ed_scratch;              // signature-verification scratch (ed25519 and secp256k1 batches)
  uint32_t* secp256k1_g_table = nullptr;  // fixed-point table of the secp256k1 generator, built by the first verify
  uint32_t* ed25519_b_table = nullptr;    // fixed-point table of the ed25519 base point, built by the first verify_each
  uint32_t* p256_g_table = nullptr;       // fixed-point table of the P-256 generator, built by the first P-256 verify
  uint32_t* p384_g_table = nullptr;       // fixed-point table of the P-384 generator, built by the first P-384 verify
  uint32_t* kzg_roots = nullptr;          // the EIP-4844 bit-reversed domain (Montgomery form), built by the first blob verify
  Buf ntt_data, ntt_work, ntt_tmp, ntt_roots, ntt_aux;  // NTT staging / work / output / root table (ntt.cu)
  int ntt_key_field = -1, ntt_key_bits = -1;            // which root table ntt_roots holds
  uint64_t ntt_key_gen = 0;
  bool profiling = false;
  bool trace = false;
  int forced_c = 0;
  int forced_groups = 0;  // 0 = automatic (nmsm_set_window_groups)
  float last_ms[NMSM_TIMING_SLOTS] = {};
  nmsm_plan_info last_info = {};
  std::string last_error;
  long long last_error_index = -1;
};

// H2D copy of a caller's host array, ordered before later work on `stream`.  Pinned (cudaHostAlloc / cudaHostRegister /
// nmsm_host_alloc) sources go out as one cudaMemcpyAsync.  Large PAGEABLE sources — what a JS typed array or a Python
// bytes object is — would be staged by the driver on ONE thread, well below the pinned PCIe rate; instead a few worker
// threads copy chunks into a ring of pinned staging buffers
// and issue the chunk DMAs themselves, which keeps PCIe near its pinned rate.  capi.cu.
int h2d_any(void* dst, const void* src, size_t bytes, cudaStream_t stream);
void h2d_release();

// NCCL entry points resolved at run time (dlopen "libnccl.so.2": inside a torch process that is the copy torch already
// loaded), so libnmsm.so has no link-time dependency on NCCL and loads on machines without it.
struct NcclComm;
static constexpr int MAX_PEERS = 16;  // ranks of one NVLink domain
struct PeerPtrs {                      // passed to k_bucket_fold by value: every rank's bucket array (own entry unused)
  const uint32_t* p[MAX_PEERS];
};
struct DistState {
  bool ready = false;
  int rank = 0, world = 1;
  NcclComm* comm = nullptr;
  // Direct exchange: every rank's `buckets` workspace of a slot is mapped into every other rank through CUDA IPC, so the
  // window owners PULL the peers' partial buckets over NVLink inside the fold kernel instead of receiving copies.
  bool p2p = false;                                    // all peers reachable (same NVLink domain, IPC works)
  void* mapped[NMSM_SLOTS][MAX_PEERS] = {};            // peer r's buckets base in this process (nullptr for self)
  void* mapped_local[NMSM_SLOTS] = {};                 // the local allocation the mappings were exchanged for
};
int nccl_send(const void* buf, size_t bytes, int peer, cudaStream_t st);
int nccl_recv(void* buf, size_t bytes, int peer, cudaStream_t st);
int nccl_group_start();
int nccl_group_end();
int nccl_all_gather(const void* send, void* recv, size_t bytes_per_rank, cudaStream_t st);
int dist_map_peer_buckets(int slot, void* local_base, cudaStream_t st);  // collective: (re)exchange the IPC mappings
extern DistState g_dist;

struct ShardArgs {  // sharded MSM: this GPU holds n_local of the n_total terms, starting at global index `offset`
  uint64_t n_total, offset;
};

extern Context g_ctx;
extern std::mutex g_mu;

inline int fail(int code, const std::string& msg, long long idx = -1) {
  g_ctx.last_error = msg;
  g_ctx.last_error_index = idx;
  return code;
}
inline int cuda_fail(cudaError_t e, const char* what) {
  return fail(NMSM_ERR_CUDA, std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
}
#define CK(call)                                         \
  do {                                                   \
    cudaError_t e__ = (call);                            \
    if (e__ != cudaSuccess) return cuda_fail(e__, #call); \
  } while (0)

// the offsets drive device reads of the concatenated keys / messages: they must start at 0 and never decrease
inline int check_offsets(const uint64_t* off, const char* name, uint64_t n) {
  if (off[0] != 0) return fail(NMSM_ERR_ARG, std::string(name) + "[0] must be 0");
  for (uint64_t i = 0; i < n; i++)
    if (off[i + 1] < off[i])
      return fail(NMSM_ERR_ARG, std::string(name) + " must be non-decreasing (index " + std::to_string(i + 1) + ")",
                  (long long)(i + 1));
  return NMSM_OK;
}

// the size of one piece of a scratch layout, rounded up so that the next piece starts 256-byte aligned
inline uint64_t al256(uint64_t x) { return (x + 255) & ~255ull; }

inline int ensure_init() {
  if (g_ctx.ready) return NMSM_OK;
  return fail(NMSM_ERR_CUDA, "nmsm_init() has not been called (no CUDA context; there is no CPU fallback)");
}


// One table per curve, defined in inst_<curve>.cu
struct EngineVTable {
  int point_bytes;
  int acc_bytes;
  int (*msm_host)(const uint8_t* pts, const uint8_t* scalars, uint64_t n, uint8_t* out_xy, int* out_is_inf);
  int (*msm_device)(const uint32_t* d_pts, const uint32_t* d_scalars, uint64_t n, uint32_t* d_out_acc,
                    uint8_t* out_xy, int* out_is_inf);
  int (*fold)(const uint32_t* d_accs, int count, uint8_t* out_xy, int* out_is_inf);
  int (*mul_batch)(const uint8_t* pts, const uint8_t* scalars, uint64_t n, int allow_zero, uint8_t* out_xy,
                   uint8_t* out_is_inf);
  int (*prepare_points)(const uint8_t* pts, uint64_t n, uint32_t** out_dev);
  // table_c != 0: d_prepared carries the fixed-base table built by precompute_table for that window size
  int (*msm_prepared)(const uint32_t* d_prepared, uint64_t n_points, int table_c, const uint8_t* scalars, uint64_t n,
                      uint8_t* out_xy, int* out_is_inf);
  // replaces *d_prepared (level 0) by a buffer holding all levels 2^(c*j) * P; c_req = 0 picks c by the cost model
  int (*precompute_table)(uint32_t** d_prepared, uint64_t n_points, int c_req, int* out_c, int* out_levels);
  // fixed-point multiplication table d * 2^(16 j) * P and the batch multiply through it
  int (*build_point_table)(const uint8_t* point_xy, uint32_t** out_tbl, int* out_levels);
  int (*table_mul_batch)(const uint32_t* tbl, const uint8_t* scalars, uint64_t n, int allow_zero, uint8_t* out_xy,
                         uint8_t* out_is_inf);
  // asynchronous halves on the slot g_ctx.cur: enqueue (optionally H2D from host pointers) / wait + read back
  int (*submit)(const void* pts, const void* scalars, uint64_t n, int inputs_on_device, void* d_out_acc, const ShardArgs* shard);
  int (*collect)(uint8_t* out_xy, int* out_is_inf);
  int (*submit_prepared)(const uint32_t* d_prepared, uint64_t n_points, int table_c, const void* scalars, uint64_t n,
                         int scalars_on_device);
  int (*torsion_free)(const uint8_t* pts, uint64_t n, uint8_t* out_ok);
  int (*on_curve)(const uint8_t* pts, uint64_t n, uint8_t* out_ok);
  int (*normalize)(const void* accs, int on_device, uint64_t n, uint8_t* out_xy, uint8_t* out_is_inf);
};
int ed25519_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs, const uint64_t* msg_off,
                              uint64_t n, const uint8_t* z16, int* out_ok, long long* out_bad_index);
int ed25519_verify_each_impl(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs, const uint64_t* msg_off,
                             uint64_t n, int flags, uint8_t* out_ok);
int secp256k1_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                                const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok);
int p256_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                           const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok);
int p384_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint64_t* pk_off, const uint8_t* msgs,
                           const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok);
int secp256k1_schnorr_verify_batch_impl(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msgs,
                                        const uint64_t* msg_off, uint64_t n, uint8_t* out_ok);
int secp256k1_recover_batch_impl(const uint8_t* sigs65, const uint8_t* msgs, const uint64_t* msg_off, uint64_t n,
                                 int flags, uint8_t* out_xy, uint8_t* out_ok);
int secp256k1_ecrecover_batch_impl(const uint8_t* inputs128, uint64_t n, uint8_t* out32, uint8_t* out_ok);
int bls12_381_pairing_check_batch_impl(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                       uint64_t n_checks, uint8_t* out_ok);
int bn254_pairing_check_batch_impl(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                   uint64_t n_checks, uint8_t* out_ok);
int bls12_381_verify_batch_impl(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msg_pts, uint64_t n,
                                uint8_t* out_ok);
int bls12_381_verify_msg_batch_impl(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msgs,
                                    const uint64_t* msg_off, uint64_t n, const uint8_t* dst, uint64_t dst_len,
                                    uint8_t* out_ok);
int bls12_381_hash_to_g2_batch_impl(const uint8_t* msgs, const uint64_t* msg_off, uint64_t n, const uint8_t* dst,
                                    uint64_t dst_len, uint8_t* out_xy);
int bls12_381_hash_to_g1_batch_impl(const uint8_t* msgs, const uint64_t* msg_off, uint64_t n, const uint8_t* dst,
                                    uint64_t dst_len, uint8_t* out_xy);
int bls12_381_short_verify_batch_impl(const uint8_t* sigs48, const uint8_t* pks96, const uint8_t* msg_pts, uint64_t n,
                                      uint8_t* out_ok);
int bls12_381_short_verify_msg_batch_impl(const uint8_t* sigs48, const uint8_t* pks96, const uint8_t* msgs,
                                          const uint64_t* msg_off, uint64_t n, const uint8_t* dst, uint64_t dst_len,
                                          uint8_t* out_ok);
int bls12_381_aggregate_verify_batch_impl(const uint8_t* sigs96, const uint64_t* group_off, uint64_t n_checks,
                                          const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* keys_xy,
                                          const uint64_t* key_off, const uint8_t* dst, uint64_t dst_len,
                                          uint8_t* out_ok);
int bls12_381_kzg_verify_proof_batch_impl(const uint8_t* commitments48, const uint8_t* zs32, const uint8_t* ys32,
                                          const uint8_t* proofs48, const uint8_t* versioned_hashes32, uint64_t n,
                                          const uint8_t* setup_g2_96, uint8_t* out_ok);
int bls12_381_kzg_verify_blob_batch_impl(const uint8_t* blobs, const uint8_t* commitments48, const uint8_t* proofs48,
                                         uint64_t n, const uint8_t* setup_g2_96, uint8_t* out_ok);
int bls12_381_kzg_setup_create_impl(const uint8_t* g1_lagrange48, uint64_t* out_handle);
int bls12_381_kzg_setup_free_impl(uint64_t handle);
void kzg_release_setups();  // nmsm_shutdown: frees every setup table (the handles stay until nmsm_bls12_381_kzg_setup_free)
int bls12_381_kzg_commit_batch_impl(uint64_t setup, const uint8_t* blobs, uint64_t n, uint8_t* out_commitments48,
                                    uint8_t* out_ok);
int bls12_381_kzg_compute_proof_batch_impl(uint64_t setup, const uint8_t* blobs, const uint8_t* zs32, uint64_t n,
                                           uint8_t* out_proofs48, uint8_t* out_ys32, uint8_t* out_ok);
int bls12_381_kzg_compute_blob_proof_batch_impl(uint64_t setup, const uint8_t* blobs, const uint8_t* commitments48,
                                                uint64_t n, uint8_t* out_proofs48, uint8_t* out_ok);
int decode_points_impl(int curve, const uint8_t* enc, uint64_t n, int flags, uint8_t* out_xy, uint8_t* out_status);
int ntt_impl(int curve, void* values, int on_device, int log_n, uint64_t generator, int inverse, int brp_input,
             int brp_output);
const EngineVTable* engine_secp256k1();
const EngineVTable* engine_ed25519();
const EngineVTable* engine_bn254g1();
const EngineVTable* engine_bn254g2();
const EngineVTable* engine_bls381g1();
const EngineVTable* engine_bls381g1_any();
const EngineVTable* engine_bls381g2();
const EngineVTable* engine_bls381g2_any();

}  // namespace nmsm
