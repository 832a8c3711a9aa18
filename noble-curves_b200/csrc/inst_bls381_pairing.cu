// BLS12-381 pairing checks, BLS signature verification (SURVEY §8 row f7, pairing.cuh), hash to G2 (f10) and G1 (f13,
// hash_to_curve.cuh), short-signature verification (f13) and aggregate verification (f3, bls_aggregate.cuh): the kernels
// and the eight C-ABI implementations.  The chunked check driver is pairing_driver.cuh's (shared with bn254):
//   k_bls_hash_to_g2      (hash, verify_msg, aggregate) one thread per message: RFC 9380 hash_to_curve, affine through
//                         one inversion per warp
//   k_bls_hash_to_g1      (hash to G1, short verify_msg) the same for G1
//   k_bls_verify_prepare  (verify only) one thread per signature: decode, subgroup checks, the two pairs
//   k_bls_short_verify_prepare  (short verify only) the same with sig in G1 and pk in G2
//   k_bls_key_tiles       (aggregate only) one warp per tile of keys of one group: the partial key sums
//   k_bls_key_groups      (aggregate only) one thread per group: its key sum S_g and the pair (S_g, H(m_g))
//   k_bls_agg_prepare     (aggregate only) one thread per check: signature decode and subgroup check, the pair (-G1, sig)
//   k_bls_miller          one thread per pair: validation and f_i = f_{|x|,Q_i}(P_i) into the workspace
//   k_bls_final           one thread per check: the product of its f_i, the final exponentiation, the verdict
// The Miller values of at most PAIRING_CHUNK pairs are alive at once (PAIRING_CHUNK x 576 B = 37.7 MB).
#include "bls_aggregate.cuh"
#include "hash_to_curve.cuh"
#include "pairing.cuh"
#include "pairing_driver.cuh"

namespace nmsm {

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bls_miller(uint64_t q0, uint32_t cnt, const uint32_t* __restrict__ g1, const uint32_t* __restrict__ g2,
             uint32_t* __restrict__ W, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) pairing_miller_body<BlsPairing>(q0 + i, g1, g2, W + (size_t)i * BLS_F12_WORDS, err);
}

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bls_final(uint64_t j0, uint32_t cnt, const uint64_t* __restrict__ off, uint64_t q0, uint64_t q1,
            const uint32_t* __restrict__ W, const uint32_t* carry_in, uint32_t* carry_out,
            const uint8_t* __restrict__ pre_ok, uint8_t* __restrict__ out_ok) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) pairing_final_body<BlsPairing>(j0 + i, off, q0, q1, W, carry_in, carry_out, pre_ok, out_ok);
}

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bls_verify_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                     const uint32_t* __restrict__ msg_pts, uint32_t* __restrict__ g1, uint32_t* __restrict__ g2,
                     uint8_t* __restrict__ pre_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) bls_verify_prepare_body(i, sigs, pks, msg_pts, g1, g2, pre_ok, err);
}

// Lanes past n feed the identity, whose inversion target is 1, to the warp-shared inversion.
__global__ void __launch_bounds__(128)
k_bls_hash_to_g2(uint32_t n, const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ msg_off,
                 const uint8_t* __restrict__ dst, uint32_t dlen, uint32_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  H2cG::Acc q = H2cG::identity();
  if (i < n) q = h2c_hash_body(i, msgs, msg_off, dst, dlen);
  const H2cF2 zi = warp_batch_inverse(H2cG::inv_target(q));
  if (i < n) h2c_store(i, q, zi, out);
}

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bls_short_verify_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ pks,
                           const uint32_t* __restrict__ msg_pts, uint32_t* __restrict__ g1, uint32_t* __restrict__ g2,
                           uint8_t* __restrict__ pre_ok, unsigned int* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) bls_short_verify_prepare_body(i, sigs, pks, msg_pts, g1, g2, pre_ok, err);
}

// Lanes past n feed the identity, whose inversion target is 1, to the warp-shared inversion.
__global__ void __launch_bounds__(128)
k_bls_hash_to_g1(uint32_t n, const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ msg_off,
                 const uint8_t* __restrict__ dst, uint32_t dlen, uint32_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  H2cG1::Acc q = H2cG1::identity();
  if (i < n) q = h2c_hash_body_g1(i, msgs, msg_off, dst, dlen);
  const H2cF zi = warp_batch_inverse(H2cG1::inv_target(q));
  if (i < n) h2c_store_g1(i, q, zi, out);
}

// one warp per tile (4 per block): lane sums, then a shuffle tree whose lane 0 writes the partial and the bad flag
__global__ void __launch_bounds__(128)
k_bls_key_tiles(uint32_t n_tiles, const BlsKeyTile* __restrict__ tiles, const uint32_t* __restrict__ keys,
                uint32_t* __restrict__ partials, uint8_t* __restrict__ tile_bad, unsigned int* err) {
  const uint32_t t = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= n_tiles) return;  // the whole warp
  bool bad = false;
  BlsG1::Acc acc = bls_key_lane(tiles[t], lane, keys, bad, err);
  for (uint32_t d = BLS_KEY_LANES / 2; d; d >>= 1) {
    const int src = lane + d < 32 ? lane + d : lane;
    const BlsG1::Acc o{shfl_field(acc.X, src), shfl_field(acc.Y, src), shfl_field(acc.ZZ, src), shfl_field(acc.ZZZ, src)};
    BlsG1::add(acc, o);
  }
  bad = __any_sync(0xffffffffu, bad);
  if (lane == 0) {
    uint32_t w[BLS_ACC_WORDS];
    BlsG1::store_acc(w, acc);
    store_words<BLS_ACC_WORDS>(partials + (size_t)t * BLS_ACC_WORDS, w);
    tile_bad[t] = bad ? 1 : 0;
  }
}

// one thread per group; lanes past n and bad groups feed 1 to the warp-shared inversion
__global__ void __launch_bounds__(128)
k_bls_key_groups(uint32_t n_groups, const uint32_t* __restrict__ tile_off, const uint32_t* __restrict__ partials,
                 const uint8_t* __restrict__ tile_bad, const uint32_t* __restrict__ group_pair,
                 const uint32_t* __restrict__ h, uint32_t* __restrict__ g1, uint32_t* __restrict__ g2,
                 uint8_t* __restrict__ group_ok) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  bool ok = false;
  BlsG1::Acc s = BlsG1::identity();
  if (g < n_groups) s = bls_group_sum(g, tile_off, partials, tile_bad, ok);
  const BlsF zi = warp_batch_inverse(ok ? s.ZZZ : BlsF::one());
  if (g < n_groups) bls_group_store(g, group_pair[g], ok, s, zi, h, g1, g2, group_ok);
}

__global__ void __launch_bounds__(PAIRING_BLOCK)
k_bls_agg_prepare(uint32_t n, const uint8_t* __restrict__ sigs, const uint64_t* __restrict__ group_off,
                  const uint8_t* __restrict__ group_ok, uint32_t* __restrict__ g1, uint32_t* __restrict__ g2,
                  uint8_t* __restrict__ pre_ok) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) bls_agg_prepare_body(j, sigs, group_off, group_ok, g1, g2, pre_ok);
}

const PairingKernels BLS_KERNELS{k_bls_miller, k_bls_final};

namespace {

// keys per tile of k_bls_key_tiles, and the most tiles one group is split into (bls_key_tiles)
constexpr uint64_t BLS_KEY_TILE = 128, BLS_KEY_TILE_CAP = 256;

// messages hashed to G2 on the device: msgs / msg_off as the C ABI takes them, the tag already at most H2C_MAX_DST bytes
struct BlsMessages {
  const uint8_t* msgs;
  const uint64_t* msg_off;
  const uint8_t* dst;
  uint32_t dlen;
};

// the tag of RFC 9380 §5.3.3: a DST over 255 bytes is replaced by SHA-256("H2C-OVERSIZE-DST-" || DST)
BlsMessages bls_messages(const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* dst, uint64_t dst_len,
                         std::vector<uint8_t>& tag) {
  if (dst_len <= H2C_MAX_DST) return BlsMessages{msgs, msg_off, dst, (uint32_t)dst_len};
  static const char PREFIX[] = "H2C-OVERSIZE-DST-";
  std::vector<uint8_t> in(PREFIX, PREFIX + sizeof(PREFIX) - 1);
  in.insert(in.end(), dst, dst + dst_len);
  tag.resize(32);
  sha256(in.data(), in.size(), tag.data());
  return BlsMessages{msgs, msg_off, tag.data(), 32};
}

// workspace bytes of bls_hash_launch for n messages
uint64_t bls_hash_bytes(const BlsMessages& m, uint64_t n) { return al256(m.msg_off[n] + 16) + al256(8 * (n + 1)) + 256; }

// uploads the messages, offsets and tag to ws (bls_hash_bytes) and runs k_bls_hash_to_g2, or k_bls_hash_to_g1 when g1,
// into d_out (timing slot 0)
int bls_hash_launch(Context& X, Slot& C, const BlsMessages& m, uint64_t n, uint8_t* ws, uint32_t* d_out,
                    bool g1 = false) {
  cudaStream_t st = C.stream;
  const uint64_t msg_bytes = m.msg_off[n], o_mo = al256(msg_bytes + 16), o_dst = o_mo + al256(8 * (n + 1));
  if (msg_bytes)
    if (int r = h2d_any(ws, m.msgs, msg_bytes, st)) return r;
  if (int r = h2d_any(ws + o_mo, m.msg_off, 8 * (n + 1), st)) return r;
  if (int r = h2d_any(ws + o_dst, m.dst, m.dlen, st)) return r;
  return pairing_launch(X, C, 0, [&] {
    (g1 ? k_bls_hash_to_g1 : k_bls_hash_to_g2)<<<cdiv(n, 128), 128, 0, st>>>(
        (uint32_t)n, ws, (const uint64_t*)(ws + o_mo), ws + o_dst, m.dlen, d_out);
  });
}

// nmsm_bls12_381_verify_batch (msg_pts on the host) and nmsm_bls12_381_verify_msg_batch (hm: the messages, hashed
// into the same workspace by k_bls_hash_to_g2, which shifts the other kernels' timing slots by one); with short_sigs,
// the short-signature forms (48-byte G1 signatures, 96-byte G2 keys, G1 message points and k_bls_hash_to_g1)
int bls_verify_impl(const uint8_t* sigs, const uint8_t* pks, const uint8_t* msg_pts, const BlsMessages* hm,
                    uint64_t n, uint8_t* out_ok, bool short_sigs = false) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");
  if (X.profiling) memset(X.last_ms, 0, sizeof(X.last_ms));
  const uint64_t sig_b = short_sigs ? 48 : 96, pk_b = short_sigs ? 96 : 48, h_b = short_sigs ? 96 : 192;
  const uint64_t o_sig = 0, o_pk = o_sig + al256(sig_b * n), o_h = o_pk + al256(pk_b * n), o_g1 = o_h + al256(h_b * n),
                 o_g2 = o_g1 + al256(192 * n), o_pre = o_g2 + al256(384 * n),
                 o_w = o_pre + al256(n), o_ok = o_w + al256(pairing_workspace_bytes<BlsPairing>()),
                 o_misc = o_ok + al256(n), o_hash = o_misc + 256, bytes = o_hash + (hm ? bls_hash_bytes(*hm, n) : 0);
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  const int s0 = hm ? 1 : 0;
  if (int r = h2d_any(base + o_sig, sigs, sig_b * n, st)) return r;
  if (int r = h2d_any(base + o_pk, pks, pk_b * n, st)) return r;
  if (hm) {
    if (int r = bls_hash_launch(X, C, *hm, n, base + o_hash, (uint32_t*)(base + o_h), short_sigs)) return r;
  } else if (int r = h2d_any(base + o_h, msg_pts, h_b * n, st)) {
    return r;
  }
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  uint32_t *d_g1 = (uint32_t*)(base + o_g1), *d_g2 = (uint32_t*)(base + o_g2);
  uint8_t *d_pre = base + o_pre, *d_ok = base + o_ok;
  CK(cudaMemsetAsync(d_err, 0xff, 16, st));
  if (int r = pairing_launch(X, C, s0, [&] {
        (short_sigs ? k_bls_short_verify_prepare : k_bls_verify_prepare)<<<cdiv(n, PAIRING_BLOCK), PAIRING_BLOCK, 0,
                                                                           st>>>(
            (uint32_t)n, base + o_sig, base + o_pk, (const uint32_t*)(base + o_h), d_g1, d_g2, d_pre, d_err);
      }))
    return r;
  if (int r = pairing_checks_run<BlsPairing>(X, C, BLS_KERNELS, n, nullptr, nullptr, d_g1, d_g2, d_pre,
                                              (uint32_t*)(base + o_w), d_ok, d_err + 2, 1 + s0))
    return r;
  unsigned int err[4];
  CK(cudaMemcpyAsync(err, d_err, 16, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (err[0] != 0xffffffffu)  // hashed messages are on their curve by construction
    return fail(hm ? NMSM_ERR_CUDA : NMSM_ERR_POINT,
                (hm ? "internal error: hashed message point " : "message point ") + std::to_string(err[0]) +
                    (short_sigs ? " is out of range or not on the curve" : " is out of range or not on the twist"),
                err[0]);
  if (err[2] != 0xffffffffu || err[3] != 0xffffffffu)  // prepare only emits valid or identity pairs
    return fail(NMSM_ERR_CUDA, "internal error: a prepared pair failed validation");
  CK(cudaMemcpy(out_ok, d_ok, n, cudaMemcpyDeviceToHost));
  return NMSM_OK;
}

// nmsm_bls12_381_aggregate_verify_batch after the argument checks of capi.cu: 0 < n < 2^30, the offsets checked,
// n_groups + n < 2^31 and n_keys < 2^31
int bls_aggregate_impl(const uint8_t* sigs96, const uint64_t* group_off, uint64_t n, const BlsMessages& hm,
                       const uint8_t* keys_xy, const uint64_t* key_off, uint8_t* out_ok) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  const uint64_t n_groups = group_off[n], n_keys = n_groups ? key_off[n_groups] : 0, n_pairs = n_groups + n;
  if (n_groups == 0) {  // every check is empty
    memset(out_ok, 0, n);
    return NMSM_OK;
  }
  if (X.profiling) memset(X.last_ms, 0, sizeof(X.last_ms));
  std::vector<BlsKeyTile> tiles;
  std::vector<uint32_t> tile_off, group_pair(n_groups);
  bls_key_tiles(key_off, n_groups, BLS_KEY_TILE, BLS_KEY_TILE_CAP, tiles, tile_off);
  std::vector<uint64_t> pair_off(n + 1);
  for (uint64_t j = 0; j <= n; j++) pair_off[j] = group_off[j] + j;
  for (uint64_t j = 0; j < n; j++)
    for (uint64_t g = group_off[j]; g < group_off[j + 1]; g++) group_pair[g] = (uint32_t)(g + j);
  const uint64_t nt = tiles.size();
  const uint64_t o_sig = 0, o_goff = o_sig + al256(96 * n), o_poff = o_goff + al256(8 * (n + 1)),
                 o_keys = o_poff + al256(8 * (n + 1)), o_tiles = o_keys + al256(96 * n_keys),
                 o_toff = o_tiles + al256(8 * nt), o_gpair = o_toff + al256(4 * (n_groups + 1)),
                 o_part = o_gpair + al256(4 * n_groups), o_tbad = o_part + al256(4 * BLS_ACC_WORDS * nt),
                 o_h = o_tbad + al256(nt), o_g1 = o_h + al256(192 * n_groups), o_g2 = o_g1 + al256(96 * n_pairs),
                 o_gok = o_g2 + al256(192 * n_pairs), o_pre = o_gok + al256(n_groups), o_w = o_pre + al256(n),
                 o_ok = o_w + al256(pairing_workspace_bytes<BlsPairing>()), o_misc = o_ok + al256(n),
                 o_hash = o_misc + 256, bytes = o_hash + bls_hash_bytes(hm, n_groups);
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  cudaStream_t st = C.stream;
  if (int r = h2d_any(base + o_sig, sigs96, 96 * n, st)) return r;
  if (int r = h2d_any(base + o_goff, group_off, 8 * (n + 1), st)) return r;
  if (int r = h2d_any(base + o_poff, pair_off.data(), 8 * (n + 1), st)) return r;
  if (n_keys)
    if (int r = h2d_any(base + o_keys, keys_xy, 96 * n_keys, st)) return r;
  if (nt)
    if (int r = h2d_any(base + o_tiles, tiles.data(), 8 * nt, st)) return r;
  if (int r = h2d_any(base + o_toff, tile_off.data(), 4 * (n_groups + 1), st)) return r;
  if (int r = h2d_any(base + o_gpair, group_pair.data(), 4 * n_groups, st)) return r;
  unsigned int* d_err = (unsigned int*)(base + o_misc);
  CK(cudaMemsetAsync(d_err, 0xff, 16, st));
  uint32_t *d_h = (uint32_t*)(base + o_h), *d_g1 = (uint32_t*)(base + o_g1), *d_g2 = (uint32_t*)(base + o_g2),
           *d_part = (uint32_t*)(base + o_part);
  uint8_t *d_tbad = base + o_tbad, *d_gok = base + o_gok, *d_pre = base + o_pre, *d_ok = base + o_ok;
  if (int r = bls_hash_launch(X, C, hm, n_groups, base + o_hash, d_h)) return r;
  if (nt)
    if (int r = pairing_launch(X, C, 1, [&] {
          k_bls_key_tiles<<<cdiv(nt, 4), 128, 0, st>>>((uint32_t)nt, (const BlsKeyTile*)(base + o_tiles),
                                                       (const uint32_t*)(base + o_keys), d_part, d_tbad, d_err);
        }))
      return r;
  if (int r = pairing_launch(X, C, 1, [&] {
        k_bls_key_groups<<<cdiv(n_groups, 128), 128, 0, st>>>((uint32_t)n_groups, (const uint32_t*)(base + o_toff),
                                                              d_part, d_tbad, (const uint32_t*)(base + o_gpair), d_h,
                                                              d_g1, d_g2, d_gok);
      }))
    return r;
  if (int r = pairing_launch(X, C, 2, [&] {
        k_bls_agg_prepare<<<cdiv(n, PAIRING_BLOCK), PAIRING_BLOCK, 0, st>>>(
            (uint32_t)n, base + o_sig, (const uint64_t*)(base + o_goff), d_gok, d_g1, d_g2, d_pre);
      }))
    return r;
  if (int r = pairing_checks_run<BlsPairing>(X, C, BLS_KERNELS, n, pair_off.data(), (const uint64_t*)(base + o_poff),
                                              d_g1, d_g2, d_pre, (uint32_t*)(base + o_w), d_ok, d_err + 2, 3))
    return r;
  unsigned int err[4];
  CK(cudaMemcpyAsync(err, d_err, 16, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (err[0] != 0xffffffffu)
    return fail(NMSM_ERR_POINT, "key " + std::to_string(err[0]) + " is out of range or not on the curve", err[0]);
  if (err[2] != 0xffffffffu || err[3] != 0xffffffffu)  // key sums and hashed messages are on their curves
    return fail(NMSM_ERR_CUDA, "internal error: an aggregate pair failed validation");
  CK(cudaMemcpy(out_ok, d_ok, n, cudaMemcpyDeviceToHost));
  return NMSM_OK;
}
}  // namespace

int bls12_381_aggregate_verify_batch_impl(const uint8_t* sigs96, const uint64_t* group_off, uint64_t n_checks,
                                          const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* keys_xy,
                                          const uint64_t* key_off, const uint8_t* dst, uint64_t dst_len,
                                          uint8_t* out_ok) {
  if (n_checks == 0) return NMSM_OK;
  if (n_checks >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n_checks must be < 2^30");
  if (int r = check_offsets(group_off, "group_off", n_checks)) return r;
  const uint64_t n_groups = group_off[n_checks];
  if (n_groups >= (1ull << 31) - n_checks) return fail(NMSM_ERR_ARG, "the number of pairs must be < 2^31");
  if (int r = check_offsets(msg_off, "msg_off", n_groups)) return r;
  if (int r = check_offsets(key_off, "key_off", n_groups)) return r;
  if (key_off[n_groups] >= (1ull << 31)) return fail(NMSM_ERR_ARG, "the number of keys must be < 2^31");
  if ((msg_off[n_groups] && !msgs) || (key_off[n_groups] && !keys_xy)) return fail(NMSM_ERR_ARG, "null pointer");
  std::vector<uint8_t> tag;
  const BlsMessages hm = bls_messages(msgs, msg_off, dst, dst_len, tag);
  return bls_aggregate_impl(sigs96, group_off, n_checks, hm, keys_xy, key_off, out_ok);
}

int bls12_381_pairing_check_batch_impl(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                       uint64_t n_checks, uint8_t* out_ok) {
  return pairing_check_batch_impl<BlsPairing>(BLS_KERNELS, g1_xy, g2_xy, pair_off, n_checks, out_ok);
}

int bls12_381_verify_batch_impl(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msg_pts, uint64_t n,
                                uint8_t* out_ok) {
  return bls_verify_impl(sigs96, pks48, msg_pts, nullptr, n, out_ok);
}

int bls12_381_verify_msg_batch_impl(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msgs,
                                    const uint64_t* msg_off, uint64_t n, const uint8_t* dst, uint64_t dst_len,
                                    uint8_t* out_ok) {
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");
  if (int r = check_offsets(msg_off, "msg_off", n)) return r;
  std::vector<uint8_t> tag;
  const BlsMessages hm = bls_messages(msgs, msg_off, dst, dst_len, tag);
  return bls_verify_impl(sigs96, pks48, nullptr, &hm, n, out_ok);
}

namespace {
// nmsm_bls12_381_hash_to_g2_batch, or nmsm_bls12_381_hash_to_g1_batch when g1 (96-byte instead of 192-byte points)
int bls_hash_impl(const uint8_t* msgs, const uint64_t* msg_off, uint64_t n, const uint8_t* dst, uint64_t dst_len,
                  uint8_t* out_xy, bool g1) {
  Context& X = g_ctx;
  Slot& C = X.slot[0];
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");
  if (int r = check_offsets(msg_off, "msg_off", n)) return r;
  std::vector<uint8_t> tag;
  const BlsMessages hm = bls_messages(msgs, msg_off, dst, dst_len, tag);
  if (X.profiling) memset(X.last_ms, 0, sizeof(X.last_ms));
  const uint64_t pt_b = g1 ? 96 : 192, o_out = 0, o_hash = al256(pt_b * n), bytes = o_hash + bls_hash_bytes(hm, n);
  CK(X.ed_scratch.ensure(bytes));
  uint8_t* base = (uint8_t*)X.ed_scratch.p;
  if (int r = bls_hash_launch(X, C, hm, n, base + o_hash, (uint32_t*)(base + o_out), g1)) return r;
  CK(cudaMemcpyAsync(out_xy, base + o_out, pt_b * n, cudaMemcpyDeviceToHost, C.stream));
  CK(cudaStreamSynchronize(C.stream));
  return NMSM_OK;
}
}  // namespace

int bls12_381_hash_to_g2_batch_impl(const uint8_t* msgs, const uint64_t* msg_off, uint64_t n, const uint8_t* dst,
                                    uint64_t dst_len, uint8_t* out_xy) {
  return bls_hash_impl(msgs, msg_off, n, dst, dst_len, out_xy, false);
}

int bls12_381_hash_to_g1_batch_impl(const uint8_t* msgs, const uint64_t* msg_off, uint64_t n, const uint8_t* dst,
                                    uint64_t dst_len, uint8_t* out_xy) {
  return bls_hash_impl(msgs, msg_off, n, dst, dst_len, out_xy, true);
}

int bls12_381_short_verify_batch_impl(const uint8_t* sigs48, const uint8_t* pks96, const uint8_t* msg_pts, uint64_t n,
                                      uint8_t* out_ok) {
  return bls_verify_impl(sigs48, pks96, msg_pts, nullptr, n, out_ok, true);
}

int bls12_381_short_verify_msg_batch_impl(const uint8_t* sigs48, const uint8_t* pks96, const uint8_t* msgs,
                                          const uint64_t* msg_off, uint64_t n, const uint8_t* dst, uint64_t dst_len,
                                          uint8_t* out_ok) {
  if (n == 0) return NMSM_OK;
  if (n >= (1ull << 30)) return fail(NMSM_ERR_ARG, "n must be < 2^30");
  if (int r = check_offsets(msg_off, "msg_off", n)) return r;
  std::vector<uint8_t> tag;
  const BlsMessages hm = bls_messages(msgs, msg_off, dst, dst_len, tag);
  return bls_verify_impl(sigs48, pks96, nullptr, &hm, n, out_ok, true);
}

}  // namespace nmsm
