/* nmsm — C ABI of the H100-native (sm_90a) scalar-multiplication / MSM engine.
 *
 * This is the drop-in boundary for noble-curves' hot path (SURVEY §8b).  noble has no FFI of its
 * own; these entry points are what an N-API addon (see INTEGRATION.md) binds behind the reference's
 * public functions:
 *
 *   nmsm_msm            <- pippenger(c, points, scalars)          /root/reference/src/abstract/curve.ts:863-905
 *   nmsm_mul_batch      <- Point.multiply / Point.multiplyUnsafe  src/abstract/weierstrass.ts:900-928,
 *                                                                 src/abstract/edwards.ts:555-577
 *   nmsm_msm_partial_device / nmsm_fold_partials_device           (multi-GPU split of the same MSM; MSM is
 *                                                                 linear in its term set, curve.ts:863)
 *   nmsm_dist_init / nmsm_msm_sharded                             the same MSM sharded over the GPUs of one box with the
 *                                                                 per-window bucket exchange inside the library (SURVEY §8e)
 *   nmsm_accs_normalize <- normalizeZ(c, points)                  curve.ts:311-326 (batch normalisation, one inversion per 32)
 *   nmsm_points_on_curve <- the equation half of assertValidity   weierstrass.ts:617-624,752-771
 *   nmsm_last_error     <- the thrown Error messages              curve.ts:390-404,875
 * and, for the callers and data formats either side of that path (SURVEY §8 f1-f4):
 *   nmsm_msm_submit / _collect / nmsm_msm_points_submit           asynchronous halves (several MSMs in flight)
 *   nmsm_points_upload / _precompute / nmsm_msm_points            interleavedMSMUnsafe, Point.precompute  curve.ts:532-577,937-959
 *   nmsm_point_table_*  <- P.precompute(W) + cached P.multiply(k) curve.ts:532-606 (BASE.multiply at rate)
 *   nmsm_points_decode / nmsm_points_torsion_free  <- Point.fromBytes: decode + isTorsionFree
 *                                                                 weierstrass.ts:541-605,971-975, bls12-381.ts:377-468
 *   nmsm_ed25519_verify_batch <- ed25519.verify over a batch      edwards.ts:942-989
 *   nmsm_secp256k1_verify_batch <- secp256k1.verify over a batch, one verdict per signature (weierstrass.ts ecdsa().verify)
 *   nmsm_secp256k1_schnorr_verify_batch <- schnorr.verify over a batch, one verdict per signature (secp256k1.ts, BIP340)
 *   nmsm_secp256k1_recover_batch <- secp256k1.recoverPublicKey over a batch (weierstrass.ts Signature.recoverPublicKey)
 *   nmsm_secp256k1_ecrecover_batch <- Ethereum's ecrecover precompile (0x01) over a batch
 *   nmsm_bls12_381_pairing_check_batch / nmsm_bn254_pairing_check_batch <- pairingBatch(...) == 1, one verdict per check
 *   nmsm_bls12_381_hash_to_g2_batch <- bls12_381.G2.hashToCurve(msg, { DST }) over a batch (RFC 9380)
 *   nmsm_bls12_381_verify_msg_batch <- bls12_381.verify over a batch with the messages hashed on the GPU
 *   nmsm_ntt           <- FFT(rootsOfUnity(Fr, G), Fr).direct / .inverse   src/abstract/fft.ts:518-575
 *
 * Data formats (all little-endian, plain bytes, caller-owned):
 *   point   : canonical affine (x, y); each base-field coordinate is FpBytes little-endian bytes
 *             (32 for secp256k1 / ed25519 / bn254, 48 for BLS12-381); Fp2 coordinates are c0 then c1.
 *             Weierstrass infinity is (0, 0) (weierstrass.ts:716,966); Edwards identity is (0, 1).
 *   scalar  : 32 bytes little-endian, 0 <= s < n (curve order).
 *   result  : same point format + `is_inf` flag (1 = identity).
 * Coordinates are NOT Montgomery form at this boundary.
 *
 * Error convention: 0 = ok; negative = error (see NMSM_ERR_*), message via nmsm_last_error().
 * Threading: one context per process (per GPU); calls are serialised by an internal mutex.
 * No CPU fallback exists: every entry point fails with NMSM_ERR_CUDA when no device is usable.
 */
#ifndef NMSM_H
#define NMSM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  NMSM_SECP256K1 = 0,
  NMSM_ED25519 = 1,
  NMSM_BN254_G1 = 2,
  NMSM_BN254_G2 = 3,
  NMSM_BLS12_381_G1 = 4,      /* points in the prime-order subgroup (what assertValidity / fromBytes accept): GLV schedule */
  NMSM_BLS12_381_G2 = 5,      /* points in the prime-order subgroup: psi-GLS schedule (4 windows instead of 16) */
  NMSM_BLS12_381_G1_ANY = 6,  /* any point of E(Fp), e.g. before a subgroup check or cofactor clearing: plain windows */
  NMSM_BLS12_381_G2_ANY = 7   /* any point of the twist E'(Fp2): plain windows */
};
/* Why two ids for BLS12-381 G1: the reference's pippenger is the plain group law and accepts every Point instance.
 * The GLV endomorphism phi(P) = lambda * P this engine uses for MSMs only holds on the prime-order subgroup; the
 * curve's cofactor is 0x396c8c005555e1568c00aaab0000aaab.  With id 4 the MSM equals the reference on every input the
 * reference itself considers a valid G1 point (on curve and torsion-free, weierstrass.ts:690-707); with id 6 on every
 * on-curve point, at 16 windows instead of 8.  nmsm_mul_batch (Point.multiply) never relies on the subgroup: it is
 * what isTorsionFree / clearCofactor run.  secp256k1 and bn254 G1 have cofactor 1: no distinction needed.
 * BLS12-381 G2 likewise: id 5 splits every term four ways along psi, which is multiplication by the curve parameter
 * only on the prime-order subgroup of the twist (bls12-381.ts:600); id 7 is the plain schedule for every on-curve point. */

enum {
  NMSM_OK = 0,
  NMSM_ERR_ARG = -1,            /* bad curve id / null pointer / size                                   */
  NMSM_ERR_SCALAR = -2,         /* 'invalid scalar at index i' (curve.ts:402); i = nmsm_last_error_index */
  NMSM_ERR_POINT = -3,          /* 'invalid point at index i'  (curve.ts:393)                            */
  NMSM_ERR_LENGTH = -4,         /* 'arrays of points and scalars must have equal length' (curve.ts:875)  */
  NMSM_ERR_CUDA = -5            /* CUDA failure or no device                                             */
};

/* Bind this process to CUDA device `device` and create the context (stream, workspace). Idempotent. */
int nmsm_init(int device);
void nmsm_shutdown(void);
const char* nmsm_last_error(void);
long long nmsm_last_error_index(void);

/* Bytes per point (x||y) and per raw accumulator for a curve; negative on bad id. */
int nmsm_point_bytes(int curve);
int nmsm_acc_bytes(int curve);

/* sum_i scalars[i] * pts[i]; host buffers (copied H2D inside the call).  n == 0 -> identity. */
int nmsm_msm(int curve, const uint8_t* pts, const uint8_t* scalars, uint64_t n, uint8_t* out_xy,
             int* out_is_inf);

/* Same with inputs already resident in device memory (16-byte aligned device pointers).
 * Stream ordering: every *_device / *_submit entry point launches on the library's own non-blocking streams, which are
 * NOT ordered against the caller's streams.  The producer of d_pts / d_scalars must have completed (event / stream /
 * device synchronize on the caller's side) before the call; the buffers must stay untouched until the call (or the
 * matching *_collect) returns.  nmsm/dist.py and bench.py synchronize the torch stream before they hand pointers over. */
int nmsm_msm_device(int curve, const void* d_pts, const void* d_scalars, uint64_t n, uint8_t* out_xy,
                    int* out_is_inf);

/* Several MSMs in flight: enqueue on slot 0..NMSM_SLOTS-1 without waiting, collect later (each slot has its own
 * stream and workspace; one outstanding MSM per slot).  The latency-bound tail of one MSM
 * (second-level bucket reduction, Horner doublings, inversion: a handful of SMs) then overlaps the H2D copy and the
 * wide kernels of the next.  With inputs_on_device = 0 the host buffers (pinned, for true overlap) must stay valid
 * until nmsm_msm_collect returns.  Errors of the MSM itself (invalid point / scalar) are reported by collect. */
#define NMSM_SLOTS 4
int nmsm_msm_submit(int curve, const void* pts, const void* scalars, uint64_t n, int inputs_on_device, int slot);
int nmsm_msm_collect(int slot, uint8_t* out_xy, int* out_is_inf);
/* Same for a multi-GPU shard: the raw accumulator lands in d_out_acc (device); collect with NULL outputs. */
int nmsm_msm_submit_partial(int curve, const void* d_pts, const void* d_scalars, uint64_t n, void* d_out_acc, int slot);

/* Multi-GPU building blocks: the un-normalised accumulator of a shard is written to device memory
 * (nmsm_acc_bytes bytes, opaque Montgomery-form words), exchanged by the caller (NCCL all-gather),
 * and folded + normalised by nmsm_fold_partials_device. */
int nmsm_msm_partial_device(int curve, const void* d_pts, const void* d_scalars, uint64_t n, void* d_out_acc);
int nmsm_fold_partials_device(int curve, const void* d_accs, int count, uint8_t* out_xy, int* out_is_inf);

/* normalizeZ (/root/reference/src/abstract/curve.ts:311-326) for raw accumulators: n un-normalised results (host buffer
 * or, with on_device != 0, device pointer; nmsm_acc_bytes each, the layout nmsm_msm_partial_device writes) -> canonical
 * affine x||y per point + one infinity flag byte each, with ONE field inversion per 32 points (Montgomery's trick,
 * modular.ts:734-760 FpInvertBatch).  The identity comes back as (0,0) / Edwards (0,1) with flag 1. */
int nmsm_accs_normalize(int curve, const void* accs, int on_device, uint64_t n, uint8_t* out_xy, uint8_t* out_is_inf);

/* Multi-GPU MSM with a bucket exchange (SURVEY §8e; BASELINE north_star: "a single NCCL allreduce over NVLink of the
 * per-window bucket accumulators").  One process per GPU.  The (point, scalar) array is split across the ranks; every
 * rank accumulates its shard into the full W x B bucket array with the window size of the WHOLE MSM (n_total), window w
 * belongs to rank w % world: after a window's accumulation its dense bucket array goes to the owner (ncclSend/ncclRecv
 * on the library's own stream, overlapping the accumulation of the next windows), the owner folds the partial buckets
 * (EC addition is not an ncclRedOp_t, hence exchange + fold kernel), reduces ONE window's buckets and applies the
 * window weight 2^(c w); a final ncclAllGather of the weighted window sums (a few hundred bytes per rank) and one fold
 * give every rank the same affine result.  No host synchronisation between the shard's kernels and the exchange.
 *   nmsm_dist_unique_id : rank 0 creates the NCCL id (128 bytes) and hands it to the other ranks by any channel
 *                         (torch.distributed broadcast in the Python mirror, nmsm/dist.py)
 *   nmsm_dist_init      : every rank, after nmsm_init(local device)
 *   nmsm_msm_sharded    : collective call — every rank passes ITS shard [shard_offset, shard_offset + n_local) of the
 *                         n_total terms (n_local may be 0) and receives the full result.  Invalid points / scalars on
 *                         any rank are reported on every rank with their GLOBAL index, points before scalars.
 *   nmsm_msm_sharded_submit + nmsm_msm_collect: the asynchronous halves (ranks must submit in the same order). */
#define NMSM_DIST_ID_BYTES 128
int nmsm_dist_unique_id(uint8_t* out128);
int nmsm_dist_init(int rank, int world, const uint8_t* id128);
int nmsm_dist_info(int* out_rank, int* out_world, int* out_nccl_version);
/* How the partial buckets travel to their window owners: 0 = nmsm_dist_init not called, 1 = grouped ncclSend / ncclRecv
 * copies, 2 = the owners read the peers' buckets in place over NVLink (CUDA-IPC mappings; every rank falls back to 1
 * together when a mapping cannot be opened or NMSM_DIST_P2P=0).  Final after the first sharded MSM. */
int nmsm_dist_exchange_mode(void);
int nmsm_msm_sharded(int curve, const void* pts, const void* scalars, uint64_t n_local, uint64_t n_total,
                     uint64_t shard_offset, int inputs_on_device, uint8_t* out_xy, int* out_is_inf);
int nmsm_msm_sharded_submit(int curve, const void* pts, const void* scalars, uint64_t n_local, uint64_t n_total,
                            uint64_t shard_offset, int inputs_on_device, int slot);

/* out[i] = scalars[i] * pts[i] for i < n (host buffers).  allow_zero = 0: Point.multiply range
 * (1 <= k < n); allow_zero = 1: Point.multiplyUnsafe range (0 <= k < n).  out_is_inf: n bytes. */
int nmsm_mul_batch(int curve, const uint8_t* pts, const uint8_t* scalars, uint64_t n, int allow_zero,
                   uint8_t* out_xy, uint8_t* out_is_inf);

/* out_ok[i] = 1 iff n * pts[i] == O: the batch form of Point.isTorsionFree (/root/reference/src/abstract/
 * weierstrass.ts:971-975, edwards.ts:584-586; bls12-381.ts:567-577,599-601 and bn254.ts:241 decide the same predicate
 * with endomorphism shortcuts) — the subgroup check that follows decoding untrusted points (next-row f2).  The
 * identity counts as torsion-free.  Works on any on-curve point (no GLV on curves with a cofactor). */
int nmsm_points_torsion_free(int curve, const uint8_t* pts, uint64_t n, uint8_t* out_ok);

/* Device-resident point sets: validate + convert a point array once, then run many MSMs against it
 * (fixed-base commitments).  The analogue of interleavedMSMUnsafe's captured tables
 * (/root/reference/src/abstract/curve.ts:937-959): fewer scalars than points use the first n points
 * (except on curves that run GLV internally — secp256k1, bn254 G1, BLS12-381 G1 — where n must equal the set
 * size). */
int nmsm_points_upload(int curve, const uint8_t* pts, uint64_t n, uint64_t* out_handle);
int nmsm_points_free(uint64_t handle);
int nmsm_msm_points(uint64_t handle, const uint8_t* scalars, uint64_t n, uint8_t* out_xy, int* out_is_inf);
/* Fixed-base table for the set (next-row f4): stores 2^(c*j) * P_i for j = 0..levels-1 on the device, the counterpart
 * of Point.precompute / the per-point window tables interleavedMSMUnsafe builds once
 * (/root/reference/src/abstract/curve.ts:532-577,937-951).  Later nmsm_msm_points calls then use ONE bucket window
 * of 2^(c-1) buckets for all digits: no Horner doublings and 1/W of the bucket reduction.  window_bits = 0 lets the
 * cost model choose (19 for 2^20 BLS12-381 G1 points: 7 levels, 1.4 GB); the choice is returned.  One-off cost:
 * levels-1 kernels of c doublings + one inversion per point. */
int nmsm_points_precompute(uint64_t handle, int window_bits, int* out_window_bits, int* out_levels);
/* Asynchronous nmsm_msm_points on a slot (collect with nmsm_msm_collect): the prover loop over a fixed SRS.  The
 * scalars may already be on the device (scalars_on_device = 1, 16-byte aligned); host scalars must stay valid until
 * the collect. */
int nmsm_msm_points_submit(uint64_t handle, const void* scalars, uint64_t n, int scalars_on_device, int slot);

/* Fixed-point multiplication tables (next-row f4): the device-resident form of Point.precompute(W) and the cached
 * signed-window multiply it enables (/root/reference/src/abstract/curve.ts:532-577 table, :588-606 walk; used by
 * BASE.multiply in getPublicKey / sign, weierstrass.ts:1168,1519).  The table holds d * 2^(16 j) * P for
 * d in [1, 2^15] and every 16-bit digit position j, so k * P is 16-17 gathered mixed additions and no doublings.
 * nmsm_point_table_mul_batch: out[i] = scalars[i] * P, same ranges / outputs as nmsm_mul_batch. */
int nmsm_point_table_create(int curve, const uint8_t* point_xy, uint64_t* out_handle);
int nmsm_point_table_free(uint64_t handle);
int nmsm_point_table_mul_batch(uint64_t handle, const uint8_t* scalars, uint64_t n, int allow_zero, uint8_t* out_xy,
                               uint8_t* out_is_inf);

/* NTT over the scalar field Fr of a pairing curve (next-row f4: the MSM's companion in SNARK provers): the batch
 * form of FFT(rootsOfUnity(Fr, generator), Fr).direct / .inverse (/root/reference/src/abstract/fft.ts:518-575; root
 * tables :230-312, loops :422-480).  `values`: 2^log_n elements of 32 bytes, canonical little-endian (< r),
 * transformed in place.  curve: NMSM_BN254_G1/G2 (Fr of bn254, 2-adicity 28) or NMSM_BLS12_381_G1/G2 (2-adicity 32).
 * generator: the non-residue G of rootsOfUnity (the reference's tests pass 7); 0 = findGenerator's choice
 * (fft.ts:175-180: 5 for both fields).  The argument is G mod r and must fit in 64 bits: a caller holding a larger G
 * reduces it mod r first and cannot pass one whose residue is 0 or >= 2^64 (the Python mirror raises ValueError for
 * those rather than truncate them).  inverse = 0: direct(values, brp_input, brp_output), out[k] = a(omega^k);
 * inverse = 1: inverse(values, brp_input, brp_output) incl. the 1/n scaling.  An element >= r is reported as
 * NMSM_ERR_SCALAR with its index and leaves `values` untouched. */
int nmsm_ntt(int curve, uint8_t* values, int log_n, uint64_t generator, int inverse, int brp_input, int brp_output);
int nmsm_ntt_device(int curve, void* d_values, int log_n, uint64_t generator, int inverse, int brp_input, int brp_output);

/* Ed25519 batch verification (next-row f1).  The reference verifies one signature at a time
 * (/root/reference/src/abstract/edwards.ts:942-989, ZIP-215 decoding by default, src/ed25519.ts:168); this checks
 *   [8]( sum z_i*R_i + sum (z_i*k_i mod l)*A_i - (sum z_i*s_i mod l)*B ) == O ,  k_i = SHA-512(R_i||A_i||M_i) mod l
 * on the GPU (decompression, SHA-512, scalar arithmetic mod l, Edwards MSM of 2n+1 terms).
 * sigs: n x 64 B; pubkeys: n x 32 B; msgs: concatenated message bytes, message i = [msg_off[i], msg_off[i+1]);
 * z16: n x 16 B caller-supplied random 128-bit coefficients (little-endian).
 * out_ok = 1 iff every R_i/A_i decodes, every s_i < l and the batch equation holds.  out_bad_index = smallest
 * index that can be rejected without the equation (undecodable point or s >= l), else -1. */
int nmsm_ed25519_verify_batch(const uint8_t* sigs, const uint8_t* pubkeys, const uint8_t* msgs,
                              const uint64_t* msg_off, uint64_t n, const uint8_t* z16, int* out_ok,
                              long long* out_bad_index);

/* secp256k1 ECDSA batch verification (next-row f5): out_ok[i] = secp256k1.verify(sig_i, msg_i, pk_i, { prehash, lowS })
 * with format 'compact' (noble-curves weierstrass.ts ecdsa().verify), one independent verdict per signature.
 * sigs: n x 64 B compact r || s, big-endian.  Key i = pubkeys[pk_off[i], pk_off[i+1]): 33-byte SEC1 compressed or
 * 65-byte uncompressed; message i = msgs[msg_off[i], msg_off[i+1]), any length.  out_ok: n bytes, 1 = valid.
 * Everything about a signature's content (r or s out of [1, n), a high s under NMSM_ECDSA_LOW_S, an undecodable key, a
 * raw message over 8192 bytes, R = O) is a 0 verdict, never an error; NMSM_ERR_ARG is for null pointers, offsets that do
 * not start at 0 or decrease, unknown flag bits and n >= 2^31.  n == 0 writes nothing.  The first ECDSA or Schnorr verify
 * after nmsm_init builds the fixed-point table of G (17 x 2^15 points, 36 MB), kept until nmsm_shutdown.  With profiling on
 * (nmsm_set_profiling), nmsm_last_timing reports k_ecdsa_prepare in slot 0, k_ecdsa_check in slot 1 and both in
 * NMSM_T_TOTAL. */
#define NMSM_ECDSA_PREHASH 1 /* h = bits2int(sha256(msg_i)) (the reference's default prehash: true) */
#define NMSM_ECDSA_LOW_S 2   /* s > n/2 verifies false (the reference's default lowS: true for secp256k1) */
int nmsm_secp256k1_verify_batch(const uint8_t* sigs, const uint8_t* pubkeys, const uint64_t* pk_off, const uint8_t* msgs,
                                const uint64_t* msg_off, uint64_t n, int flags, uint8_t* out_ok);

/* secp256k1 BIP340 Schnorr batch verification (next-row f6): out_ok[i] = schnorr.verify(sig_i, msg_i, pk_i)
 * (noble-curves secp256k1.ts), one independent verdict per signature.
 * sigs: n x 64 B r || s, big-endian; pubkeys: n x 32 B x-only keys; message i = msgs[msg_off[i], msg_off[i+1]), any
 * length.  out_ok: n bytes, 1 = valid.  Everything about a signature's content (a key x >= p or without a square root,
 * r >= p, s >= n, r or s zero, R = O, an odd y(R), x(R) != r) is a 0 verdict, never an error; NMSM_ERR_ARG is for null
 * pointers, offsets that do not start at 0 or decrease, and n >= 2^31.  n == 0 writes nothing.  Shares the fixed-point
 * table of G with nmsm_secp256k1_verify_batch: whichever verifies first after nmsm_init builds it.  With profiling on,
 * nmsm_last_timing reports k_schnorr_prepare in slot 0, k_schnorr_check in slot 1 and both in NMSM_T_TOTAL. */
int nmsm_secp256k1_schnorr_verify_batch(const uint8_t* sigs, const uint8_t* pubkeys, const uint8_t* msgs,
                                        const uint64_t* msg_off, uint64_t n, uint8_t* out_ok);

/* secp256k1 ECDSA public-key recovery (next-row f9): the batch form of noble-curves v2
 * secp256k1.recoverPublicKey(signature, message, { prehash }) with the 65-byte 'recovered' signature format.
 * sigs65: n x 65 B = recovery id (1 B) || r || s (32 B each, big-endian).  message i = msgs[msg_off[i], msg_off[i+1]).
 * flags: 0 or NMSM_ECDSA_PREHASH.  out_xy: n x 64 B, the recovered key in the library's affine packing (little-endian
 * x || y, as nmsm_mul_batch writes it); out_ok: n bytes, 1 = recovered.  A failed item gets out_ok 0 and 64 zero
 * bytes, never an error.  The rules (weierstrass.ts Signature.recoverPublicKey; each failure is where it throws):
 *   recovery id rec in {0, 1, 2, 3};  1 <= r < n, 1 <= s < n (no lowS rule: a high s recovers);
 *   x = r + n if rec & 2, else r;  x < p;  R = the SEC1 decode of (rec & 1 ? 03 : 02) || x (x^3 + 7 must be a square);
 *   h = bits2int_modN(prehash ? sha256(msg) : msg), a raw message over 8192 bytes fails as in verify;
 *   u1 = -h r^-1, u2 = s r^-1 (mod n);  Q = u1 G + u2 R;  Q = O fails.
 * NMSM_ERR_ARG is for null pointers, offsets that do not start at 0 or decrease, unknown flag bits and n >= 2^31.  n == 0
 * writes nothing.  Shares the fixed-point table of G with the ECDSA and Schnorr verifiers and
 * nmsm_secp256k1_ecrecover_batch: whichever of the four runs first after nmsm_init builds it.  With profiling on,
 * nmsm_last_timing reports k_recover_prepare in slot 0, k_recover_check in slot 1 and both in NMSM_T_TOTAL. */
int nmsm_secp256k1_recover_batch(const uint8_t* sigs65, const uint8_t* msgs, const uint64_t* msg_off, uint64_t n,
                                 int flags, uint8_t* out_xy, uint8_t* out_ok);

/* Ethereum ecrecover (precompile 0x01, Yellow Paper appendix E), batched.  inputs128: n x 128 B = h (32) || v (32,
 * big-endian integer) || r || s.  v must equal 27 or 28 as a 256-bit integer (bytes 32..62 zero), rec = v - 27;
 * 1 <= r, s < n with no lowS rule (EIP-2 is a transaction rule, not the precompile's); h is the 32 raw bytes
 * (bits2int_modN without prehash); then recovery runs as in nmsm_secp256k1_recover_batch.
 * out32: n x 32 B = 12 zero bytes || the last 20 bytes of keccak256(x_be || y_be) of the recovered key; out_ok: n bytes.
 * Where the precompile returns empty output: out_ok 0 and 32 zero bytes.  Errors, the table of G and the profiling
 * slots as for nmsm_secp256k1_recover_batch. */
int nmsm_secp256k1_ecrecover_batch(const uint8_t* inputs128, uint64_t n, uint8_t* out32, uint8_t* out_ok);

/* BLS12-381 batch pairing checks (next-row f7): out_ok[j] = 1 iff prod_{i in [pair_off[j], pair_off[j+1])} e(P_i, Q_i)
 * == 1 in GT, the optimal-ate pairing of the reference (src/abstract/bls.ts, bls12-381.ts), one verdict per check.
 * g1_xy: P_i in the affine packing above (96 B: x, y); g2_xy: Q_i (192 B: x.c0, x.c1, y.c0, y.c1), each coordinate 48 B
 * little-endian; pair_off: n_checks + 1 offsets, the pair count is pair_off[n_checks].  An empty check is 1.  A pair
 * with an identity point ((0, 0)) contributes 1, its mathematical value; the reference's pairing throws on the zero
 * point instead.  Points are NOT subgroup-checked (as for the MSM ids 4 and 5; nmsm_points_torsion_free does that):
 * outside the subgroups the verdict is whatever the same formulas give.  NMSM_ERR_POINT, with nmsm_last_error_index =
 * the pair index, for a coordinate >= p or a point off its curve (every G1 point is checked before any G2 point);
 * NMSM_ERR_ARG for null pointers, offsets that do not start at 0 or decrease, and 2^31 or more pairs.  n_checks == 0
 * writes nothing.  Miller loops run in chunks of 2^16 pairs (a 38 MB workspace).  With profiling on,
 * nmsm_last_timing reports k_bls_miller in slot 0, k_bls_final in slot 1 (each summed over the chunks) and their sum
 * in NMSM_T_TOTAL. */
int nmsm_bls12_381_pairing_check_batch(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                       uint64_t n_checks, uint8_t* out_ok);

/* bn254 batch pairing checks (next-row f8): the contract of nmsm_bls12_381_pairing_check_batch on bn254 (the
 * reference's bn254.pairing / pairingBatch; Ethereum's ecPairing precompile, EIP-197; Groth16 and KZG verification).
 * out_ok[j] = 1 iff prod_{i in [pair_off[j], pair_off[j+1])} e(P_i, Q_i) == 1 in GT, the optimal-ate pairing.
 * g1_xy: P_i in the affine packing above (64 B: x, y); g2_xy: Q_i (128 B: x.c0, x.c1, y.c0, y.c1), each coordinate 32 B
 * little-endian (the NMSM_BN254_G1 / G2 packing).  An empty check is 1; a pair with an identity point ((0, 0))
 * contributes 1.  Points are NOT subgroup-checked (nmsm_points_torsion_free(NMSM_BN254_G2, ...) does that; EIP-197
 * requires it for G2).  NMSM_ERR_POINT, with nmsm_last_error_index = the pair index, for a coordinate >= p or a point
 * off its curve (every G1 point is checked before any G2 point); NMSM_ERR_ARG for null pointers, offsets that do not
 * start at 0 or decrease, and 2^31 or more checks or pairs.  n_checks == 0 writes nothing.  Miller loops run in chunks
 * of 2^16 pairs (a 25 MB workspace).  With profiling on, nmsm_last_timing reports k_bn254_miller in slot 0,
 * k_bn254_final in slot 1 (each summed over the chunks) and their sum in NMSM_T_TOTAL. */
int nmsm_bn254_pairing_check_batch(const uint8_t* g1_xy, const uint8_t* g2_xy, const uint64_t* pair_off,
                                   uint64_t n_checks, uint8_t* out_ok);

/* BLS12-381 batch signature verification (next-row f7): out_ok[i] = bls12_381.verify(sig_i, H_i, pk_i) for long
 * signatures (public key in G1, signature in G2), one independent verdict per signature.
 * sigs96: n x 96 B Zcash-flag compressed G2 signatures; pks48: n x 48 B Zcash-flag compressed G1 keys; msg_pts: n x
 * 192 B messages ALREADY HASHED to G2, in the affine G2 packing (nmsm_bls12_381_hash_to_g2_batch computes them;
 * nmsm_bls12_381_verify_msg_batch takes the message bytes instead).
 * out_ok[i] = 1 iff pk decodes, is not the identity and is in G1, sig decodes, is not the identity and is in G2, H is
 * not the identity, and e(pk, H) e(-G1, sig) == 1.  Everything about a signature's or key's content is a 0 verdict,
 * never an error.  H comes from the caller's hash-to-curve and is in G2 by construction, so it is only checked for
 * range and curve: NMSM_ERR_POINT with nmsm_last_error_index = i for an H with a coordinate >= p or off the twist.
 * NMSM_ERR_ARG for null pointers and n >= 2^30.  n == 0 writes nothing.  With profiling on, nmsm_last_timing reports
 * k_bls_verify_prepare in slot 0, k_bls_miller in slot 1, k_bls_final in slot 2 and their sum in NMSM_T_TOTAL. */
int nmsm_bls12_381_verify_batch(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msg_pts, uint64_t n,
                                uint8_t* out_ok);

/* BLS12-381 hash to G2 (next-row f10): out_xy[i] = hash_to_curve(msg_i) on BLS12-381 G2, suite
 * BLS12381G2_XMD:SHA-256_SSWU_RO_ (RFC 9380 §8.8.2; noble's bls12_381.G2.hashToCurve(msg, { DST })): expand_message_xmd
 * with SHA-256, hash_to_field to two Fp2 elements, the simplified SWU map on the 3-isogenous curve and the isogeny, the
 * sum of the two points, and cofactor clearing by h_eff.  message i = msgs[msg_off[i], msg_off[i+1]), any length
 * including 0; dst: the domain separation tag, dst_len >= 1 bytes (noble's default for long signatures is
 * "BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_", Ethereum's "..._POP_"); a tag over 255 bytes is replaced by
 * SHA-256("H2C-OVERSIZE-DST-" || DST) (RFC 9380 §5.3.3).  out_xy: n x 192 B in the affine G2 packing (x.c0, x.c1,
 * y.c0, y.c1, 48 B little-endian each); the points are in G2; the identity, which only arises with negligible
 * probability, is written as (0, 0).  NMSM_ERR_ARG for null pointers, an empty tag, offsets that do not start at 0 or
 * decrease, and n >= 2^30.  n == 0 writes nothing.  With profiling on, nmsm_last_timing reports k_bls_hash_to_g2 in
 * slot 0 and in NMSM_T_TOTAL. */
int nmsm_bls12_381_hash_to_g2_batch(const uint8_t* msgs, const uint64_t* msg_off, uint64_t n, const uint8_t* dst,
                                    uint64_t dst_len, uint8_t* out_xy);

/* nmsm_bls12_381_verify_batch with message i = msgs[msg_off[i], msg_off[i+1]) hashed to G2 on the GPU under dst, as
 * nmsm_bls12_381_hash_to_g2_batch hashes it: out_ok[i] = bls12_381.verify(sig_i, G2.hashToCurve(msg_i, { DST }), pk_i).
 * Every verdict rule of nmsm_bls12_381_verify_batch holds; the message points are in G2 by construction, so there is
 * no message-point error.  NMSM_ERR_ARG as for nmsm_bls12_381_hash_to_g2_batch.  With profiling on, nmsm_last_timing
 * reports k_bls_hash_to_g2 in slot 0, k_bls_verify_prepare in slot 1, k_bls_miller in slot 2, k_bls_final in slot 3
 * and their sum in NMSM_T_TOTAL. */
int nmsm_bls12_381_verify_msg_batch(const uint8_t* sigs96, const uint8_t* pks48, const uint8_t* msgs,
                                    const uint64_t* msg_off, uint64_t n, const uint8_t* dst, uint64_t dst_len,
                                    uint8_t* out_ok);

/* Batched wire-format decoding on the GPU (next-row f2): encodings -> canonical affine points in the packing
 * above, ready for nmsm_msm.  secp256k1: 33-byte SEC1 compressed (weierstrass.ts:565-588); BLS12-381 G1: 48-byte
 * Zcash-flag compressed (bls12-381.ts:377-468); BLS12-381 G2: 96-byte Zcash-flag compressed, x = c1 || c0
 * (bls12-381.ts:354-367,488-491; Fp2 square root tower.ts:476-498); ed25519: 32-byte RFC 8032, strict like the
 * reference's fromBytes default (edwards.ts:405-436; ZIP-215 acceptance: nmsm_points_decode_ex).  out_status[i]: 0 = invalid encoding, 1 = point, 2 = point at infinity.  Mirrors
 * the reference's decode step only; the subgroup check its fromBytes adds is nmsm_points_torsion_free.  Other
 * curves: NMSM_ERR_ARG. */
int nmsm_points_decode(int curve, const uint8_t* enc, uint64_t n, uint8_t* out_xy, uint8_t* out_status);
/* Same with flags.  nmsm_points_decode == flags 0 == the reference's defaults: for ed25519 that is the strict RFC 8032
 * decoding of `Point.fromBytes(bytes, zip215 = false)` (/root/reference/src/abstract/edwards.ts:405-436: y >= p
 * rejected, x = 0 with the sign bit set rejected); NMSM_DECODE_ZIP215 selects the ZIP-215 acceptance rules that
 * ed25519.verify (and nmsm_ed25519_verify_batch) decode with.  Invalid encodings return status 0 and zeroed bytes. */
#define NMSM_DECODE_ZIP215 1
int nmsm_points_decode_ex(int curve, const uint8_t* enc, uint64_t n, int flags, uint8_t* out_xy, uint8_t* out_status);

/* out_ok[i] = 1 iff pts[i] has in-range coordinates and satisfies the curve equation: the `isValidXY` half of the
 * reference's assertValidity (/root/reference/src/abstract/weierstrass.ts:617-624,766; edwards.ts:461-480) in batch
 * form; together with nmsm_points_torsion_free it is what Point.assertValidity checks.  The affine identity encoding
 * counts as on the curve.  pippenger itself never validates ("Does NOT validate", weierstrass.ts:695,711). */
int nmsm_points_on_curve(int curve, const uint8_t* pts, uint64_t n, uint8_t* out_ok);

/* Tuning / introspection ------------------------------------------------------------------- */
/* Force the window size c (0 = automatic cost model).  Returns the previous value. */
int nmsm_set_window_bits(int c);
/* Force the number of window groups an MSM is pipelined over (1..8; 0 = automatic: one group for small inputs, one
 * group per window (at most 8) once the accumulation is long enough to hide the bucket reduction and the Horner
 * doublings of the finished groups underneath it).  Results never depend on it.  Returns the previous value. */
int nmsm_set_window_groups(int groups);

/* Plan + device times (ms, CUDA events on the library's streams) of the last MSM call.  `ms` receives
 * NMSM_TIMING_SLOTS floats, see the NMSM_T_* indices.  NMSM_T_TOTAL (first kernel to the inversion, the whole MSM
 * on the device) is always measured; the per-kernel entries only while profiling is on, which also forces the
 * linear one-group pipeline (per-kernel times of overlapping launches would not add up). */
enum {
  NMSM_T_PREPARE = 0, NMSM_T_COUNT, NMSM_T_SCAN, NMSM_T_SCATTER, NMSM_T_ACCUMULATE, NMSM_T_STITCH,
  NMSM_T_REDUCE1, NMSM_T_REDUCE23, NMSM_T_FINAL, NMSM_T_TOTAL, NMSM_TIMING_SLOTS
};
typedef struct {
  int c, windows, buckets_per_window, entries_per_thread, reduce_chunk;
  uint64_t sorted_entries;      /* non-zero digits = mixed additions issued + bucket starts       */
  uint64_t modmul_equiv;        /* field multiplications executed by the plan (SURVEY §8d formula) */
  int launches;                 /* kernels launched by the call                                   */
  int window_groups;            /* window groups the call was pipelined over (1 = linear pipeline) */
  uint64_t bucket_starts;       /* of sorted_entries: copies into an empty accumulator (no multiplications); counted
                                   while profiling is on, else 0 */
  uint64_t bucket_pairs;        /* same-bucket neighbour pairs k_accumulate adds in affine first (3 + 3 multiplications
                                   each, then ONE mixed addition for the pair); counted while profiling is on, else 0.
                                   executed multiplications of k_accumulate =
                                   10 * (sorted_entries - bucket_starts) - 4 * bucket_pairs + 12 * accumulate_threads */
  uint64_t accumulate_threads;  /* threads with work in k_accumulate (each pays 12 multiplications for the warp-shared inversion) */
} nmsm_plan_info;
int nmsm_set_profiling(int enabled);
int nmsm_last_timing(float* ms, nmsm_plan_info* info);

/* Register-resident Montgomery-multiplication throughput (the roofline denominator, SURVEY §8d).
 * field: 0 = 256-bit (bn254 Fp, 8 limbs), 1 = 381-bit (BLS12-381 Fp, 12 limbs).
 * Returns modmul/s measured with CUDA events; <= 0 on error. */
double nmsm_bench_modmul(int field, int blocks_per_sm, int threads, int iters, int ilp);

/* Pinned host memory helpers for the end-to-end path. */
void* nmsm_host_alloc(size_t bytes);
void nmsm_host_free(void* p);

#ifdef __cplusplus
}
#endif
#endif /* NMSM_H */
