"""ctypes binding of libnmsm.so (C ABI: include/nmsm.h).

The library is built in-tree by `make -C noble-curves_b200` (see __graft_entry__.build()).  There is
no CPU fallback: if the shared object is missing, or no CUDA device can be initialised, every
operation raises — loudly — instead of computing anything on the host.
"""
from __future__ import annotations

import ctypes
import os
import threading

# The library overlaps kernels on several CUDA streams per MSM; give the device enough hardware work queues that they
# do not alias (takes effect if the CUDA context has not been created yet; never overrides an explicit setting).
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
# The sharded MSM moves one 6 MB bucket array per window and peer with ncclSend/ncclRecv; NCCL's default of 1-2 channels
# (CTAs) per peer caps such a transfer far below the NVLink rate.  More point-to-point channels
# = more CTAs copying in parallel.  NCCL caches these parameters at its first communicator, so they must be in the
# environment before torch.distributed / the library create one; explicit user settings win.
os.environ.setdefault("NCCL_MIN_P2P_NCHANNELS", "16")
os.environ.setdefault("NCCL_MAX_P2P_NCHANNELS", "32")
os.environ.setdefault("NCCL_NCHANNELS_PER_NET_PEER", "16")

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NMSM_LIB") or os.path.join(_HERE, "libnmsm.so")  # NMSM_LIB: build-variant experiments

NMSM_OK = 0
ERR_ARG, ERR_SCALAR, ERR_POINT, ERR_LENGTH, ERR_CUDA = -1, -2, -3, -4, -5

TIMING_SLOTS = 10
TIMING_NAMES = ["prepare", "count", "scan", "scatter", "accumulate", "stitch", "reduce1", "reduce23", "final", "total"]

# every symbol include/nmsm.h declares (tests check that the library exports all of them)
EXPORTS = [
    "nmsm_init", "nmsm_shutdown", "nmsm_last_error", "nmsm_last_error_index", "nmsm_point_bytes",
    "nmsm_acc_bytes", "nmsm_msm", "nmsm_msm_device", "nmsm_msm_partial_device", "nmsm_fold_partials_device",
    "nmsm_mul_batch", "nmsm_set_window_bits", "nmsm_set_profiling", "nmsm_last_timing", "nmsm_bench_modmul",
    "nmsm_host_alloc", "nmsm_host_free", "nmsm_points_upload", "nmsm_points_free", "nmsm_msm_points", "nmsm_points_precompute", "nmsm_msm_points_submit", "nmsm_point_table_create", "nmsm_point_table_free",
    "nmsm_point_table_mul_batch", "nmsm_ntt", "nmsm_ntt_device", "nmsm_points_torsion_free",
    "nmsm_ed25519_verify_batch", "nmsm_ed25519_verify_each", "nmsm_msm_submit", "nmsm_msm_collect", "nmsm_points_decode", "nmsm_msm_submit_partial",
    "nmsm_points_decode_ex", "nmsm_points_on_curve", "nmsm_set_window_groups", "nmsm_accs_normalize",
    "nmsm_dist_unique_id", "nmsm_dist_init", "nmsm_dist_info", "nmsm_dist_exchange_mode", "nmsm_msm_sharded", "nmsm_msm_sharded_submit",
    "nmsm_secp256k1_verify_batch", "nmsm_p256_verify_batch", "nmsm_p384_verify_batch", "nmsm_secp256k1_schnorr_verify_batch",
    "nmsm_secp256k1_recover_batch", "nmsm_secp256k1_ecrecover_batch",
    "nmsm_bls12_381_pairing_check_batch", "nmsm_bls12_381_verify_batch", "nmsm_bn254_pairing_check_batch",
    "nmsm_bls12_381_hash_to_g2_batch", "nmsm_bls12_381_verify_msg_batch", "nmsm_bls12_381_aggregate_verify_batch",
    "nmsm_bls12_381_hash_to_g1_batch", "nmsm_bls12_381_short_verify_batch", "nmsm_bls12_381_short_verify_msg_batch",
    "nmsm_bls12_381_kzg_verify_proof_batch", "nmsm_bls12_381_kzg_verify_blob_batch",
    "nmsm_bls12_381_kzg_setup_create", "nmsm_bls12_381_kzg_setup_free", "nmsm_bls12_381_kzg_commit_batch",
    "nmsm_bls12_381_kzg_compute_proof_batch", "nmsm_bls12_381_kzg_compute_blob_proof_batch",
]


class PlanInfo(ctypes.Structure):
    _fields_ = [
        ("c", ctypes.c_int),
        ("windows", ctypes.c_int),
        ("buckets_per_window", ctypes.c_int),
        ("entries_per_thread", ctypes.c_int),
        ("reduce_chunk", ctypes.c_int),
        ("sorted_entries", ctypes.c_uint64),
        ("modmul_equiv", ctypes.c_uint64),
        ("launches", ctypes.c_int),
        ("window_groups", ctypes.c_int),
        ("bucket_starts", ctypes.c_uint64),
        ("bucket_pairs", ctypes.c_uint64),
        ("accumulate_threads", ctypes.c_uint64),
    ]


class NmsmError(RuntimeError):
    def __init__(self, code: int, message: str, index: int = -1):
        super().__init__(message)
        self.code = code
        self.index = index


_lib = None
_lock = threading.Lock()
_initialised_device = None


def load() -> ctypes.CDLL:
    """Load libnmsm.so and declare prototypes.  Raises if the extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `make -C noble-curves_b200 -j8` "
                "(there is no CPU fallback for the MSM / scalar-mult path)"
            )
        lib = ctypes.CDLL(LIB_PATH)
        u8p = ctypes.c_void_p
        lib.nmsm_init.argtypes = [ctypes.c_int]
        lib.nmsm_init.restype = ctypes.c_int
        lib.nmsm_shutdown.argtypes = []
        lib.nmsm_shutdown.restype = None
        lib.nmsm_last_error.argtypes = []
        lib.nmsm_last_error.restype = ctypes.c_char_p
        lib.nmsm_last_error_index.argtypes = []
        lib.nmsm_last_error_index.restype = ctypes.c_longlong
        lib.nmsm_point_bytes.argtypes = [ctypes.c_int]
        lib.nmsm_point_bytes.restype = ctypes.c_int
        lib.nmsm_acc_bytes.argtypes = [ctypes.c_int]
        lib.nmsm_acc_bytes.restype = ctypes.c_int
        lib.nmsm_msm.argtypes = [ctypes.c_int, u8p, u8p, ctypes.c_uint64, u8p, ctypes.POINTER(ctypes.c_int)]
        lib.nmsm_msm.restype = ctypes.c_int
        lib.nmsm_msm_device.argtypes = [ctypes.c_int, u8p, u8p, ctypes.c_uint64, u8p, ctypes.POINTER(ctypes.c_int)]
        lib.nmsm_msm_device.restype = ctypes.c_int
        lib.nmsm_msm_partial_device.argtypes = [ctypes.c_int, u8p, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_msm_partial_device.restype = ctypes.c_int
        lib.nmsm_fold_partials_device.argtypes = [ctypes.c_int, u8p, ctypes.c_int, u8p, ctypes.POINTER(ctypes.c_int)]
        lib.nmsm_fold_partials_device.restype = ctypes.c_int
        lib.nmsm_accs_normalize.argtypes = [ctypes.c_int, u8p, ctypes.c_int, ctypes.c_uint64, u8p, u8p]
        lib.nmsm_accs_normalize.restype = ctypes.c_int
        lib.nmsm_mul_batch.argtypes = [ctypes.c_int, u8p, u8p, ctypes.c_uint64, ctypes.c_int, u8p, u8p]
        lib.nmsm_mul_batch.restype = ctypes.c_int
        lib.nmsm_set_window_bits.argtypes = [ctypes.c_int]
        lib.nmsm_set_window_bits.restype = ctypes.c_int
        lib.nmsm_dist_unique_id.argtypes = [u8p]
        lib.nmsm_dist_unique_id.restype = ctypes.c_int
        lib.nmsm_dist_init.argtypes = [ctypes.c_int, ctypes.c_int, u8p]
        lib.nmsm_dist_init.restype = ctypes.c_int
        lib.nmsm_dist_info.argtypes = [ctypes.POINTER(ctypes.c_int)] * 3
        lib.nmsm_dist_info.restype = ctypes.c_int
        lib.nmsm_dist_exchange_mode.argtypes = []
        lib.nmsm_dist_exchange_mode.restype = ctypes.c_int
        lib.nmsm_msm_sharded.argtypes = [ctypes.c_int, u8p, u8p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int,
                                         u8p, ctypes.POINTER(ctypes.c_int)]
        lib.nmsm_msm_sharded.restype = ctypes.c_int
        lib.nmsm_msm_sharded_submit.argtypes = [ctypes.c_int, u8p, u8p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64,
                                                ctypes.c_int, ctypes.c_int]
        lib.nmsm_msm_sharded_submit.restype = ctypes.c_int
        lib.nmsm_set_window_groups.argtypes = [ctypes.c_int]
        lib.nmsm_set_window_groups.restype = ctypes.c_int
        lib.nmsm_set_profiling.argtypes = [ctypes.c_int]
        lib.nmsm_set_profiling.restype = ctypes.c_int
        lib.nmsm_last_timing.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(PlanInfo)]
        lib.nmsm_last_timing.restype = ctypes.c_int
        lib.nmsm_bench_modmul.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        lib.nmsm_bench_modmul.restype = ctypes.c_double
        lib.nmsm_host_alloc.argtypes = [ctypes.c_size_t]
        lib.nmsm_host_alloc.restype = ctypes.c_void_p
        lib.nmsm_host_free.argtypes = [ctypes.c_void_p]
        lib.nmsm_host_free.restype = None
        lib.nmsm_points_upload.argtypes = [ctypes.c_int, u8p, ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64)]
        lib.nmsm_points_upload.restype = ctypes.c_int
        lib.nmsm_points_free.argtypes = [ctypes.c_uint64]
        lib.nmsm_points_free.restype = ctypes.c_int
        lib.nmsm_msm_points.argtypes = [ctypes.c_uint64, u8p, ctypes.c_uint64, u8p, ctypes.POINTER(ctypes.c_int)]
        lib.nmsm_msm_points.restype = ctypes.c_int
        lib.nmsm_points_precompute.argtypes = [ctypes.c_uint64, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                               ctypes.POINTER(ctypes.c_int)]
        lib.nmsm_points_precompute.restype = ctypes.c_int
        lib.nmsm_msm_points_submit.argtypes = [ctypes.c_uint64, u8p, ctypes.c_uint64, ctypes.c_int, ctypes.c_int]
        lib.nmsm_msm_points_submit.restype = ctypes.c_int
        for f in (lib.nmsm_ntt, lib.nmsm_ntt_device):
            f.argtypes = [ctypes.c_int, u8p, ctypes.c_int, ctypes.c_uint64, ctypes.c_int, ctypes.c_int, ctypes.c_int]
            f.restype = ctypes.c_int
        lib.nmsm_points_torsion_free.argtypes = [ctypes.c_int, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_points_torsion_free.restype = ctypes.c_int
        lib.nmsm_point_table_create.argtypes = [ctypes.c_int, u8p, ctypes.POINTER(ctypes.c_uint64)]
        lib.nmsm_point_table_create.restype = ctypes.c_int
        lib.nmsm_point_table_free.argtypes = [ctypes.c_uint64]
        lib.nmsm_point_table_free.restype = ctypes.c_int
        lib.nmsm_point_table_mul_batch.argtypes = [ctypes.c_uint64, u8p, ctypes.c_uint64, ctypes.c_int, u8p, u8p]
        lib.nmsm_point_table_mul_batch.restype = ctypes.c_int
        lib.nmsm_ed25519_verify_batch.argtypes = [u8p, u8p, u8p, u8p, ctypes.c_uint64, u8p, ctypes.POINTER(ctypes.c_int),
                                                  ctypes.POINTER(ctypes.c_longlong)]
        lib.nmsm_ed25519_verify_batch.restype = ctypes.c_int
        lib.nmsm_ed25519_verify_each.argtypes = [u8p, u8p, u8p, u8p, ctypes.c_uint64, ctypes.c_int, u8p]
        lib.nmsm_ed25519_verify_each.restype = ctypes.c_int
        lib.nmsm_secp256k1_verify_batch.argtypes = [u8p, u8p, u8p, u8p, u8p, ctypes.c_uint64, ctypes.c_int, u8p]
        lib.nmsm_secp256k1_verify_batch.restype = ctypes.c_int
        lib.nmsm_p256_verify_batch.argtypes = [u8p, u8p, u8p, u8p, u8p, ctypes.c_uint64, ctypes.c_int, u8p]
        lib.nmsm_p256_verify_batch.restype = ctypes.c_int
        lib.nmsm_p384_verify_batch.argtypes = [u8p, u8p, u8p, u8p, u8p, ctypes.c_uint64, ctypes.c_int, u8p]
        lib.nmsm_p384_verify_batch.restype = ctypes.c_int
        lib.nmsm_secp256k1_schnorr_verify_batch.argtypes = [u8p, u8p, u8p, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_secp256k1_schnorr_verify_batch.restype = ctypes.c_int
        lib.nmsm_secp256k1_recover_batch.argtypes = [u8p, u8p, u8p, ctypes.c_uint64, ctypes.c_int, u8p, u8p]
        lib.nmsm_secp256k1_recover_batch.restype = ctypes.c_int
        lib.nmsm_secp256k1_ecrecover_batch.argtypes = [u8p, ctypes.c_uint64, u8p, u8p]
        lib.nmsm_secp256k1_ecrecover_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_pairing_check_batch.argtypes = [u8p, u8p, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_bls12_381_pairing_check_batch.restype = ctypes.c_int
        lib.nmsm_bn254_pairing_check_batch.argtypes = [u8p, u8p, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_bn254_pairing_check_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_verify_batch.argtypes = [u8p, u8p, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_bls12_381_verify_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_hash_to_g2_batch.argtypes = [u8p, u8p, ctypes.c_uint64, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_bls12_381_hash_to_g2_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_verify_msg_batch.argtypes = [u8p, u8p, u8p, u8p, ctypes.c_uint64, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_bls12_381_verify_msg_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_hash_to_g1_batch.argtypes = [u8p, u8p, ctypes.c_uint64, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_bls12_381_hash_to_g1_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_short_verify_batch.argtypes = [u8p, u8p, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_bls12_381_short_verify_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_kzg_verify_proof_batch.argtypes = [u8p, u8p, u8p, u8p, u8p, ctypes.c_uint64, u8p, u8p]
        lib.nmsm_bls12_381_kzg_verify_proof_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_kzg_verify_blob_batch.argtypes = [u8p, u8p, u8p, ctypes.c_uint64, u8p, u8p]
        lib.nmsm_bls12_381_kzg_verify_blob_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_kzg_setup_create.argtypes = [u8p, ctypes.POINTER(ctypes.c_uint64)]
        lib.nmsm_bls12_381_kzg_setup_create.restype = ctypes.c_int
        lib.nmsm_bls12_381_kzg_setup_free.argtypes = [ctypes.c_uint64]
        lib.nmsm_bls12_381_kzg_setup_free.restype = ctypes.c_int
        lib.nmsm_bls12_381_kzg_commit_batch.argtypes = [ctypes.c_uint64, u8p, ctypes.c_uint64, u8p, u8p]
        lib.nmsm_bls12_381_kzg_commit_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_kzg_compute_proof_batch.argtypes = [ctypes.c_uint64, u8p, u8p, ctypes.c_uint64, u8p, u8p,
                                                               u8p]
        lib.nmsm_bls12_381_kzg_compute_proof_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_kzg_compute_blob_proof_batch.argtypes = [ctypes.c_uint64, u8p, u8p, ctypes.c_uint64, u8p,
                                                                    u8p]
        lib.nmsm_bls12_381_kzg_compute_blob_proof_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_short_verify_msg_batch.argtypes = [u8p, u8p, u8p, u8p, ctypes.c_uint64, u8p, ctypes.c_uint64,
                                                              u8p]
        lib.nmsm_bls12_381_short_verify_msg_batch.restype = ctypes.c_int
        lib.nmsm_bls12_381_aggregate_verify_batch.argtypes = [u8p, u8p, ctypes.c_uint64, u8p, u8p, u8p, u8p, u8p,
                                                              ctypes.c_uint64, u8p]
        lib.nmsm_bls12_381_aggregate_verify_batch.restype = ctypes.c_int
        lib.nmsm_msm_submit.argtypes = [ctypes.c_int, u8p, u8p, ctypes.c_uint64, ctypes.c_int, ctypes.c_int]
        lib.nmsm_msm_submit.restype = ctypes.c_int
        lib.nmsm_msm_collect.argtypes = [ctypes.c_int, u8p, ctypes.POINTER(ctypes.c_int)]
        lib.nmsm_msm_collect.restype = ctypes.c_int
        lib.nmsm_points_decode.argtypes = [ctypes.c_int, u8p, ctypes.c_uint64, u8p, u8p]
        lib.nmsm_points_decode.restype = ctypes.c_int
        lib.nmsm_points_decode_ex.argtypes = [ctypes.c_int, u8p, ctypes.c_uint64, ctypes.c_int, u8p, u8p]
        lib.nmsm_points_decode_ex.restype = ctypes.c_int
        lib.nmsm_points_on_curve.argtypes = [ctypes.c_int, u8p, ctypes.c_uint64, u8p]
        lib.nmsm_points_on_curve.restype = ctypes.c_int
        lib.nmsm_msm_submit_partial.argtypes = [ctypes.c_int, u8p, u8p, ctypes.c_uint64, u8p, ctypes.c_int]
        lib.nmsm_msm_submit_partial.restype = ctypes.c_int
        _lib = lib
        return lib


def check(code: int) -> None:
    if code == NMSM_OK:
        return
    lib = load()
    msg = (lib.nmsm_last_error() or b"").decode()
    raise NmsmError(code, msg, int(lib.nmsm_last_error_index()))


def init(device: int | None = None) -> int:
    """Bind the process to one GPU (default: LOCAL_RANK or 0).  Raises NmsmError without a device."""
    global _initialised_device
    lib = load()
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    if _initialised_device == device:
        return device
    check(lib.nmsm_init(device))
    _initialised_device = device
    return device


def ensure_init() -> None:
    if _initialised_device is None:
        init()
