#!/usr/bin/env python3
"""P-384 ECDSA batch verification on one H100 (nmsm_p384_verify_batch), next to P-256 ECDSA in the same process.
Not a BASELINE.json config.

    python tests/bench_p384.py

Rows (one JSON line each):
  p384-setup    the card's name / power limit / max SM clock, the one-off build of the P-384 table of G (first call
                after nmsm_init minus a second call), and a single-thread OpenSSL P-384 verify rate on the host (labelled)
  p384-16/20    2^16 / 2^20 signatures: 48-byte messages, prehash on (SHA-384), lowS off (noble's p384 defaults),
                compressed keys, 4096 unique OpenSSL-signed signatures tiled.  Wall time best of K through the C ABI on
                packed arrays (H2D included), k_p384_ecdsa_prepare / k_p384_ecdsa_check from CUDA events,
                modmul-equivalents per signature (P384_MODMUL below) against nmsm_bench_modmul(1, ...) of the same run,
                the 381-bit 12-limb field (BLS12-381 Fp): the closest peak the library measures to P-384's 384-bit one
  p256-20       P-256 ECDSA at 2^20 in the same process (tests/bench_p256.py's configuration), for the ratio
  p384-card-after  the card read again after the timed rows
The script lives under tests/ because it uses the oracle and tests/p384_cases.py; pytest does not collect it.
"""
import json
import os
import struct
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "noble-curves_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import nmsm  # noqa: E402
import bench_ecdsa as BE  # noqa: E402
import bench_p256 as B256  # noqa: E402
import p384_cases as C  # noqa: E402
from oracle import p384_ref as PR  # noqa: E402

# Field multiplications (1S = 1M) of 384-bit numbers one signature costs on the GPU, from the kernels' formulas
# (ec.cuh SwXyzz with a = -3: mixed addition 10, addition 14, doubling 9).  SHA-384 is not counted.
P384_MODMUL = {
    "u2*Q (no GLV, 4-bit signed windows over 385 bits)": 9 + 6 * 10 + 96 * 4 * 9 + 97 * 14 * 15 // 16,
    "u1*G (25 table mixed additions)": 25 * 10,
    "R = u1*G + u2*Q, x comparison": 14 + 4,
    # fp_sqrt_3mod4 is square-and-multiply over (p + 1) / 4, 382 bits with 288 one bits
    "compressed key: sqrt (381 squarings + 288 multiplications) + 3 for x^3 - 3x + b + 2 to Montgomery": 381 + 288 + 3 + 2,
    "s^-1 share of the warp inversion + u1, u2 mod n": 12 + 6,
}


def p384_config(tag, logn, unique, reps=5):
    items = C.openssl_sign(unique, seed=logn, compressed_ratio=1.0, prehash=True, msg_len=48)
    n = 1 << logn
    tiled = (items * (n // unique + 1))[:n]
    sigs = b"".join(i[0] for i in tiled)
    msgs = b"".join(i[1] for i in tiled)
    pks = b"".join(i[2] for i in tiled)
    msg_off = struct.pack("<%dQ" % (n + 1), *range(0, 48 * n + 1, 48))
    pk_off = struct.pack("<%dQ" % (n + 1), *range(0, 49 * n + 1, 49))
    res = {}

    def run():
        res["ok"] = nmsm.p384_ecdsa_verify_batch_packed(sigs, pks, pk_off, msgs, msg_off, n)

    run()
    best = BE.time_best(run, reps)
    nmsm.set_profiling(True)
    k_prep, k_check = [], []
    for _ in range(reps):
        run()
        ms = list(nmsm.last_timing()[0].values())  # slot 0: k_p384_ecdsa_prepare, slot 1: k_p384_ecdsa_check
        k_prep.append(ms[0])
        k_check.append(ms[1])
    nmsm.set_profiling(False)
    ok = res["ok"] == b"\x01" * n and all(PR.p384_ecdsa_verify(*items[i]) for i in range(4))
    per_sig = sum(P384_MODMUL.values())
    kern_s = (min(k_prep) + min(k_check)) * 1e-3
    peak_mm = max(nmsm.bench_modmul(1, bps, thr, 3000, ilp) for (bps, thr, ilp) in ((4, 128, 1), (8, 128, 1), (8, 128, 2)))
    return {"config": tag, "what": "P-384 ECDSA verify, 2^%d signatures (%d unique, tiled), prehash SHA-384, no lowS, "
                                   "compressed keys, 48-byte messages" % (logn, unique), "n": n,
            "gpu_ms_through_c_abi": best * 1e3, "signatures_per_s": n / best,
            "kernels_ms": {"k_p384_ecdsa_prepare": min(k_prep), "k_p384_ecdsa_check": min(k_check)},
            "modmul_per_signature": per_sig,
            "roofline": {"achieved_gmodmul_s": per_sig * n / kern_s / 1e9, "peak_gmodmul_s": peak_mm / 1e9,
                         "frac": per_sig * n / kern_s / peak_mm,
                         "peak_source": "nmsm_bench_modmul(field=381-bit, 12 limbs), same run; P-384 products are "
                                        "384-bit at the same 12 limbs"},
            "check": "all accepted, 4 oracle verifies agree" if ok else "MISMATCH"}


def rows():
    sig, msg, pk = C.edge_cases()[0][1:]
    t0 = time.perf_counter()
    assert nmsm.p384.verify(sig, msg, pk)  # first call after nmsm_init: builds the G table
    first_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    assert nmsm.p384.verify(sig, msg, pk)
    second_ms = (time.perf_counter() - t0) * 1e3
    items = C.openssl_sign(1000, seed=1, compressed_ratio=1.0)
    t0 = time.perf_counter()
    for it in items:
        C.openssl_verify(*it)
    cpu = len(items) / (time.perf_counter() - t0)
    yield {"config": "p384-setup", "card": BE.card_info(), "g_table_build_ms": first_ms - second_ms,
           "first_call_ms": first_ms, "second_call_ms": second_ms,
           "cpu_openssl_p384_verifies_per_s": cpu,
           "cpu_label": "OpenSSL via the Python cryptography package, 1 host thread, incl. key parsing per call"}
    yield p384_config("p384-16", 16, 4096)
    p20 = p384_config("p384-20", 20, 4096)
    yield p20
    r20 = B256.p256_config("p256-20", 20, 4096)
    yield r20
    yield {"config": "p384-vs-p256-20",
           "check_kernel_ratio": p20["kernels_ms"]["k_p384_ecdsa_check"] / r20["kernels_ms"]["k_p256_ecdsa_check"],
           "prepare_kernel_ratio": p20["kernels_ms"]["k_p384_ecdsa_prepare"] / r20["kernels_ms"]["k_p256_ecdsa_prepare"],
           "wall_ratio": p20["gpu_ms_through_c_abi"] / r20["gpu_ms_through_c_abi"],
           "modmul_ratio_384_vs_256_bit": p20["modmul_per_signature"] / r20["modmul_per_signature"]}
    yield {"config": "p384-card-after", "card": BE.card_info()}


def main():
    nmsm.init(0)
    for row in rows():
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
