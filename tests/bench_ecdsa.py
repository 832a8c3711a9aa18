#!/usr/bin/env python3
"""secp256k1 ECDSA batch verification on one H100 (nmsm_secp256k1_verify_batch).  Not a BASELINE.json config.

    python tests/bench_ecdsa.py

Rows (one JSON line each):
  ecdsa-setup   the card's name / power limit / max SM clock, the one-off build of the table of G (first call after
                nmsm_init minus a second call), and a single-thread OpenSSL verify rate on the host (labelled)
  ecdsa-16/20   2^16 / 2^20 signatures: 32-byte messages, prehash on, lowS on, compressed keys, 4096 unique
                OpenSSL-signed (low-S normalised) signatures tiled.  Wall time best of K through the C ABI on packed
                arrays (H2D included), k_ecdsa_prepare / k_ecdsa_check from CUDA events, modmul-equivalents per
                signature (ECDSA_MODMUL below) against nmsm_bench_modmul(0, ...) of the same run
  ecdsa-card-after  the card read again after the timed rows
The script lives under tests/ because it uses the oracle and tests/ecdsa_cases.py; pytest does not collect it.
"""
import json
import os
import struct
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "noble-curves_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import nmsm  # noqa: E402
import ecdsa_cases as E  # noqa: E402
from oracle import ecdsa_ref as ER  # noqa: E402

# Field multiplications (1S = 1M) one signature costs on the GPU, from the kernels' formulas (ec.cuh SwXyzz: mixed
# addition 10, addition 14, doubling 9).  SHA-256 is not counted.
ECDSA_MODMUL = {
    "u2*Q (GLV, 4-bit signed windows over two 129-bit halves)": 9 + 6 * 10 + 32 * 4 * 9 + 33 * 2 * 14 * 15 // 16 + 33,
    "u1*G (17 table mixed additions)": 17 * 10,
    "R = u1*G + u2*Q, x comparison": 14 + 4,
    "compressed key: sqrt (255 squarings + 11 multiplications) + 2 to Montgomery": 255 + 11 + 2 + 2,
    "s^-1 share of the warp inversion + u1, u2 mod n": 12 + 6,
}


def time_best(fn, reps):
    best = 1e9
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return best


def card_info():
    """Name, power limit and max SM clock of device 0, read in the same run as the measurement."""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": "unknown", "error": str(e)}


def ecdsa_config(tag, logn, unique, reps=5):
    items = E.openssl_sign(unique, seed=logn, compressed_ratio=1.0, prehash=True, msg_len=32)
    items = [(E.sig_for(int.from_bytes(s[:32], "big"), min(int.from_bytes(s[32:], "big"), E.N - int.from_bytes(s[32:], "big"))),
              m, pk) for s, m, pk in items]
    n = 1 << logn
    tiled = (items * (n // unique + 1))[:n]
    sigs = b"".join(i[0] for i in tiled)
    msgs = b"".join(i[1] for i in tiled)
    pks = b"".join(i[2] for i in tiled)
    msg_off = struct.pack("<%dQ" % (n + 1), *range(0, 32 * n + 1, 32))
    pk_off = struct.pack("<%dQ" % (n + 1), *range(0, 33 * n + 1, 33))
    res = {}

    def run():
        res["ok"] = nmsm.ecdsa_verify_batch_packed(sigs, pks, pk_off, msgs, msg_off, n)

    run()
    best = time_best(run, reps)
    nmsm.set_profiling(True)
    k_prep, k_check = [], []
    for _ in range(reps):
        run()
        ms = list(nmsm.last_timing()[0].values())  # slot 0: k_ecdsa_prepare, slot 1: k_ecdsa_check (include/nmsm.h)
        k_prep.append(ms[0])
        k_check.append(ms[1])
    nmsm.set_profiling(False)
    ok = res["ok"] == b"\x01" * n and all(ER.secp256k1_ecdsa_verify(*items[i]) for i in range(4))
    per_sig = sum(ECDSA_MODMUL.values())
    kern_s = (min(k_prep) + min(k_check)) * 1e-3
    peak_mm = max(nmsm.bench_modmul(0, bps, thr, 3000, ilp) for (bps, thr, ilp) in ((4, 128, 1), (8, 128, 1), (8, 128, 2)))
    return {"config": tag, "what": "secp256k1 ECDSA verify, 2^%d signatures (%d unique, tiled), prehash, lowS, "
                                   "compressed keys, 32-byte messages" % (logn, unique), "n": n,
            "gpu_ms_through_c_abi": best * 1e3, "signatures_per_s": n / best,
            "kernels_ms": {"k_ecdsa_prepare": min(k_prep), "k_ecdsa_check": min(k_check)},
            "modmul_per_signature": per_sig,
            "roofline": {"achieved_gmodmul_s": per_sig * n / kern_s / 1e9, "peak_gmodmul_s": peak_mm / 1e9,
                         "frac": per_sig * n / kern_s / peak_mm, "peak_source": "nmsm_bench_modmul(field=256-bit), same run"},
            "check": "all accepted, 4 oracle verifies agree" if ok else "MISMATCH"}


def rows():
    sig, msg, pk = E.edge_cases()[0][1:]
    t0 = time.perf_counter()
    assert nmsm.secp256k1.verify(sig, msg, pk)  # first call after nmsm_init: builds the G table
    first_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    assert nmsm.secp256k1.verify(sig, msg, pk)
    second_ms = (time.perf_counter() - t0) * 1e3
    items = E.openssl_sign(2000, seed=1, compressed_ratio=1.0)
    t0 = time.perf_counter()
    for it in items:
        E.openssl_verify(*it, lowS=False)
    cpu = len(items) / (time.perf_counter() - t0)
    yield {"config": "ecdsa-setup", "card": card_info(), "g_table_build_ms": first_ms - second_ms,
           "first_call_ms": first_ms, "second_call_ms": second_ms,
           "cpu_openssl_verifies_per_s": cpu,
           "cpu_label": "OpenSSL via the Python cryptography package, 1 host thread, incl. key parsing per call"}
    yield ecdsa_config("ecdsa-16", 16, 4096)
    yield ecdsa_config("ecdsa-20", 20, 4096)
    yield {"config": "ecdsa-card-after", "card": card_info()}


def main():
    nmsm.init(0)
    for row in rows():
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
