#!/usr/bin/env python3
"""secp256k1 BIP340 Schnorr batch verification on one H100 (nmsm_secp256k1_schnorr_verify_batch), next to ECDSA in the
same process on the same card.  Not a BASELINE.json config.

    python tests/bench_schnorr.py

Rows (one JSON line each):
  schnorr-setup    the card's name / power limit / max SM clock, and the one-off build of the table of G by the first
                   Schnorr verify after nmsm_init (first call minus a second call)
  ecdsa-20         tests/bench_ecdsa.py's 2^20 ECDSA row, run here so both schemes are measured in one process
  schnorr-16/20    2^16 / 2^20 signatures: 32-byte messages, 4096 unique signatures from the oracle signer
                   (oracle/schnorr_ref.py, signed before any timed window) tiled.  Wall time best of K through the C ABI
                   on packed arrays (H2D included), k_schnorr_prepare / k_schnorr_check from CUDA events,
                   modmul-equivalents per signature (SCHNORR_MODMUL below) against nmsm_bench_modmul(0, ...) of the same run
  schnorr-card-after  the card read again after the timed rows
The script lives under tests/ because it uses the oracle and tests/schnorr_cases.py; pytest does not collect it.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_ecdsa as BE  # noqa: E402  (sets up the import paths, nmsm and the ECDSA rows)

nmsm = BE.nmsm
import schnorr_cases as S  # noqa: E402
from oracle import schnorr_ref as SR  # noqa: E402

# Field multiplications (1S = 1M) one signature costs on the GPU, counted as bench_ecdsa.ECDSA_MODMUL: u*P and s*G as
# u2*Q and u1*G there; no s^-1 mod n, instead one share of a warp inversion of ZZZ for the parity of y(R).  SHA-256
# (two blocks past the constant T || T midstate for a 32-byte message) is not counted.
SCHNORR_MODMUL = {
    "u*P (GLV, 4-bit signed windows over two 129-bit halves)":
        BE.ECDSA_MODMUL["u2*Q (GLV, 4-bit signed windows over two 129-bit halves)"],
    "s*G (17 table mixed additions)": 17 * 10,
    "R = s*G + u*P, x comparison X == r*ZZ": 14 + 2,
    "lift_x: sqrt (255 squarings + 11 multiplications) + 2 to Montgomery": 255 + 11 + 2 + 2,
    "ZZZ^-1 share of the warp inversion + y = Y*ZZZ^-1, canonical": 12 + 2,
}


def schnorr_config(tag, logn, items, reps=5):
    n = 1 << logn
    tiled = (items * (n // len(items) + 1))[:n]
    sigs, pks, msgs, msg_off = S.pack([i[0] for i in tiled], [i[1] for i in tiled], [i[2] for i in tiled])
    res = {}

    def run():
        res["ok"] = nmsm.schnorr_verify_batch_packed(sigs, pks, msgs, msg_off, n)

    run()
    best = BE.time_best(run, reps)
    nmsm.set_profiling(True)
    k_prep, k_check = [], []
    for _ in range(reps):
        run()
        ms = list(nmsm.last_timing()[0].values())  # slot 0: k_schnorr_prepare, slot 1: k_schnorr_check (include/nmsm.h)
        k_prep.append(ms[0])
        k_check.append(ms[1])
    nmsm.set_profiling(False)
    ok = res["ok"] == b"\x01" * n and all(SR.secp256k1_schnorr_verify(*items[i]) for i in range(4))
    per_sig = sum(SCHNORR_MODMUL.values())
    kern_s = (min(k_prep) + min(k_check)) * 1e-3
    peak_mm = max(nmsm.bench_modmul(0, bps, thr, 3000, ilp) for (bps, thr, ilp) in ((4, 128, 1), (8, 128, 1), (8, 128, 2)))
    return {"config": tag, "what": "secp256k1 BIP340 Schnorr verify, 2^%d signatures (%d unique, tiled), x-only keys, "
                                   "32-byte messages" % (logn, len(items)), "n": n,
            "gpu_ms_through_c_abi": best * 1e3, "signatures_per_s": n / best,
            "kernels_ms": {"k_schnorr_prepare": min(k_prep), "k_schnorr_check": min(k_check)},
            "modmul_per_signature": per_sig, "modmul_formula": SCHNORR_MODMUL,
            "roofline": {"achieved_gmodmul_s": per_sig * n / kern_s / 1e9, "peak_gmodmul_s": peak_mm / 1e9,
                         "frac": per_sig * n / kern_s / peak_mm, "peak_source": "nmsm_bench_modmul(field=256-bit), same run"},
            "check": "all accepted, 4 oracle verifies agree" if ok else "MISMATCH"}


def rows():
    items = S.signed_batch(4096, seed=20, msg_len=32)  # signed before any timed window
    sig, msg, pk = items[0]
    t0 = time.perf_counter()
    assert nmsm.schnorr.verify(sig, msg, pk)  # first verify after nmsm_init: builds the shared table of G
    first_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    assert nmsm.schnorr.verify(sig, msg, pk)
    second_ms = (time.perf_counter() - t0) * 1e3
    yield {"config": "schnorr-setup", "card": BE.card_info(), "g_table_build_ms": first_ms - second_ms,
           "first_call_ms": first_ms, "second_call_ms": second_ms}
    yield BE.ecdsa_config("ecdsa-20", 20, 4096)
    yield schnorr_config("schnorr-16", 16, items)
    yield schnorr_config("schnorr-20", 20, items)
    yield {"config": "schnorr-card-after", "card": BE.card_info()}


def main():
    nmsm.init(0)
    for row in rows():
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
