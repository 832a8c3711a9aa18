#!/usr/bin/env python3
"""BLS12-381 pairing checks and BLS signature verification on one H100 (nmsm_bls12_381_pairing_check_batch,
nmsm_bls12_381_verify_batch).  Not a BASELINE.json config.

    python tests/bench_bls.py

Rows (one JSON line each):
  bls-card          the card's name / power limit / max SM clock
  bls-verify-12/16  2^12 / 2^16 signatures (16 unique from the oracle signer, signed before any timed window, tiled).
                    Wall time best of K through the C ABI on packed arrays (H2D included), the three kernels from the
                    profiling slots, 381-bit modmul-equivalents per signature (VERIFY_MODMUL below) against
                    nmsm_bench_modmul(1, ...) of the same run
  bls-check-14      2^14 pairing checks of 4 pairs each (8 unique checks built by bilinearity, tiled)
  bls-card-after    the card read again after the timed rows
There is no host pairing library to compare with, and the Python oracle is not a baseline: no CPU speed-up is given.
The script lives under tests/ because it uses the oracle and tests/bls_cases.py; pytest does not collect it.
"""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_ecdsa as BE  # noqa: E402  (sets up the import paths, nmsm, card_info and time_best)

nmsm = BE.nmsm
import bls_cases as C  # noqa: E402

# 381-bit Montgomery multiplications (1S = 1M; an Fp2 product = 3M, an Fp2 square = 2M, Fp2 x Fp = 2M) executed per
# unit, read off csrc/fp12.cuh and csrc/pairing.cuh.  Additions, the Fp inversions (one per Fp12 inversion, two per G2
# decode square root) and the torsion checks' window tables are not counted.
FP6_MUL, FP12_MUL, FP12_SQR, MUL_014, CYC_SQR = 18, 54, 36, 39, 18
DBL_STEP, ADD_STEP = 6 * 2 + 3 * 3 + 2 * 2, 11 * 3 + 2 * 2 + 2 * 2
MILLER = 63 * DBL_STEP + 68 * MUL_014 + 62 * FP12_SQR + 5 * ADD_STEP
EXP_X = 63 * CYC_SQR + 5 * FP12_MUL
FROB = 11 * 3
FINAL_EXP = (2 * (2 * 3 + 3 * 2) + 9 * 3 + 2 * FP6_MUL) + 2 * FP12_MUL + FROB + 5 * EXP_X + 8 * FP12_MUL + CYC_SQR + 3 * FROB
SQRT_FP = 381 + 60  # (p + 1) / 4 by square-and-multiply
SCALAR_MUL = 255 * 8 + 64 * 12  # n P, 4-bit signed windows, XYZZ doubling 8M / addition 12M
VERIFY_MODMUL = {
    "pk decode (one Fp square root)": SQRT_FP,
    "sig decode (three Fp square roots, Fp2 checks)": 3 * SQRT_FP + 20,
    "pk in G1 (n pk over Fp)": SCALAR_MUL,
    "sig in G2 (n sig over Fp2)": 3 * SCALAR_MUL,
    "two Miller loops": 2 * MILLER,
    "product of two Miller values": 2 * FP12_MUL,
    "final exponentiation": FINAL_EXP,
}
CHECK4_MODMUL = 4 * MILLER + 4 * FP12_MUL + FINAL_EXP


def _peak_381():
    return max(nmsm.bench_modmul(1, bps, thr, 3000, ilp) for (bps, thr, ilp) in ((4, 128, 1), (8, 128, 1), (8, 128, 2)))


def _kernels(run, reps, names):
    nmsm.set_profiling(True)
    best = [float("inf")] * len(names)
    for _ in range(reps):
        run()
        ms = list(nmsm.last_timing()[0].values())
        best = [min(b, m) for b, m in zip(best, ms)]
    nmsm.set_profiling(False)
    return dict(zip(names, best))


def verify_config(tag, logn, items, reps=5):
    n = 1 << logn
    tiled = (items * (n // len(items) + 1))[:n]
    sigs = b"".join(i[0] for i in tiled)
    pks = b"".join(i[2] for i in tiled)
    hs = b"".join(C.g2_bytes(i[1]) for i in tiled)
    res = {}

    def run():
        res["ok"] = nmsm.bls_verify_batch_packed(sigs, pks, hs, n)

    run()
    best = BE.time_best(run, reps)
    kern = _kernels(run, reps, ["k_bls_verify_prepare", "k_bls_miller", "k_bls_final"])
    per = sum(VERIFY_MODMUL.values())
    kern_s = sum(kern.values()) * 1e-3
    peak = _peak_381()
    return {"config": tag, "what": "BLS12-381 verify (pk in G1, sig in G2, H(m) given as a G2 point), 2^%d signatures "
                                   "(%d unique, tiled)" % (logn, len(items)), "n": n,
            "gpu_ms_through_c_abi": best * 1e3, "signatures_per_s": n / best, "kernels_ms": kern,
            "modmul_per_signature": per, "modmul_formula": VERIFY_MODMUL,
            "roofline": {"achieved_gmodmul_s": per * n / kern_s / 1e9, "peak_gmodmul_s": peak / 1e9,
                         "frac": per * n / kern_s / peak, "peak_source": "nmsm_bench_modmul(field=381-bit), same run"},
            "check": "all accepted" if res["ok"] == b"\x01" * n else "MISMATCH"}


def check_config(tag, logn, pool, reps=5):
    n = 1 << logn
    checks = (pool * (n // len(pool) + 1))[:n]
    g1, g2, off = C.pack_checks(checks)
    res = {}

    def run():
        res["ok"] = nmsm.pairing_check_batch_packed(g1, g2, off, n)

    run()
    best = BE.time_best(run, reps)
    kern = _kernels(run, reps, ["k_bls_miller", "k_bls_final"])
    kern_s = sum(kern.values()) * 1e-3
    peak = _peak_381()
    return {"config": tag, "what": "BLS12-381 pairing checks, 4 pairs each, 2^%d checks (%d unique, tiled)"
                                   % (logn, len(pool)), "n": n,
            "gpu_ms_through_c_abi": best * 1e3, "checks_per_s": n / best, "kernels_ms": kern,
            "modmul_per_check": CHECK4_MODMUL,
            "roofline": {"achieved_gmodmul_s": CHECK4_MODMUL * n / kern_s / 1e9, "peak_gmodmul_s": peak / 1e9,
                         "frac": CHECK4_MODMUL * n / kern_s / peak,
                         "peak_source": "nmsm_bench_modmul(field=381-bit), same run"},
            "check": "all true" if res["ok"] == b"\x01" * n else "MISMATCH"}


def rows():
    rnd = random.Random(30)
    items = [C.keypair_item(rnd) for _ in range(16)]  # signed before any timed window
    pool = [C.true_check(rnd, 4) for _ in range(8)]
    yield {"config": "bls-card", "card": BE.card_info()}
    yield verify_config("bls-verify-12", 12, items)
    yield verify_config("bls-verify-16", 16, items)
    yield check_config("bls-check-14", 14, pool)
    yield {"config": "bls-card-after", "card": BE.card_info()}


def main():
    nmsm.init(0)
    for row in rows():
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
