#!/usr/bin/env python3
"""bn254 pairing checks on one H100 (nmsm_bn254_pairing_check_batch).  Not a BASELINE.json config.

    python tests/bench_bn254_pairing.py

Rows (one JSON line each):
  bn254-card          the card's name / power limit / max SM clock
  bn254-check2-16     2^16 checks of 2 pairs (the KZG opening shape; 8 unique checks built by bilinearity, tiled)
  bn254-check4-14/16  2^14 / 2^16 checks of 4 pairs (the Groth16 shape e(A, B) e(-alpha, beta) e(-L, gamma)
                      e(-C, delta); 8 unique, tiled)
  bls-check-14        tests/bench_bls.py's row (2^14 BLS12-381 checks of 4 pairs) in the same process, for a same-card
                      comparison
  bn254-card-after    the card read again after the timed rows
Each row: wall time best of K through the C ABI on packed arrays (H2D included), k_bn254_miller / k_bn254_final from
the profiling slots, 256-bit modmul-equivalents per check (the formula below) against nmsm_bench_modmul(0, ...) of the
same run.  There is no host pairing library to compare with, and the Python oracle is not a baseline.
The script lives under tests/ because it uses the oracle and tests/bn254_pairing_cases.py; pytest does not collect it.
"""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_bls as BB  # noqa: E402  (sets up the import paths, nmsm and the BLS12-381 row)
import bench_ecdsa as BE  # noqa: E402  (card_info and time_best)

nmsm = BE.nmsm
import bn254_pairing_cases as C  # noqa: E402

# 256-bit Montgomery multiplications (1S = 1M; an Fp2 product = 3M, an Fp2 square = 2M, Fp2 x Fp = 2M) executed per
# unit, read off csrc/fp12.cuh and csrc/pairing_bn254.cuh.  Additions and the one Fp inversion per Fp12 inversion are
# not counted.
FP6_MUL, FP12_MUL, FP12_SQR, MUL_034, CYC_SQR = 18, 54, 36, 39, 18
FP12_INV = 2 * (2 * 3 + 3 * 2) + (9 * 3 + 3 * 2 + 4) + 2 * FP6_MUL  # two Fp6 squares, the Fp6 inverse, two Fp6 products
FROB = 7 * 3
DBL_STEP, ADD_STEP = 6 * 2 + 4 * 3 + 2 * 2, 11 * 3 + 2 * 2 + 2 * 2
# 65 doublings and 21 NAF additions, then the pi(Q) and -pi^2(Q) steps (their twist constants: 2 Fp2 and 1 Fp2 x Fp)
MILLER = 65 * DBL_STEP + 23 * ADD_STEP + 88 * MUL_034 + 64 * FP12_SQR + 2 * 3 + 2
EXP_U = 62 * CYC_SQR + 27 * FP12_MUL  # u = 0x44e992b44a6909f1: 63 bits, 28 ones
FINAL_EXP = FP12_INV + 2 * FP12_MUL + FROB + 3 * EXP_U + 3 * CYC_SQR + 9 * FP12_MUL + 3 * FROB


def check_modmul(k):
    """k Miller loops, the product of their k values (first one multiplied into 1) and one final exponentiation"""
    return k * MILLER + k * FP12_MUL + FINAL_EXP


def _peak_256():
    return max(nmsm.bench_modmul(0, bps, thr, 3000, ilp) for (bps, thr, ilp) in ((4, 128, 1), (8, 128, 1), (8, 128, 2)))


def check_config(tag, logn, k, pool, reps=5):
    n = 1 << logn
    checks = (pool * (n // len(pool) + 1))[:n]
    g1, g2, off = C.pack_checks(checks)
    res = {}

    def run():
        res["ok"] = nmsm.bn254_pairing_check_batch_packed(g1, g2, off, n)

    run()
    best = BE.time_best(run, reps)
    kern = BB._kernels(run, reps, ["k_bn254_miller", "k_bn254_final"])
    kern_s = sum(kern.values()) * 1e-3
    per = check_modmul(k)
    peak = _peak_256()
    return {"config": tag, "what": "bn254 pairing checks, %d pairs each, 2^%d checks (%d unique, tiled)"
                                   % (k, logn, len(pool)), "n": n, "pairs": n * k,
            "gpu_ms_through_c_abi": best * 1e3, "checks_per_s": n / best, "kernels_ms": kern,
            "modmul_per_check": per,
            "modmul_formula": {"miller": MILLER, "fp12_mul": FP12_MUL, "final_exp": FINAL_EXP},
            "roofline": {"achieved_gmodmul_s": per * n / kern_s / 1e9, "peak_gmodmul_s": peak / 1e9,
                         "frac": per * n / kern_s / peak, "peak_source": "nmsm_bench_modmul(field=256-bit), same run"},
            "check": "all true" if res["ok"] == b"\x01" * n else "MISMATCH"}


def rows():
    rnd = random.Random(31)
    pool2 = [C.true_check(rnd, 2) for _ in range(8)]
    pool4 = [C.groth16_check(rnd) for _ in range(8)]
    bls_pool = [BB.C.true_check(rnd, 4) for _ in range(8)]
    yield {"config": "bn254-card", "card": BE.card_info()}
    yield check_config("bn254-check2-16", 16, 2, pool2)
    yield check_config("bn254-check4-14", 14, 4, pool4)
    yield check_config("bn254-check4-16", 16, 4, pool4)
    yield BB.check_config("bls-check-14", 14, bls_pool)
    yield {"config": "bn254-card-after", "card": BE.card_info()}


def main():
    nmsm.init(0)
    for row in rows():
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
