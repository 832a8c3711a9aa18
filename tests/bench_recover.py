#!/usr/bin/env python3
"""secp256k1 ECDSA public-key recovery and Ethereum ecrecover on one H100 (nmsm_secp256k1_recover_batch,
nmsm_secp256k1_ecrecover_batch), next to ECDSA verification in the same process on the same card.  Not a
BASELINE.json config.

    python tests/bench_recover.py

Rows (one JSON line each):
  recover-card-before  the card's name / power limit / max SM clock, and the one-off build of the table of G by the
                       first recovery after nmsm_init (first call minus a second call)
  ecdsa-20             tests/bench_ecdsa.py's 2^20 ECDSA row, run here so both are measured in one process
  recover-16/20        2^16 / 2^20 65-byte signatures rec || r || s, 32-byte messages, prehash on, 4096 unique
                       signatures from the oracle signer (tests/recover_cases.py, signed before any timed window)
                       tiled.  Wall time best of K through the C ABI on packed arrays (H2D included),
                       k_recover_prepare / k_recover_check from CUDA events, modmul-equivalents per item
                       (RECOVER_MODMUL below) against nmsm_bench_modmul(0, ...) of the same run
  ecrecover-20         2^20 precompile inputs h || v || r || s (4096 unique, tiled), measured as recover-20; Keccak-256
                       is not in the modmul count
  recover-card-after   the card read again after the timed rows
The script lives under tests/ because it uses the oracle and tests/recover_cases.py; pytest does not collect it.
"""
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_ecdsa as BE  # noqa: E402  (sets up the import paths, nmsm and the ECDSA rows)

nmsm = BE.nmsm
import ecdsa_cases as E  # noqa: E402
import recover_cases as RC  # noqa: E402
from oracle import recover_ref as RR  # noqa: E402

# Field multiplications (1S = 1M) one recovery costs on the GPU, counted as bench_ecdsa.ECDSA_MODMUL: u2*R and u1*G as
# u2*Q and u1*G there; r^-1 instead of s^-1; the square root of the key decode moves to R; no x comparison, instead one
# share of a warp inversion of ZZZ and the affine output.  SHA-256 and Keccak-256 are not counted.
RECOVER_MODMUL = {
    "u2*R (GLV, 4-bit signed windows over two 129-bit halves)":
        BE.ECDSA_MODMUL["u2*Q (GLV, 4-bit signed windows over two 129-bit halves)"],
    "u1*G (17 table mixed additions)": 17 * 10,
    "Q = u1*G + u2*R": 14,
    "lift R: sqrt (255 squarings + 11 multiplications) + 2 to Montgomery": 255 + 11 + 2 + 2,
    "r^-1 share of the warp inversion + u1, u2 mod n": 12 + 6,
    "affine Q: ZZZ^-1 share of the warp inversion, x = X (ZZ ZZZ^-1)^2, y = Y ZZZ^-1, canonical": 12 + 4 + 2,
}


def _rows_timed(run, reps):
    run()
    best = BE.time_best(run, reps)
    nmsm.set_profiling(True)
    k_prep, k_check = [], []
    for _ in range(reps):
        run()
        ms = list(nmsm.last_timing()[0].values())  # slot 0: k_recover_prepare, slot 1: k_recover_check (include/nmsm.h)
        k_prep.append(ms[0])
        k_check.append(ms[1])
    nmsm.set_profiling(False)
    return best, min(k_prep), min(k_check)


def _row(tag, what, n, best, k_prep, k_check, ok):
    per_item = sum(RECOVER_MODMUL.values())
    kern_s = (k_prep + k_check) * 1e-3
    peak_mm = max(nmsm.bench_modmul(0, bps, thr, 3000, ilp) for (bps, thr, ilp) in ((4, 128, 1), (8, 128, 1), (8, 128, 2)))
    return {"config": tag, "what": what, "n": n, "gpu_ms_through_c_abi": best * 1e3, "items_per_s": n / best,
            "kernels_ms": {"k_recover_prepare": k_prep, "k_recover_check": k_check},
            "modmul_per_item": per_item, "modmul_formula": RECOVER_MODMUL,
            "roofline": {"achieved_gmodmul_s": per_item * n / kern_s / 1e9, "peak_gmodmul_s": peak_mm / 1e9,
                         "frac": per_item * n / kern_s / peak_mm, "peak_source": "nmsm_bench_modmul(field=256-bit), same run"},
            "check": "all recovered, 4 oracle recoveries agree" if ok else "MISMATCH"}


def recover_config(tag, logn, items, reps=5):
    n = 1 << logn
    tiled = (items * (n // len(items) + 1))[:n]
    sigs, msgs, msg_off = RC.pack([i[0] for i in tiled], [i[1] for i in tiled])
    res = {}

    def run():
        res["out"] = nmsm.ecdsa_recover_batch_packed(sigs, msgs, msg_off, n, nmsm.ECDSA_PREHASH)

    best, k_prep, k_check = _rows_timed(run, reps)
    xy, ok = res["out"]
    good = ok == b"\x01" * n and all(xy[64 * k:64 * k + 64] == RC.xy_bytes(tiled[k][2]) for k in range(n))
    good = good and all(RR.secp256k1_recover_public_key(*items[k][:2]) == items[k][2] for k in range(4))
    return _row(tag, "secp256k1 ECDSA public-key recovery, 2^%d signatures (%d unique, tiled), prehash, 32-byte "
                     "messages" % (logn, len(items)), n, best, k_prep, k_check, good)


def ecrecover_config(tag, logn, inputs, reps=5):
    n = 1 << logn
    tiled = (inputs * (n // len(inputs) + 1))[:n]
    data = b"".join(i[0] for i in tiled)
    res = {}

    def run():
        res["out"] = nmsm.eth_ecrecover_batch_packed(data, n)

    best, k_prep, k_check = _rows_timed(run, reps)
    words, ok = res["out"]
    good = ok == b"\x01" * n and all(words[32 * k:32 * k + 32] == tiled[k][1] for k in range(n))
    good = good and all(RR.eth_ecrecover(inputs[k][0]) == inputs[k][1] for k in range(4))
    return _row(tag, "Ethereum ecrecover (precompile 0x01), 2^%d inputs (%d unique, tiled)" % (logn, len(inputs)), n,
                best, k_prep, k_check, good)


def ecrecover_inputs(count, seed):
    """count precompile inputs from the oracle signer with v = 27 or 28, and their expected output words"""
    rnd = random.Random(seed)
    ds = [rnd.randrange(1, E.N) for _ in range(8)]
    words = [bytes(12) + RR.eth_address(*RC.key_of(d)) for d in ds]
    out = []
    while len(out) < count:
        j = rnd.randrange(len(ds))
        h = E.be32(rnd.randrange(2**256))
        sig = RC.sign_rec(ds[j], E.bits2int_modn(h), rnd)
        if sig[0] < 2:
            out.append((h + E.be32(27 + sig[0]) + sig[1:], words[j]))
    return out


def rows():
    items = RC.signed_batch(4096, seed=30, msg_len=32)  # signed before any timed window
    inputs = ecrecover_inputs(4096, seed=31)
    sig, msg, _ = items[0]
    t0 = time.perf_counter()
    assert nmsm.ecdsa_recover_batch([sig], [msg])[0] is not None  # first call after nmsm_init: builds the table of G
    first_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    assert nmsm.ecdsa_recover_batch([sig], [msg])[0] is not None
    second_ms = (time.perf_counter() - t0) * 1e3
    yield {"config": "recover-card-before", "card": BE.card_info(), "g_table_build_ms": first_ms - second_ms,
           "first_call_ms": first_ms, "second_call_ms": second_ms}
    yield BE.ecdsa_config("ecdsa-20", 20, 4096)
    yield recover_config("recover-16", 16, items)
    yield recover_config("recover-20", 20, items)
    yield ecrecover_config("ecrecover-20", 20, inputs)
    yield {"config": "recover-card-after", "card": BE.card_info()}


def main():
    nmsm.init(0)
    for row in rows():
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
