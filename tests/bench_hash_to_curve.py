#!/usr/bin/env python3
"""BLS12-381 hash to G2 and BLS verification from message bytes on one H100 (nmsm_bls12_381_hash_to_g2_batch,
nmsm_bls12_381_verify_msg_batch), next to nmsm_bls12_381_verify_batch in the same process.  Not a BASELINE.json config.

    python tests/bench_hash_to_curve.py

Rows (one JSON line each):
  h2c-card            the card's name / power limit / max SM clock
  h2c-hash-16 / -20   2^16 / 2^20 messages of 32 bytes under the _POP_ tag: wall time best of K through the C ABI
                      (H2D of the messages and D2H of the points included) and k_bls_hash_to_g2 from the profiling slot
  h2c-verify-msg-16   2^16 signatures from message bytes (16 unique signed messages, tiled): wall time and the four kernels
  h2c-verify-16       nmsm_bls12_381_verify_batch on the same 2^16 items with the messages hashed beforehand
  h2c-oracle          the Python oracle's rate for one hash on the host (not a baseline: no speed-up is claimed)
  h2c-card-after      the card read again after the timed rows
"""
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_ecdsa as BE  # noqa: E402  (sets up the import paths, nmsm, card_info and time_best)

nmsm = BE.nmsm
import h2c_cases as C  # noqa: E402
from oracle import bls_pairing_ref as B  # noqa: E402
from oracle import hash_to_curve_ref as H  # noqa: E402

DST = H.DST_G2_POP


def _slots(run, reps, names):
    nmsm.set_profiling(True)
    best = [float("inf")] * len(names)
    for _ in range(reps):
        run()
        ms, _ = nmsm.last_timing()
        for k, nm in enumerate(names):
            best[k] = min(best[k], ms[nm])
    nmsm.set_profiling(False)
    return best


def hash_row(logn, reps):
    n = 1 << logn
    rnd = random.Random(logn)
    msgs = [rnd.randbytes(32) for _ in range(n)]
    data, off = C.pack_messages(msgs)
    run = lambda: nmsm.bls_hash_to_g2_batch_packed(data, off, n, DST)  # noqa: E731
    out = run()
    sample = [0, n // 2, n - 1]
    assert [out[192 * k:192 * k + 192] for k in sample] == C.oracle_packed([msgs[k] for k in sample], DST, workers=1)
    wall = BE.time_best(run, reps)
    (kern,) = _slots(run, 3, ["prepare"])
    return {"row": "h2c-hash-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2), "rate_per_s": round(n / wall),
            "k_bls_hash_to_g2_ms": round(kern, 2)}


def verify_rows(logn, reps):
    n = 1 << logn
    rnd = random.Random(99)
    uniq = []
    for k in range(16):
        msg = rnd.randbytes(32)
        sk = rnd.randrange(1, B.N)
        h = H.hash_to_g2(msg, DST)
        uniq.append((B.sign(sk, B.G2.fromAffine({"x": h[0], "y": h[1]})), msg, B.public_key(sk)))
    items = [uniq[k % 16] for k in range(n)]
    sigs, pks = b"".join(i[0] for i in items), b"".join(i[2] for i in items)
    msgs = [i[1] for i in items]
    data, off = C.pack_messages(msgs)
    pts = nmsm.bls_hash_to_g2_batch_packed(data, off, n, DST)
    run_msg = lambda: nmsm.bls_verify_messages_batch_packed(sigs, pks, data, off, n, DST)  # noqa: E731
    run_pts = lambda: nmsm.bls_verify_batch_packed(sigs, pks, pts, n)  # noqa: E731
    assert run_msg() == b"\1" * n and run_pts() == b"\1" * n
    rows = []
    wall = BE.time_best(run_msg, reps)
    ks = _slots(run_msg, 3, ["prepare", "count", "scan", "scatter", "total"])
    rows.append({"row": "h2c-verify-msg-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2),
                 "rate_per_s": round(n / wall),
                 "kernels_ms": {"k_bls_hash_to_g2": round(ks[0], 2), "k_bls_verify_prepare": round(ks[1], 2),
                                "k_bls_miller": round(ks[2], 2), "k_bls_final": round(ks[3], 2),
                                "total": round(ks[4], 2)}})
    wall = BE.time_best(run_pts, reps)
    ks = _slots(run_pts, 3, ["prepare", "count", "scan", "total"])
    rows.append({"row": "h2c-verify-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2), "rate_per_s": round(n / wall),
                 "kernels_ms": {"k_bls_verify_prepare": round(ks[0], 2), "k_bls_miller": round(ks[1], 2),
                                "k_bls_final": round(ks[2], 2), "total": round(ks[3], 2)}})
    return rows


def main():
    nmsm.init(0)
    print(json.dumps({"row": "h2c-card", **BE.card_info()}), flush=True)
    print(json.dumps(hash_row(16, 5)), flush=True)
    print(json.dumps(hash_row(20, 3)), flush=True)
    for row in verify_rows(16, 5):
        print(json.dumps(row), flush=True)
    t0 = time.perf_counter()
    for k in range(20):
        H.hash_to_g2(bytes([k]) * 32, DST)
    dt = (time.perf_counter() - t0) / 20
    print(json.dumps({"row": "h2c-oracle", "ms_per_hash": round(dt * 1e3, 2), "rate_per_s": round(1 / dt, 1)}),
          flush=True)
    print(json.dumps({"row": "h2c-card-after", **BE.card_info()}), flush=True)


if __name__ == "__main__":
    main()
