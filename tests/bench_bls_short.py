#!/usr/bin/env python3
"""BLS12-381 hash to G1 and short-signature verification on one H100 (nmsm_bls12_381_hash_to_g1_batch,
nmsm_bls12_381_short_verify_msg_batch), next to hash to G2 and long-signature verification from bytes in the same
process.  Not a BASELINE.json config.

    python tests/bench_bls_short.py

Rows (one JSON line each):
  short-card            the card's name / power limit / max SM clock
  short-h2g1-16 / -20   2^16 / 2^20 messages of 32 bytes under DST_G1_NUL: wall time best of K through the C ABI (H2D
                        of the messages and D2H of the points included) and k_bls_hash_to_g1 from the profiling slot
  short-verify-msg-16   2^16 short signatures from message bytes (16 keys, 64 signed messages, tiled): wall time and the
                        four kernels, with the prepare kernel's share of the kernel total
  short-verify-16       nmsm_bls12_381_short_verify_batch on the same items with the messages hashed beforehand
  long-h2g2-16          hash to G2 at 2^16 (32-byte messages) in the same process
  long-verify-msg-16    nmsm_bls12_381_verify_msg_batch at 2^16 in the same process
  short-card-after      the card read again after the timed rows
"""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_ecdsa as BE  # noqa: E402  (sets up the import paths, nmsm, card_info and time_best)

nmsm = BE.nmsm
import h2c_cases as C2  # noqa: E402
import h2g1_cases as C  # noqa: E402
from oracle import bls_pairing_ref as B  # noqa: E402
from oracle import hash_to_curve_ref as H2  # noqa: E402
from oracle import hash_to_g1_ref as H  # noqa: E402

DST = H.DST_G1_NUL


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


def h2g1_row(logn, reps):
    n = 1 << logn
    rnd = random.Random(logn)
    msgs = [rnd.randbytes(32) for _ in range(n)]
    data, off = C.pack_messages(msgs)
    run = lambda: nmsm.bls_hash_to_g1_batch_packed(data, off, n, DST)  # noqa: E731
    out = run()
    sample = [0, n // 2, n - 1]
    assert [out[96 * k:96 * k + 96] for k in sample] == C.oracle_packed([msgs[k] for k in sample], DST, workers=1)
    wall = BE.time_best(run, reps)
    (kern,) = _slots(run, 3, ["prepare"])
    return {"row": "short-h2g1-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2), "rate_per_s": round(n / wall),
            "k_bls_hash_to_g1_ms": round(kern, 2)}


def short_rows(logn, reps):
    n = 1 << logn
    rnd = random.Random(99)
    sks = [rnd.randrange(1, H.N) for _ in range(16)]
    pks = [H.public_key(sk) for sk in sks]
    uniq = []
    for k in range(64):
        msg = rnd.randbytes(32)
        uniq.append((H.sign(sks[k % 16], H.hash_to_g1(msg, DST)), msg, pks[k % 16]))
    items = [uniq[k % 64] for k in range(n)]
    sigs, keys = b"".join(i[0] for i in items), b"".join(i[2] for i in items)
    msgs = [i[1] for i in items]
    data, off = C.pack_messages(msgs)
    pts = nmsm.bls_hash_to_g1_batch_packed(data, off, n, DST)
    run_msg = lambda: nmsm.bls_short_verify_messages_batch_packed(sigs, keys, data, off, n, DST)  # noqa: E731
    run_pts = lambda: nmsm.bls_short_verify_batch_packed(sigs, keys, pts, n)  # noqa: E731
    assert run_msg() == b"\1" * n and run_pts() == b"\1" * n
    rows = []
    wall = BE.time_best(run_msg, reps)
    ks = _slots(run_msg, 3, ["prepare", "count", "scan", "scatter", "total"])
    rows.append({"row": "short-verify-msg-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2),
                 "rate_per_s": round(n / wall),
                 "kernels_ms": {"k_bls_hash_to_g1": round(ks[0], 2), "k_bls_short_verify_prepare": round(ks[1], 2),
                                "k_bls_miller": round(ks[2], 2), "k_bls_final": round(ks[3], 2),
                                "total": round(ks[4], 2)},
                 "prepare_share": round(ks[1] / ks[4], 3)})
    wall = BE.time_best(run_pts, reps)
    ks = _slots(run_pts, 3, ["prepare", "count", "scan", "total"])
    rows.append({"row": "short-verify-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2),
                 "rate_per_s": round(n / wall),
                 "kernels_ms": {"k_bls_short_verify_prepare": round(ks[0], 2), "k_bls_miller": round(ks[1], 2),
                                "k_bls_final": round(ks[2], 2), "total": round(ks[3], 2)}})
    return rows


def long_rows(logn, reps):
    n = 1 << logn
    rnd = random.Random(logn)
    msgs = [rnd.randbytes(32) for _ in range(n)]
    data, off = C.pack_messages(msgs)
    dst = H2.DST_G2_NUL
    run = lambda: nmsm.bls_hash_to_g2_batch_packed(data, off, n, dst)  # noqa: E731
    run()
    wall = BE.time_best(run, reps)
    (kern,) = _slots(run, 3, ["prepare"])
    rows = [{"row": "long-h2g2-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2), "rate_per_s": round(n / wall),
             "k_bls_hash_to_g2_ms": round(kern, 2)}]
    uniq = []
    for k in range(16):
        msg = rnd.randbytes(32)
        sk = rnd.randrange(1, B.N)
        h = H2.hash_to_g2(msg, dst)
        uniq.append((B.sign(sk, B.G2.fromAffine({"x": h[0], "y": h[1]})), msg, B.public_key(sk)))
    items = [uniq[k % 16] for k in range(n)]
    sigs, pks = b"".join(i[0] for i in items), b"".join(i[2] for i in items)
    data, off = C2.pack_messages([i[1] for i in items])
    run_msg = lambda: nmsm.bls_verify_messages_batch_packed(sigs, pks, data, off, n, dst)  # noqa: E731
    assert run_msg() == b"\1" * n
    wall = BE.time_best(run_msg, reps)
    ks = _slots(run_msg, 3, ["prepare", "count", "scan", "scatter", "total"])
    rows.append({"row": "long-verify-msg-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2),
                 "rate_per_s": round(n / wall),
                 "kernels_ms": {"k_bls_hash_to_g2": round(ks[0], 2), "k_bls_verify_prepare": round(ks[1], 2),
                                "k_bls_miller": round(ks[2], 2), "k_bls_final": round(ks[3], 2),
                                "total": round(ks[4], 2)}})
    return rows


def main():
    nmsm.init(0)
    print(json.dumps({"row": "short-card", **BE.card_info()}), flush=True)
    print(json.dumps(h2g1_row(16, 5)), flush=True)
    print(json.dumps(h2g1_row(20, 3)), flush=True)
    for row in short_rows(16, 5) + long_rows(16, 5):
        print(json.dumps(row), flush=True)
    print(json.dumps({"row": "short-card-after", **BE.card_info()}), flush=True)


if __name__ == "__main__":
    main()
