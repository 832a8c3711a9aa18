#!/usr/bin/env python3
"""BLS12-381 aggregate verification on one H100 (nmsm_bls12_381_aggregate_verify_batch), next to
nmsm_bls12_381_verify_msg_batch in the same process.  Not a BASELINE.json config.

    python tests/bench_bls_aggregate.py

Rows (one JSON line each; every verdict of a timed row must be 1, reported as "all accepted"):
  agg-card              the card's name / power limit / max SM clock
  agg-fav-14x128        FastAggregateVerify: 2^14 checks of 128 keys, one 32-byte message each, _POP_ tag
  agg-fav-12x512        2^12 checks of 512 keys
  agg-fav-10x2048       2^10 checks of 2048 keys
  agg-verifybatch-12    noble's verifyBatch: one check of 2^12 distinct messages, one key each (bounded by the
                        one-thread Fp12 product of k_bls_final over the check's pairs)
  agg-verify-msg-14     baseline: nmsm_bls12_381_verify_msg_batch, 2^14 one-key signatures
  agg-card-after        the card read again after the timed rows
Wall time is best of K through the C ABI with H2D of every input included; kernel times come from the profiling slots
in a separate pass.  "model_kmul" is the issue's modmul count (381-bit multiplications, thousands), not a measurement.
"""
import json
import os
import random
import struct
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_ecdsa as BE  # noqa: E402  (sets up the import paths, nmsm, card_info and time_best)

nmsm = BE.nmsm
from oracle import bls_pairing_ref as B  # noqa: E402

DST = nmsm.DST_G2_POP
N = B.N
SLOTS = ["prepare", "count", "scan", "scatter", "accumulate", "total"]
KERNELS = ["k_bls_hash_to_g2", "key_sums", "k_bls_agg_prepare", "k_bls_miller", "k_bls_final", "total"]
# modmuls per unit (tests/bench_bls.py's constants): signature decode + G2 subgroup check, one Miller loop, one final
# exponentiation, one hash, one key addition
M_SIG, M_MILLER, M_FINAL, M_HASH, M_KEY = 9.8e3, 6.65e3, 7.8e3, 9e3, 10


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


def _u64(v):
    return struct.pack("<%dQ" % len(v), *v)


def _scalars(ks):
    return b"".join((k % N).to_bytes(32, "little") for k in ks)


_TABLE = None


def _keys(sks) -> bytes:
    global _TABLE
    if _TABLE is None:
        _TABLE = nmsm.PointTable(nmsm.BLS12_381_G1, nmsm.bls12_381.G1.Point.BASE.to_packed())
    out, _ = _TABLE.mul_batch(_scalars(sks), len(sks), False)
    return out


def _sig_points(msgs, scalars):
    off = [0]
    for m in msgs:
        off.append(off[-1] + len(m))
    hs = nmsm.bls_hash_to_g2_batch_packed(b"".join(msgs), _u64(off), len(msgs), DST)
    out, infs = nmsm.mul_batch_packed(nmsm.BLS12_381_G2, hs, _scalars(scalars), len(msgs), True)
    G2 = nmsm.bls12_381.G2.Point
    return [G2.from_packed(out[192 * i:192 * i + 192], infs[i], True) for i in range(len(msgs))]


def _row(name, args, n_checks, model, reps):
    run = lambda: nmsm.bls_aggregate_verify_batch_packed(*args, n_checks, DST)  # noqa: E731
    accepted = run() == b"\1" * n_checks
    wall = BE.time_best(run, reps)
    ks = _slots(run, 3, SLOTS)
    return {"row": name, "checks": n_checks, "wall_ms": round(wall * 1e3, 2), "checks_per_s": round(n_checks / wall),
            "all_accepted": accepted, "kernels_ms": {k: round(v, 3) for k, v in zip(KERNELS, ks)},
            "model_kmul": round(model / 1e3)}


def fav_row(log_checks, size, reps):
    n = 1 << log_checks
    rnd = random.Random(log_checks * 7919 + size)
    sks = [rnd.randrange(1, N) for _ in range(n * size)]
    keys = _keys(sks)
    msgs = [rnd.randbytes(32) for _ in range(n)]
    sums = [sum(sks[j * size:(j + 1) * size]) % N for j in range(n)]
    sigs = b"".join(nmsm._bls_g2_compress(p) for p in _sig_points(msgs, sums))
    args = (sigs, _u64(range(n + 1)), b"".join(msgs), _u64(range(0, 32 * (n + 1), 32)), keys,
            _u64(range(0, size * (n + 1), size)))
    model = n * (M_SIG + 2 * M_MILLER + M_FINAL + M_HASH) + n * size * M_KEY
    return _row("agg-fav-%dx%d" % (log_checks, size), args, n, model, reps)


def verifybatch_row(log_msgs, reps):
    g = 1 << log_msgs
    rnd = random.Random(log_msgs)
    sks = [rnd.randrange(1, N) for _ in range(g)]
    keys = _keys(sks)
    msgs = [rnd.randbytes(32) for _ in range(g)]
    sig = nmsm._bls_g2_compress(nmsm.aggregate_points(nmsm.bls12_381.G2.Point, _sig_points(msgs, sks)))
    args = (sig, _u64([0, g]), b"".join(msgs), _u64(range(0, 32 * (g + 1), 32)), keys, _u64(range(g + 1)))
    model = M_SIG + (g + 1) * M_MILLER + M_FINAL + g * M_HASH + g * M_KEY
    return _row("agg-verifybatch-%d" % log_msgs, args, 1, model, reps)


def verify_msg_row(logn, reps):
    n = 1 << logn
    rnd = random.Random(logn)
    sks = [rnd.randrange(1, N) for _ in range(n)]
    G1 = nmsm.bls12_381.G1.Point
    raw = _keys(sks)
    pks = b"".join(G1.from_packed(raw[96 * i:96 * i + 96], 0, True).toBytes(True) for i in range(n))
    msgs = [rnd.randbytes(32) for _ in range(n)]
    sigs = b"".join(nmsm._bls_g2_compress(p) for p in _sig_points(msgs, sks))
    data, off = b"".join(msgs), _u64(range(0, 32 * (n + 1), 32))
    run = lambda: nmsm.bls_verify_messages_batch_packed(sigs, pks, data, off, n, DST)  # noqa: E731
    accepted = run() == b"\1" * n
    wall = BE.time_best(run, reps)
    ks = _slots(run, 3, ["prepare", "count", "scan", "scatter", "total"])
    names = ["k_bls_hash_to_g2", "k_bls_verify_prepare", "k_bls_miller", "k_bls_final", "total"]
    return {"row": "agg-verify-msg-%d" % logn, "checks": n, "wall_ms": round(wall * 1e3, 2),
            "checks_per_s": round(n / wall), "all_accepted": accepted,
            "kernels_ms": {k: round(v, 3) for k, v in zip(names, ks)}}


def main():
    nmsm.init(0)
    print(json.dumps({"row": "agg-card", **BE.card_info()}), flush=True)
    for log_checks, size in ((14, 128), (12, 512), (10, 2048)):
        print(json.dumps(fav_row(log_checks, size, 5)), flush=True)
    print(json.dumps(verifybatch_row(12, 3)), flush=True)
    print(json.dumps(verify_msg_row(14, 5)), flush=True)
    print(json.dumps({"row": "agg-card-after", **BE.card_info()}), flush=True)


if __name__ == "__main__":
    main()
