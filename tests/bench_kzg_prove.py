#!/usr/bin/env python3
"""The EIP-4844 prover on one H100 (nmsm.KzgSetup: nmsm_bls12_381_kzg_setup_create, _commit_batch,
_compute_blob_proof_batch, _compute_proof_batch) next to the per-blob MSM-engine path it replaces.  Not a BASELINE.json
config.  The setup is the oracle's Lagrange points of a seeded test tau (tests/kzg_cases.py): the work is the same as
with the ceremony's points.

    python tests/bench_kzg_prove.py

Rows (one JSON line each):
  kzg-prove-card            the card's name / power limit / max SM clock
  kzg-setup-create          nmsm_bls12_381_kzg_setup_create: wall time (one build; the setup is built twice and the
                            second is timed) and the table's bytes, with the point check and table kernel slots
  kzg-commit-6 / -10 / -12  blob_to_kzg_commitment of 6, 2^10, 2^12 blobs (4 distinct, tiled): wall time best of K
                            through the C ABI (H2D of the blobs and D2H included) and the lincomb kernel slot.  6 and
                            2^10 sit on either side of the lincomb's lanes-per-blob choice (4096 and 128 lanes)
  kzg-blob-proof-6 / -10    compute_blob_kzg_proof: slots challenge (+ commitment check), eval, quotient, lincomb
  kzg-proof-10              compute_kzg_proof at 2^10 random z: slots eval, quotient, lincomb
  kzg-commit-engine-10      the reference path: the same 2^10 commitments through the MSM engine, one
                            nmsm_msm_points_submit per blob over the four slots on a PointSet of the bit-reversed setup
                            points with precompute(); scalars byte-reversed to the engine's little-endian layout before
                            timing.  Results are checked against the comb's
  kzg-prove-card-after      the card read again after the timed rows
"""
import ctypes
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_ecdsa as BE  # noqa: E402  (sets up the import paths, nmsm, card_info and time_best)

nmsm = BE.nmsm
import kzg_cases as C  # noqa: E402
from oracle import hash_to_g1_ref as H  # noqa: E402
from oracle import kzg_ref as K  # noqa: E402
import kzg_prove_ref as KP  # noqa: E402

NAMES = ["prepare", "count", "scan", "scatter", "total"]  # timing slots 0-3 and NMSM_T_TOTAL


def _slots(run, reps, k):
    nmsm.set_profiling(True)
    best = [float("inf")] * (k + 1)
    for _ in range(reps):
        run()
        ms, _ = nmsm.last_timing()
        for j, nm in enumerate(NAMES[:k] + ["total"]):
            best[j] = min(best[j], ms[nm])
    nmsm.set_profiling(False)
    return [round(v, 2) for v in best]


def _blobs(n):
    base = [C.blob_item(s) for s in range(1, 5)]
    items = [base[k % 4] for k in range(n)]
    return items, b"".join(i[0] for i in items)


def setup_row(lagrange):
    t0 = time.perf_counter()
    first = nmsm.KzgSetup(lagrange)
    first_s = time.perf_counter() - t0
    first.close()
    nmsm.set_profiling(True)
    t0 = time.perf_counter()
    s = nmsm.KzgSetup(lagrange)
    wall = time.perf_counter() - t0
    ms, _ = nmsm.last_timing()
    nmsm.set_profiling(False)
    levels = (255 + 1 + 7) // 8
    return s, {"row": "kzg-setup-create", "wall_s": round(wall, 3), "first_wall_s": round(first_s, 3),
               "table_bytes": levels * 4096 * 128 * 96,
               "kernels_ms": {"point_check": round(ms["prepare"], 2), "table": round(ms["count"], 2)}}


def commit_row(s, logn, reps):
    n = 6 if logn is None else 1 << logn
    items, blobs = _blobs(n)
    run = lambda: s.blob_to_kzg_commitment_batch_packed(blobs, n)  # noqa: E731
    out, ok = run()
    assert ok == b"\1" * n and out == b"".join(i[1] for i in items)
    wall = BE.time_best(run, reps)
    ks = _slots(run, 3, 1)
    return {"row": "kzg-commit-%s" % (6 if logn is None else logn), "n": n, "wall_ms": round(wall * 1e3, 2),
            "rate_per_s": round(n / wall), "kernels_ms": {"k_kzg_lincomb": ks[0], "total": ks[1]}}


def blob_proof_row(s, logn, reps):
    n = 6 if logn is None else 1 << logn
    items, blobs = _blobs(n)
    cs = b"".join(i[1] for i in items)
    run = lambda: s.compute_blob_kzg_proof_batch_packed(blobs, cs, n)  # noqa: E731
    out, ok = run()
    assert ok == b"\1" * n and out == b"".join(i[2] for i in items)
    wall = BE.time_best(run, reps)
    ks = _slots(run, 3, 4)
    return {"row": "kzg-blob-proof-%s" % (6 if logn is None else logn), "n": n, "wall_ms": round(wall * 1e3, 2),
            "rate_per_s": round(n / wall),
            "kernels_ms": {"k_kzg_challenge+commit_check": ks[0], "k_kzg_eval": ks[1], "k_kzg_quotient": ks[2],
                           "k_kzg_lincomb": ks[3], "total": ks[4]}}


def proof_row(s, logn, reps):
    n = 1 << logn
    items, blobs = _blobs(n)
    rnd = random.Random(logn)
    zs = [rnd.randrange(C.R) for _ in range(4)]
    zb = b"".join(C.be(zs[k % 4]) for k in range(n))
    run = lambda: s.compute_kzg_proof_batch_packed(blobs, zb, n)  # noqa: E731
    out, ys, ok = run()
    assert ok == b"\1" * n
    for k in range(4):  # each distinct (blob, z) opens under the verifier
        assert nmsm.kzg_verify_proof_batch([items[k][1]], [zs[k]], [ys[32 * k:32 * k + 32]],
                                           [out[48 * k:48 * k + 48]], C.SETUP) == [True]
    wall = BE.time_best(run, reps)
    ks = _slots(run, 3, 3)
    return {"row": "kzg-proof-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2), "rate_per_s": round(n / wall),
            "kernels_ms": {"k_kzg_eval": ks[0], "k_kzg_quotient": ks[1], "k_kzg_lincomb": ks[2], "total": ks[3]}}


def engine_row(lagrange, logn, reps):
    from nmsm import _lib

    n = 1 << logn
    items, _ = _blobs(n)
    pts = KP.bit_reversal_permutation(lagrange)
    packed = b"".join(H.g1_packed(K.g1_decode(p)) for p in pts)
    ps = nmsm.PointSet(4, packed, 4096)  # BLS12-381 G1: the setup points lie in G1
    bits, levels = ps.precompute(0)
    lib = _lib.load()
    # scalars in the engine's layout: each 32-byte big-endian element byte-reversed (done before timing)
    scal = [b"".join(i[0][32 * k:32 * k + 32][::-1] for k in range(4096)) for i in items]
    bufs = [ctypes.create_string_buffer(s, len(s)) for s in scal]
    outs = [ctypes.create_string_buffer(96) for _ in range(n)]
    infs = [ctypes.c_int(0) for _ in range(n)]

    def run():
        for b in range(n):
            slot = b % 4
            if b >= 4:
                _lib.check(lib.nmsm_msm_collect(slot, outs[b - 4], ctypes.byref(infs[b - 4])))
            _lib.check(lib.nmsm_msm_points_submit(ps.handle, bufs[b], 4096, 0, slot))
        for b in range(max(0, n - 4), n):
            _lib.check(lib.nmsm_msm_collect(b % 4, outs[b], ctypes.byref(infs[b])))

    run()
    for b in range(4):
        raw = outs[b].raw
        got = H.g1_encode((int.from_bytes(raw[:48], "little"), int.from_bytes(raw[48:], "little")))
        assert got == items[b][1]
    wall = BE.time_best(run, reps)
    ps.close()
    return {"row": "kzg-commit-engine-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2),
            "rate_per_s": round(n / wall), "table_window_bits": bits, "table_levels": levels}


def main():
    nmsm.init(0)
    print(json.dumps({"row": "kzg-prove-card", **BE.card_info()}), flush=True)
    lagrange = KP.setup_g1_lagrange(C.TAU)
    s, row = setup_row(lagrange)
    print(json.dumps(row), flush=True)
    print(json.dumps(commit_row(s, None, 5)), flush=True)
    print(json.dumps(commit_row(s, 10, 5)), flush=True)
    print(json.dumps(commit_row(s, 12, 3)), flush=True)
    print(json.dumps(blob_proof_row(s, None, 5)), flush=True)
    print(json.dumps(blob_proof_row(s, 10, 3)), flush=True)
    print(json.dumps(proof_row(s, 10, 3)), flush=True)
    s.close()
    print(json.dumps(engine_row(lagrange, 10, 3)), flush=True)
    print(json.dumps({"row": "kzg-prove-card-after", **BE.card_info()}), flush=True)


if __name__ == "__main__":
    main()
