#!/usr/bin/env python3
"""EIP-4844 KZG proof verification on one H100 (nmsm_bls12_381_kzg_verify_proof_batch with versioned hashes, i.e. the
point-evaluation precompile, and nmsm_bls12_381_kzg_verify_blob_batch), next to BLS signature verification in the same
process.  Not a BASELINE.json config.  The setup point is a seeded test tau (tests/kzg_cases.py): the pairing work is
the same as with the ceremony's point.

    python tests/bench_kzg.py

Rows (one JSON line each):
  kzg-card              the card's name / power limit / max SM clock
  kzg-point-eval-16     2^16 precompile inputs (64 distinct, tiled): wall time best of K through the C ABI (H2D of the
                        inputs, the setup check and D2H included) and the three kernel slots
  kzg-blob-10 / -12     2^10 / 2^12 blobs (128 MiB / 512 MiB, 4 distinct, tiled): wall time best of K through the C ABI
                        and the five kernel slots; h2d_ms is a separate pageable host-to-device copy of the same bytes
                        (torch), wall_minus_kernels_ms what the call spends outside the kernels (mostly that copy)
  bls-verify-16         nmsm_bls12_381_verify_batch at 2^16 (16 distinct, tiled) in the same process
  kzg-card-after        the card read again after the timed rows
"""
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_ecdsa as BE  # noqa: E402  (sets up the import paths, nmsm, card_info and time_best)

nmsm = BE.nmsm
import bls_cases as BC  # noqa: E402
import kzg_cases as C  # noqa: E402


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


def point_eval_row(logn, reps):
    n = 1 << logn
    items = C.proof_items(n, distinct=64, seed=logn)
    c, z, y, pi = C.pack_proofs(items)
    vh = b"".join(C.versioned_hash(i[0]) for i in items)
    run = lambda: nmsm.kzg_verify_proof_batch_packed(c, z, y, pi, vh, n, C.SETUP)  # noqa: E731
    assert run() == b"\1" * n
    wall = BE.time_best(run, reps)
    ks = _slots(run, 3, ["prepare", "count", "scan", "total"])
    return {"row": "kzg-point-eval-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2), "rate_per_s": round(n / wall),
            "kernels_ms": {"k_kzg_prepare+setup": round(ks[0], 2), "k_bls_miller": round(ks[1], 2),
                           "k_bls_final": round(ks[2], 2), "total": round(ks[3], 2)}}


def _h2d_ms(data: bytes, reps):
    import torch

    src = torch.frombuffer(bytearray(data), dtype=torch.uint8)
    dst = torch.empty(len(data), dtype=torch.uint8, device="cuda")
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dst.copy_(src)
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    del dst
    torch.cuda.empty_cache()
    return best * 1e3


def blob_row(logn, reps):
    n = 1 << logn
    base = [C.blob_item(s) for s in range(1, 5)]
    items = [base[k % 4] for k in range(n)]
    blobs = b"".join(i[0] for i in items)
    cs, pis = b"".join(i[1] for i in items), b"".join(i[2] for i in items)
    run = lambda: nmsm.kzg_verify_blob_proof_batch_packed(blobs, cs, pis, n, C.SETUP)  # noqa: E731
    assert run() == b"\1" * n
    wall = BE.time_best(run, reps)
    ks = _slots(run, 3, ["prepare", "count", "scan", "scatter", "accumulate", "total"])
    return {"row": "kzg-blob-%d" % logn, "n": n, "blob_bytes": len(blobs), "wall_ms": round(wall * 1e3, 2),
            "rate_per_s": round(n / wall),
            "kernels_ms": {"k_kzg_challenge": round(ks[0], 2), "k_kzg_eval": round(ks[1], 2),
                           "k_kzg_prepare+setup": round(ks[2], 2), "k_bls_miller": round(ks[3], 2),
                           "k_bls_final": round(ks[4], 2), "total": round(ks[5], 2)},
            "wall_minus_kernels_ms": round(wall * 1e3 - ks[5], 2), "h2d_ms": round(_h2d_ms(blobs, 3), 2)}


def bls_verify_row(logn, reps):
    n = 1 << logn
    rnd = random.Random(logn)
    uniq = [BC.keypair_item(rnd) for _ in range(16)]
    items = [uniq[k % 16] for k in range(n)]
    sigs, pks = b"".join(i[0] for i in items), b"".join(i[2] for i in items)
    hs = b"".join(BC.g2_bytes(i[1]) for i in items)
    run = lambda: nmsm.bls_verify_batch_packed(sigs, pks, hs, n)  # noqa: E731
    assert run() == b"\1" * n
    wall = BE.time_best(run, reps)
    ks = _slots(run, 3, ["prepare", "count", "scan", "total"])
    return {"row": "bls-verify-%d" % logn, "n": n, "wall_ms": round(wall * 1e3, 2), "rate_per_s": round(n / wall),
            "kernels_ms": {"k_bls_verify_prepare": round(ks[0], 2), "k_bls_miller": round(ks[1], 2),
                           "k_bls_final": round(ks[2], 2), "total": round(ks[3], 2)}}


def main():
    nmsm.init(0)
    print(json.dumps({"row": "kzg-card", **BE.card_info()}), flush=True)
    print(json.dumps(point_eval_row(16, 5)), flush=True)
    print(json.dumps(blob_row(10, 3)), flush=True)
    print(json.dumps(blob_row(12, 3)), flush=True)
    print(json.dumps(bls_verify_row(16, 5)), flush=True)
    print(json.dumps({"row": "kzg-card-after", **BE.card_info()}), flush=True)


if __name__ == "__main__":
    main()
