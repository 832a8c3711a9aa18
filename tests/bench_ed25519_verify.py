#!/usr/bin/env python3
"""ed25519 verification with one verdict per signature on one H100 (nmsm_ed25519_verify_each), next to the batch
equation (nmsm_ed25519_verify_batch) in the same process on the same card.  Not a BASELINE.json config.

    python tests/bench_ed25519_verify.py

Rows (one JSON line each):
  ed-each-setup     the card's name / power limit / max SM clock, and the one-off build of the table of B by the first
                    per-signature verify after nmsm_init (first call minus a second call)
  ed-batch-16       the batch equation over 2^16 signatures (one verdict for the batch)
  ed-each-16/20     2^16 / 2^20 signatures in ZIP-215 mode; ed-each-20-strict the same 2^20 in strict mode.  32-byte
                    messages, 4096 unique OpenSSL-signed signatures (signed before any timed window) tiled.  Wall time
                    best of K through the C ABI on packed arrays (H2D included), k_ed_verify_prepare / k_ed_verify_check
                    from CUDA events, modmul-equivalents per signature (ED_VERIFY_MODMUL below) against
                    nmsm_bench_modmul(0, ...) of the same run
  ed-forgery-16     the 2^16 batch with one signature whose s is off by one (it decodes): what each entry point returns
                    and in what time
  ed-cpu            OpenSSL verifies/s on one host thread (labelled)
  ed-each-card-after  the card read again after the timed rows
The script lives under tests/ because it uses the oracle and tests/ed25519_cases.py; pytest does not collect it.
"""
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_ecdsa as BE  # noqa: E402  (sets up the import paths, nmsm, card_info and time_best)

nmsm = BE.nmsm
import ed25519_cases as C  # noqa: E402
from oracle import noble_ref as R  # noqa: E402

# Field multiplications (1S = 1M) one signature costs on the GPU, from the kernels' formulas (ec.cuh EdExt: mixed
# addition 7, addition 9, doubling 8).  SHA-512 is not counted, nor the strict mode's [8]A (31 more).
ED_VERIFY_MODMUL = {
    "decode A and R: 2 x (x^((p-5)/8): 252 squarings + 11 multiplications, uvRatio 12)": 2 * (252 + 11 + 12),
    "s*B (16 table mixed additions)": 16 * 7,
    "k*A table (1..8)A: from_affine, 1 doubling, 6 mixed additions, prepare": 7 + 8 + 6 * 7 + 4,
    "k*A: 63 x 4 doublings + 15/16 of 64 additions": 63 * 4 * 8 + 60 * 9,
    "- k*A, - R, [8]": 9 + 7 + 4 + 3 * 8,
    "k mod l, s and k conversions": 6,
}


def _packed(logn, items):
    n = 1 << logn
    tiled = (items * (n // len(items) + 1))[:n]
    return n, tiled, C.pack([i[0] for i in tiled], [i[1] for i in tiled], [i[2] for i in tiled])


def _peak_modmul():
    return max(nmsm.bench_modmul(0, bps, thr, 3000, ilp) for (bps, thr, ilp) in ((4, 128, 1), (8, 128, 1), (8, 128, 2)))


def each_config(tag, logn, items, zip215=True, reps=5):
    n, _, (sigs, pks, msgs, msg_off) = _packed(logn, items)
    res = {}

    def run():
        res["ok"] = nmsm.ed25519_verify_each_packed(sigs, pks, msgs, msg_off, n, zip215)

    run()
    best = BE.time_best(run, reps)
    nmsm.set_profiling(True)
    k_prep, k_check = [], []
    for _ in range(reps):
        run()
        ms = list(nmsm.last_timing()[0].values())  # slot 0: k_ed_verify_prepare, slot 1: k_ed_verify_check
        k_prep.append(ms[0])
        k_check.append(ms[1])
    nmsm.set_profiling(False)
    ok = res["ok"] == b"\x01" * n and all(R.ed25519_verify(*items[i], zip215=zip215) for i in range(4))
    per_sig = sum(ED_VERIFY_MODMUL.values())
    kern_s = (min(k_prep) + min(k_check)) * 1e-3
    peak_mm = _peak_modmul()
    return {"config": tag, "what": "ed25519 verify, one verdict per signature, %s, 2^%d signatures (%d unique, tiled), "
                                   "32-byte messages" % ("ZIP-215" if zip215 else "strict", logn, len(items)), "n": n,
            "gpu_ms_through_c_abi": best * 1e3, "signatures_per_s": n / best,
            "kernels_ms": {"k_ed_verify_prepare": min(k_prep), "k_ed_verify_check": min(k_check)},
            "modmul_per_signature": per_sig, "modmul_formula": ED_VERIFY_MODMUL,
            "roofline": {"achieved_gmodmul_s": per_sig * n / kern_s / 1e9, "peak_gmodmul_s": peak_mm / 1e9,
                         "frac": per_sig * n / kern_s / peak_mm, "peak_source": "nmsm_bench_modmul(field=256-bit), same run"},
            "check": "all accepted, 4 oracle verifies agree" if ok else "MISMATCH"}


def batch_config(tag, logn, items, reps=5):
    n, _, (sigs, pks, msgs, msg_off) = _packed(logn, items)
    z = random.Random(logn).randbytes(16 * n)
    res = {}

    def run():
        res["out"] = nmsm.ed25519_verify_batch_packed(sigs, pks, msgs, msg_off, n, z)

    run()
    best = BE.time_best(run, reps)
    return {"config": tag, "what": "ed25519 batch equation (one verdict for the batch), 2^%d signatures (%d unique, "
                                   "tiled), 32-byte messages" % (logn, len(items)), "n": n,
            "gpu_ms_through_c_abi": best * 1e3, "signatures_per_s": n / best,
            "check": "batch accepted" if res["out"] == (True, -1) else "MISMATCH"}


def forgery_config(tag, logn, items, reps=5):
    n, tiled, _ = _packed(logn, items)
    idx = n // 3
    sig, msg, pk = tiled[idx]
    tiled = list(tiled)
    tiled[idx] = (sig[:32] + C.le32((int.from_bytes(sig[32:], "little") + 1) % C.L), msg, pk)
    sigs, pks, msgs, msg_off = C.pack([i[0] for i in tiled], [i[1] for i in tiled], [i[2] for i in tiled])
    z = random.Random(logn + 1).randbytes(16 * n)
    res = {}

    def run_batch():
        res["batch"] = nmsm.ed25519_verify_batch_packed(sigs, pks, msgs, msg_off, n, z)

    def run_each():
        res["each"] = nmsm.ed25519_verify_each_packed(sigs, pks, msgs, msg_off, n)

    run_batch()
    run_each()
    t_batch = BE.time_best(run_batch, reps)
    t_each = BE.time_best(run_each, reps)
    zeros = [k for k, v in enumerate(res["each"]) if v != 1]
    ok = res["batch"] == (False, -1) and zeros == [idx] and not R.ed25519_verify(*tiled[idx])
    return {"config": tag, "what": "2^%d signatures, one decodable forgery (s + 1) at index %d" % (logn, idx), "n": n,
            "batch_equation": {"returns": {"ok": res["batch"][0], "bad_index": res["batch"][1]}, "ms": t_batch * 1e3},
            "verify_each": {"returns": {"zero_verdicts_at": zeros}, "ms": t_each * 1e3},
            "check": "batch False without an index, verify_each names the forgery" if ok else "MISMATCH"}


def rows():
    items = C.openssl_sign(4096, seed=20, msg_len=32)  # signed before any timed window
    sig, msg, pk = items[0]
    t0 = time.perf_counter()
    assert nmsm.ed25519.verify(sig, msg, pk)  # first per-signature verify after nmsm_init: builds the table of B
    first_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    assert nmsm.ed25519.verify(sig, msg, pk)
    second_ms = (time.perf_counter() - t0) * 1e3
    yield {"config": "ed-each-setup", "card": BE.card_info(), "b_table_build_ms": first_ms - second_ms,
           "first_call_ms": first_ms, "second_call_ms": second_ms}
    yield batch_config("ed-batch-16", 16, items)
    yield each_config("ed-each-16", 16, items)
    yield each_config("ed-each-20", 20, items)
    yield each_config("ed-each-20-strict", 20, items, zip215=False)
    yield forgery_config("ed-forgery-16", 16, items)
    cpu_items = items[:2000]
    t0 = time.perf_counter()
    for it in cpu_items:
        C.openssl_verify(*it)
    yield {"config": "ed-cpu", "cpu_openssl_verifies_per_s": len(cpu_items) / (time.perf_counter() - t0),
           "cpu_label": "OpenSSL via the Python cryptography package, 1 host thread, incl. key parsing per call"}
    yield {"config": "ed-each-card-after", "card": BE.card_info()}


def main():
    nmsm.init(0)
    for row in rows():
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
