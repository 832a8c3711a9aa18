#!/usr/bin/env python3
"""Measure every BASELINE.json config on one H100 (parity-checked, CUDA-event kernel times where the MSM
pipeline is used).  The headline (configs[1]/metric at 2^20) is bench.py; this writes the companion table.

    python tests/bench_configs.py

configs (BASELINE.json):
  0  secp256k1 Point.multiply batch of 1024 random scalars      (reference: CPU bigint; here also the GPU batch)
  1  BLS12-381 G1 MSM, 2^16
  2  bn254 G1 MSM, 2^20
  3  BLS12-381 G2 MSM, 2^18
  4  ed25519 batch-verify 2^16 signatures
Each line: {"config", "n", "gpu_ms" (best of K, wall through the C ABI incl. H2D), "per_s", "kernels_ms", "check"}.
CPU comparison numbers use the oracle (tests-only code) on a bounded sample and are labelled.  The script lives under
tests/ because it uses the oracle as its checker; pytest does not collect it.
"""
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "noble-curves_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import nmsm  # noqa: E402
import helpers as H  # noqa: E402
from oracle import noble_ref as R  # noqa: E402


def gen_terms(name, n, seed):
    P = R.CURVES[name]
    rnd = random.Random(seed)
    ks = [rnd.randrange(1, P.Fn.ORDER) for _ in range(n)]
    sc = [rnd.randrange(P.Fn.ORDER) for _ in range(n)]
    cid = H.CURVE_IDS[name]
    pts, infs = nmsm.mul_batch_packed(cid, H.point_bytes(name, P.BASE) * n, H.pack_scalars(ks), n, False)
    total = sum(k * s for k, s in zip(ks, sc)) % P.Fn.ORDER
    return pts, H.pack_scalars(sc), total


def time_best(fn, reps):
    best = 1e9
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    return best


def msm_config(idx, name, logn, reps=5):
    n = 1 << logn
    P = R.CURVES[name]
    pts, sc, total = gen_terms(name, n, 100 + idx)
    exp = H.expected_tuple(name, H.expected_from_total(P, total))
    cid = H.CURVE_IDS[name]
    nmsm.set_profiling(True)
    out = {}

    def run():
        o, inf = nmsm.msm_packed(cid, pts, sc, n)
        out["r"] = (*H.unpack_point(name, o), inf)

    run()
    best = time_best(run, reps)
    ms, info = nmsm.last_timing()
    return {"config": idx, "what": "%s MSM, 2^%d terms" % (name, logn), "n": n, "gpu_ms_e2e_host_buffers": best * 1e3,
            "gpu_ms_device": ms["total"], "points_per_s_device": n / (ms["total"] * 1e-3),
            "kernels_ms": {k: round(v, 4) for k, v in ms.items()},
            "plan": {"c": info.c, "windows": info.windows, "entries": info.sorted_entries, "modmul_equiv": info.modmul_equiv},
            "check": "bit-exact vs (sum k_i s_i)*G" if out["r"] == exp else "MISMATCH"}


def fixed_base_config(tag, name, logn, reps=5):
    """Same workload through a device-resident point set with a fixed-base table (nmsm_points_precompute)."""
    n = 1 << logn
    P = R.CURVES[name]
    pts, sc, total = gen_terms(name, n, 300 + logn)
    exp = H.expected_tuple(name, H.expected_from_total(P, total))
    cid = H.CURVE_IDS[name]
    nmsm.set_profiling(True)
    rows = {}
    for label, pre in (("plain_set", False), ("table", True)):
        ps = nmsm.PointSet(cid, pts, n)
        t0 = time.perf_counter()
        c, levels = ps.precompute(0) if pre else (0, 1)
        t_pre = time.perf_counter() - t0
        out = {}

        def run():
            o, inf = ps.msm(sc, n)
            out["r"] = (*H.unpack_point(name, o), inf)

        run()
        best = time_best(run, reps)
        ms, info = nmsm.last_timing()
        rows[label] = {"gpu_ms_host_scalars": best * 1e3, "gpu_ms_device": ms["total"],
                       "points_per_s_device": n / (ms["total"] * 1e-3),
                       "kernels_ms": {k: round(v, 4) for k, v in ms.items()},
                       "plan": {"c": info.c, "windows": info.windows, "entries": info.sorted_entries},
                       "table": {"window_bits": c, "levels": levels, "precompute_ms": t_pre * 1e3} if pre else None,
                       "check": "bit-exact vs (sum k_i s_i)*G" if out["r"] == exp else "MISMATCH"}
        ps.close()
    return {"config": tag, "what": "%s fixed-base MSM, 2^%d terms (point set resident on the device)" % (name, logn),
            "n": n, **rows}


def point_table_config(tag, name, logn, reps=3):
    """k_i * G for 2^logn random scalars: generic nmsm_mul_batch vs the fixed-point table (nmsm_point_table_*)."""
    n = 1 << logn
    P = R.CURVES[name]
    rnd = random.Random(500 + logn)
    ks = [rnd.randrange(1, P.Fn.ORDER) for _ in range(n)]
    sb = H.pack_scalars(ks)
    gb = H.point_bytes(name, P.BASE)
    cid = H.CURVE_IDS[name]
    t0 = time.perf_counter()
    tbl = nmsm.PointTable(cid, gb)
    t_build = time.perf_counter() - t0
    res = {}

    def run_tbl():
        res["t"] = tbl.mul_batch(sb, n, False)

    nmsm.set_profiling(True)
    run_tbl()
    best_t = time_best(run_tbl, reps)
    k_tbl = nmsm.last_timing()[0]["total"]
    # the same call at the C ABI with pinned host buffers (what an N-API addon with registered ArrayBuffers sees)
    import ctypes
    lib = nmsm._lib.load()
    pbytes = len(gb)
    h_sc, h_out, h_inf = lib.nmsm_host_alloc(n * 32), lib.nmsm_host_alloc(n * pbytes), lib.nmsm_host_alloc(n)
    ctypes.memmove(h_sc, sb, n * 32)

    def run_cabi():
        nmsm._lib.check(lib.nmsm_point_table_mul_batch(tbl.handle, h_sc, n, 0, h_out, h_inf))

    run_cabi()
    best_c = time_best(run_cabi, reps)
    cabi_ok = ctypes.string_at(h_out, n * pbytes) == res["t"][0]
    for hp in (h_sc, h_out, h_inf):
        lib.nmsm_host_free(hp)
    ng = min(n, 1 << 16)

    def run_gen():
        res["g"] = nmsm.mul_batch_packed(cid, gb * ng, sb[: ng * 32], ng, False)

    run_gen()
    best_g = time_best(run_gen, reps)
    k_gen = nmsm.last_timing()[0]["total"]
    pb = len(gb)
    ok = cabi_ok and res["t"][0][: ng * pb] == res["g"][0]
    ok &= H.unpack_point(name, res["t"][0][(n - 1) * pb:]) == R.affine_tuple(P, P.BASE.multiply(ks[-1]))
    tbl.close()
    return {"config": tag, "what": "%s BASE.multiply x 2^%d random scalars (getPublicKey shape), host buffers in and out" % (name, logn),
            "n": n, "table_kernel_ms": k_tbl, "table_kernel_multiplies_per_s": n / (k_tbl * 1e-3),
            "generic_kernel_ms": k_gen, "generic_kernel_multiplies_per_s": ng / (k_gen * 1e-3), "table_cabi_pinned_ms": best_c * 1e3, "table_cabi_pinned_multiplies_per_s": n / best_c,
            "table_python_binding_ms": best_t * 1e3, "table_python_binding_multiplies_per_s": n / best_t, "table_build_ms": t_build * 1e3,
            "generic_mul_batch_n": ng, "generic_ms": best_g * 1e3, "generic_multiplies_per_s": ng / best_g,
            "check": "table == generic batch bit-exact; oracle spot check" if ok else "MISMATCH"}


def ntt_config(tag, field, logn, reps=5):
    """Forward + inverse NTT over Fr, device-resident data (nmsm_ntt_device), CUDA-event time of the transform."""
    import ctypes

    import numpy as np
    import torch

    from nmsm import fft as GF

    n = 1 << logn
    rs = np.random.RandomState(logn)
    raw = rs.randint(0, 256, size=(n, 32), dtype=np.uint8)
    raw[:, 31] &= 0x0F
    host = torch.from_numpy(raw.reshape(-1))
    dev = host.cuda()
    nmsm.set_profiling(True)
    GF.ntt_device(field, dev.data_ptr(), logn, generator=7)             # builds the root table
    t_roots = nmsm.last_timing()[0]["prepare"]
    GF.ntt_device(field, dev.data_ptr(), logn, inverse=True, generator=7)
    ok = bool(torch.equal(dev.cpu(), host))
    fwd, inv = [], []
    for _ in range(reps):
        GF.ntt_device(field, dev.data_ptr(), logn, generator=7)
        fwd.append(nmsm.last_timing()[0]["total"])
        GF.ntt_device(field, dev.data_ptr(), logn, inverse=True, generator=7)
        inv.append(nmsm.last_timing()[0]["total"])
    ok &= bool(torch.equal(dev.cpu(), host))
    brp = []
    for _ in range(reps):
        GF.ntt_device(field, dev.data_ptr(), logn, brp_output=True, generator=7)
        brp.append(nmsm.last_timing()[0]["total"])
        GF.ntt_device(field, dev.data_ptr(), logn, inverse=True, brp_input=True, generator=7)
    ok &= bool(torch.equal(dev.cpu(), host))
    t = min(fwd)
    passes = (logn + 9) // 10
    # the bound (ncu: fmaheavy pipe ~62 % active, DRAM < 5 %): one 256-bit Montgomery multiplication per butterfly
    modmuls = (n // 2) * logn
    peak_mm = max(nmsm.bench_modmul(0, bps, thr, 3000, ilp) for (bps, thr, ilp) in ((4, 128, 1), (8, 128, 1), (4, 256, 1), (8, 128, 2)))
    # algorithmic HBM bytes: ingest (r+w) + passes x (r+w) + emit (r+w) + copy back (r+w), 32 B elements
    alg_bytes = (passes + 3) * 2 * n * 32
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("hbm_gbs", 3350.0)
    except Exception:
        peak = 3350.0  # H100 SXM data sheet
    return {"config": tag, "what": "NTT over Fr(%s), 2^%d elements, device-resident (generator 7)" % (field, logn), "n": n,
            "direct_ms": t, "inverse_ms": min(inv), "direct_brp_out_ms": min(brp), "root_table_ms": t_roots,
            "elements_per_s": n / (t * 1e-3), "butterflies_per_s": (n // 2) * logn / (t * 1e-3),
            "roofline": {"bound": "int-modmul", "achieved": modmuls / (t * 1e-3) / 1e9, "peak": peak_mm / 1e9,
                         "unit": "Gmodmul/s (256-bit Montgomery)", "frac": modmuls / (t * 1e-3) / peak_mm,
                         "peak_source": "nmsm_bench_modmul(field=256-bit), same run",
                         "hbm": {"achieved_gbs": alg_bytes / (t * 1e-3) / 1e9, "peak_gbs": peak,
                                 "frac": alg_bytes / (t * 1e-3) / 1e9 / peak, "algorithmic_bytes": alg_bytes}},
            "check": "inverse(direct(a)) == a bit-exact (natural and brp layouts)" if ok else "MISMATCH"}


def config0():
    P = R.CURVES["secp256k1"]
    rnd = random.Random(11)
    base = R.normalizeZ(P, [P.BASE.multiplyUnsafe(rnd.randrange(1, P.Fn.ORDER))])[0]
    ks = [rnd.randrange(1, P.Fn.ORDER) for _ in range(1024)]
    pb, sb = H.point_bytes("secp256k1", base) * 1024, H.pack_scalars(ks)
    res = {}

    def run():
        res["o"] = nmsm.mul_batch_packed(0, pb, sb, 1024, False)

    run()
    best = time_best(run, 5)
    t0 = time.perf_counter()
    ok = True
    for i in range(0, 1024, 64):  # CPU oracle (Python bigint restatement of the reference's blinded fixed-window path)
        ok &= H.unpack_point("secp256k1", res["o"][0][i * 64:(i + 1) * 64]) == R.affine_tuple(P, base.multiply(ks[i]))
    cpu_per = (time.perf_counter() - t0) / 16
    return {"config": 0, "what": "secp256k1 Point.multiply x 1024 random scalars", "n": 1024, "gpu_ms": best * 1e3,
            "multiplies_per_s_gpu": 1024 / best,
            "cpu_python_oracle_multiplies_per_s": 1 / cpu_per, "cpu_sample": "16 multiplies, Python-int oracle, 1 core",
            "check": "bit-exact on 16 sampled results" if ok else "MISMATCH"}


def config4():
    from conftest import load_golden

    vec = load_golden("ed25519.json")["vectors"]
    reps = (1 << 16) // len(vec)
    sigs = [bytes.fromhex(v["sig"]) for v in vec] * reps
    msgs = [bytes.fromhex(v["msg"]) for v in vec] * reps
    pks = [bytes.fromhex(v["pk"]) for v in vec] * reps
    z = os.urandom(16 * len(sigs))
    res = {}

    def run():
        res["r"] = nmsm.ed25519_verify_batch(sigs, msgs, pks, z)

    run()
    best = time_best(run, 3)
    t0 = time.perf_counter()
    for i in range(8):
        assert R.ed25519_verify(sigs[i], msgs[i], pks[i])
    cpu_per = (time.perf_counter() - t0) / 8
    return {"config": 4, "what": "ed25519 batch verification, 2^16 signatures (RFC 8032 vectors tiled)", "n": len(sigs),
            "gpu_ms_through_python_binding": best * 1e3, "signatures_per_s": len(sigs) / best,
            "cpu_python_oracle_verifies_per_s": 1 / cpu_per, "cpu_sample": "8 individual verifies, Python-int oracle, 1 core",
            "check": "accepted; equals AND of individual verifies" if res["r"] == (True, -1) else "MISMATCH"}


def main():
    nmsm.init(0)
    if "--fixed-base" in sys.argv:
        rows = (lambda: fixed_base_config("f4-a", "bls12_381_G1", 20), lambda: fixed_base_config("f4-b", "bls12_381_G1", 16),
                lambda: fixed_base_config("f4-c", "bls12_381_G2", 18), lambda: fixed_base_config("f4-d", "bn254_G1", 20),
                lambda: point_table_config("f4-e", "secp256k1", 20), lambda: point_table_config("f4-f", "ed25519", 20),
                lambda: point_table_config("f4-g", "bls12_381_G1", 18),
                lambda: ntt_config("f4-h", "bls12_381", 20), lambda: ntt_config("f4-i", "bls12_381", 24),
                lambda: ntt_config("f4-j", "bn254", 20))
    else:
        rows = (config0, lambda: msm_config(1, "bls12_381_G1", 16), lambda: msm_config(2, "bn254_G1", 20),
                lambda: msm_config(3, "bls12_381_G2", 18), config4)
    only = os.environ.get("NMSM_ROWS")  # e.g. NMSM_ROWS=0,2 : positions in the row list
    for i, row in enumerate(rows):
        if only and str(i) not in only.split(","):
            continue
        print(json.dumps(row()), flush=True)


if __name__ == "__main__":
    main()
