"""CPU ORACLE (test infrastructure only) — builds/loads the C restatement (oracle/ref_msm.c) and times it.

Used by tests/, __graft_entry__ (build + smoke) and bench.py's cpu_baseline / `--impl reference` legs only.
The reference itself (TypeScript on Node) cannot run in this image, so `kind` is "port": the reference's
algorithm (curve.ts:863-905 + weierstrass.ts:793-880) restated in C, pinned to oracle/noble_ref.py which is
pinned to the reference's golden vectors.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile
import time

from . import noble_ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ref_msm.c")
_SO = os.path.join(_HERE, "_build", "libref_msm.so")
_lib = None


def build(force: bool = False) -> str:
    if not force and os.path.exists(_SO) and os.path.getmtime(_SO) >= os.path.getmtime(_SRC):
        return _SO
    so = _SO
    try:
        os.makedirs(os.path.dirname(so), exist_ok=True)
        writable = os.access(os.path.dirname(so), os.W_OK)
    except OSError:
        writable = False
    if not writable:  # read-only tree (e.g. bench.py after build()): compile into a temporary directory instead
        so = os.path.join(tempfile.mkdtemp(prefix="nmsm_ref_msm_"), "libref_msm.so")
    subprocess.check_call(["gcc", "-O3", "-march=native", "-shared", "-fPIC", "-pthread", _SRC, "-o", so])
    return so


def load():
    global _lib
    if _lib is None:
        lib = ctypes.CDLL(build())
        lib.ref_pippenger_bls12_381_g1.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_int,
                                                   ctypes.c_void_p]
        lib.ref_pippenger_bls12_381_g1.restype = ctypes.c_int
        lib.ref_make_points_bls12_381_g1.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p]
        lib.ref_make_points_bls12_381_g1.restype = None
        lib.ref_pippenger_add_count.argtypes = [ctypes.c_uint64, ctypes.c_int]
        lib.ref_pippenger_add_count.restype = ctypes.c_uint64
        _lib = lib
    return _lib


def host_threads() -> int:
    try:
        return len(os.sched_getaffinity(0))
    except AttributeError:
        return os.cpu_count() or 1


def c_pippenger_bls_g1(pts: bytes, scalars: bytes, n: int, threads: int = 1):
    """(x, y, is_inf) of the reference algorithm's result; inputs in the C-ABI packing (include/nmsm.h)."""
    lib = load()
    out = ctypes.create_string_buffer(96)
    pb = ctypes.create_string_buffer(pts, len(pts)) if n else None
    sb = ctypes.create_string_buffer(scalars, len(scalars)) if n else None
    inf = lib.ref_pippenger_bls12_381_g1(pb, sb, n, threads, out)
    return int.from_bytes(out.raw[:48], "little"), int.from_bytes(out.raw[48:], "little"), inf


def make_points_bls_g1(n: int, seed: int):
    """P_i = (k0 + i*ks)*G (test/slow-curves.test.ts:204-222); returns (packed points, k0, ks)."""
    P = R.CURVES["bls12_381_G1"]
    rng = R.Xorshift64(0x6D736D0000000000 + 3 + seed)
    k0 = rng.rndBelow(P.Fn.ORDER - 1) + 1
    ks = rng.rndBelow(P.Fn.ORDER - 1) + 1

    def aff(k):
        a = P.BASE.multiplyUnsafe(k).toAffine()
        return a["x"].to_bytes(48, "little") + a["y"].to_bytes(48, "little")

    out = ctypes.create_string_buffer(96 * n)
    load().ref_make_points_bls12_381_g1(ctypes.create_string_buffer(aff(k0), 96), ctypes.create_string_buffer(aff(ks), 96), n, out)
    return out.raw, k0, ks


def random_scalars(n: int, seed: int):
    import random

    rnd = random.Random(seed)
    order = R.CURVES["bls12_381_G1"].Fn.ORDER
    return [rnd.randrange(order) for _ in range(n)]


class Workload:
    """Inputs of one timed CPU run: generated once, then `run()` is the timed region."""

    def __init__(self, n: int, seed: int = 1):
        self.n = n
        self.threads = host_threads()
        self.pts, k0, ks = make_points_bls_g1(n, seed)
        sc = random_scalars(n, seed)
        self.sb = b"".join(s.to_bytes(32, "little") for s in sc)
        order = R.CURVES["bls12_381_G1"].Fn.ORDER
        tot, kk = 0, k0
        for s in sc:
            tot = (tot + kk * s) % order
            kk = (kk + ks) % order
        exp = R.CURVES["bls12_381_G1"].BASE.multiplyUnsafe(tot).toAffine() if tot else {"x": 0, "y": 0}
        self.expected = (exp["x"], exp["y"])

    def run(self) -> float:
        t0 = time.perf_counter()
        x, y, inf = c_pippenger_bls_g1(self.pts, self.sb, self.n, self.threads)
        dt = time.perf_counter() - t0
        assert (x, y) == self.expected, "C reference port produced a wrong MSM result"
        return dt


def choose_sample(max_seconds: float = 30.0, full_log2: int = 20) -> int:
    """Full 2^full_log2 workload when a 2^13 calibration run predicts it fits the budget, else 2^16."""
    lib = load()
    w = Workload(1 << 13, 7)
    tcal = w.run()
    adds_cal = lib.ref_pippenger_add_count(1 << 13, 255)
    adds_full = lib.ref_pippenger_add_count(1 << full_log2, 255)
    return (1 << full_log2) if tcal * adds_full / adds_cal <= max_seconds / 3 else (1 << 16)


def describe(n_sample: int, dt: float, full_log2: int = 20):
    """points/s at the full size + the `cpu_baseline` fields for a run of `dt` seconds on n_sample terms."""
    lib = load()
    full = 1 << full_log2
    adds_full = lib.ref_pippenger_add_count(full, 255)
    adds_sample = lib.ref_pippenger_add_count(n_sample, 255)
    threads = host_threads()
    windows = 15 if n_sample == full else ((255 - 1) // max(1, (n_sample.bit_length() - 3))) + 1
    if n_sample == full:
        pps = full / dt
        sample = "full workload: one 2^%d-term MSM, %.2f s, %d point adds" % (full_log2, dt, adds_full)
    else:
        pps = full / (dt * adds_full / adds_sample)
        sample = ("2^%d-term MSM (%.2f s, %d adds), EXTRAPOLATED to 2^%d by the exact add-count ratio %d/%d"
                  % (n_sample.bit_length() - 1, dt, adds_sample, full_log2, adds_full, adds_sample))
    return {"points_per_s_at_full_size": pps, "cores": min(threads, windows), "kind": "port",
            "sample": sample + "; C port of curve.ts:863-905 (oracle/ref_msm.c), windows spread over host threads",
            "seconds": dt, "n": n_sample}


def time_bls_g1_msm(n_sample, seed: int = 1, max_seconds: float = 30.0, full_log2: int = 20):
    """One-shot helper: pick the sample, build inputs, time one run."""
    if n_sample is None:
        n_sample = choose_sample(max_seconds, full_log2)
    w = Workload(n_sample, seed)
    return describe(n_sample, w.run(), full_log2)
