"""Shared test helpers: oracle-side input generation and byte packing for the C ABI formats.

Uses the CPU oracle (oracle/noble_ref.py) — allowed in tests only.
"""
import ctypes
import os
import subprocess

import numpy as np

from oracle import noble_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# "bls12_381_G1_any" / "bls12_381_G2_any" = NMSM_BLS12_381_G{1,2}_ANY: the same curve without the subgroup assumption
# (no endomorphism split)
CURVE_IDS = {"secp256k1": 0, "ed25519": 1, "bn254_G1": 2, "bn254_G2": 3, "bls12_381_G1": 4, "bls12_381_G2": 5,
             "bls12_381_G1_any": 6, "bls12_381_G2_any": 7}
FP_BYTES = {"secp256k1": 32, "ed25519": 32, "bn254_G1": 32, "bn254_G2": 32, "bls12_381_G1": 48, "bls12_381_G2": 48,
            "bls12_381_G1_any": 48, "bls12_381_G2_any": 48}
PARTS = {"secp256k1": 1, "ed25519": 1, "bn254_G1": 1, "bn254_G2": 2, "bls12_381_G1": 1, "bls12_381_G2": 2,
         "bls12_381_G1_any": 1, "bls12_381_G2_any": 2}


def bls_g1_non_subgroup_points(count, seed=3):
    """On-curve points of BLS12-381 E(Fp) that are NOT in the prime-order subgroup (cofactor part non-trivial):
    what isTorsionFree rejects (weierstrass.ts:951-969) and what an MSM over unvalidated points can contain."""
    import random

    P = R.CURVES["bls12_381_G1"]
    p, r = P.Fp.ORDER, P.Fn.ORDER
    rnd = random.Random(seed)
    out = []
    while len(out) < count:
        x = rnd.randrange(p)
        y2 = (x * x * x + 4) % p
        y = pow(y2, (p + 1) // 4, p)
        if y * y % p != y2:
            continue
        cand = P.fromAffine({"x": x, "y": y})
        if cand.multiplyUnsafe(r - 1).add(cand).is0():
            continue  # happens with probability 1/h
        out.append(cand)
    return out


def bls_g2_non_subgroup_points(count, seed=5):
    """On-curve points of the BLS12-381 twist E'(Fp2): y^2 = x^3 + 4(1 + u) outside the prime-order subgroup G2."""
    import random

    P = R.CURVES["bls12_381_G2"]
    Fp2 = P.Fp
    p, r = Fp2.Fp.ORDER, P.Fn.ORDER
    rnd = random.Random(seed)
    out = []
    while len(out) < count:
        x = (rnd.randrange(p), rnd.randrange(p))
        y2 = Fp2.add(Fp2.mul(Fp2.sqr(x), x), (4, 4))
        try:
            y = Fp2.sqrt(y2)
        except ValueError:
            continue
        cand = P.fromAffine({"x": x, "y": y})
        if cand.multiplyUnsafe(r - 1).add(cand).is0():
            continue
        out.append(cand)
    return out


# curve index in test/slow-curves.test.ts:186-194
SOAK_INDEX = {"secp256k1": 0, "ed25519": 2, "bls12_381_G1": 3, "bls12_381_G2": 4, "bn254_G1": 5, "bn254_G2": 6}


def coord_bytes(name, v) -> bytes:
    nb = FP_BYTES[name]
    if PARTS[name] == 1:
        return v.to_bytes(nb, "little")
    return v[0].to_bytes(nb, "little") + v[1].to_bytes(nb, "little")


def point_bytes(name, P) -> bytes:
    """Canonical affine packing of an oracle point (C ABI format, include/nmsm.h)."""
    a = P.toAffine()
    return coord_bytes(name, a["x"]) + coord_bytes(name, a["y"])


def pack_points(name, pts) -> bytes:
    return b"".join(point_bytes(name, p) for p in pts)


def pack_scalars(scalars) -> bytes:
    return b"".join(int(s).to_bytes(32, "little") for s in scalars)


def unpack_point(name, xy: bytes):
    nb = FP_BYTES[name]
    cb = nb * PARTS[name]

    def coord(b):
        if PARTS[name] == 1:
            return int.from_bytes(b[:nb], "little")
        return (int.from_bytes(b[:nb], "little"), int.from_bytes(b[nb:2 * nb], "little"))

    return coord(xy[:cb]), coord(xy[cb:2 * cb])


def expected_tuple(name, P):
    """(x, y, is_inf) of an oracle point in the output convention of the C ABI."""
    a = P.toAffine()
    return a["x"], a["y"], 1 if P.is0() else 0


def soak_inputs(name, n, zero_every=17, seed_offset=0):
    """Points (k0 + i*ks)*G and scalars per test/slow-curves.test.ts:199-222; returns expected total scalar."""
    P = R.CURVES[name]
    order = P.Fn.ORDER
    rng = R.Xorshift64(0x6D736D0000000000 + SOAK_INDEX[name] + seed_offset)
    start = rng.rndBelow(order - 1) + 1
    step = rng.rndBelow(order - 1) + 1
    step_point = P.BASE.multiplyUnsafe(step)
    pts, scalars = [], []
    point = P.BASE.multiplyUnsafe(start)
    ps = start
    total = 0
    for i in range(n):
        s = 0 if (zero_every and i % zero_every == 0) else rng.rndBelow(order)
        pts.append(point)
        scalars.append(s)
        total = (total + ps * s) % order
        point = point.add(step_point)
        ps = (ps + step) % order
    # normalise once so packing does not invert per point
    pts = R.normalizeZ(P, pts)
    return P, pts, scalars, total


def expected_from_total(P, total):
    return P.BASE.multiplyUnsafe(total) if total else P.ZERO


# ------------------------------------------------------------------------------------------
# host-emulation library (tests/hostemu): the device code compiled for the CPU
# ------------------------------------------------------------------------------------------
_emu = None


def hostemu():
    global _emu
    if _emu is not None:
        return _emu
    src = os.path.join(ROOT, "tests", "hostemu", "hostemu.cpp")
    so = os.path.join(ROOT, "tests", "hostemu", "libhostemu.so")
    csrc = os.path.join(ROOT, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


# ------------------------------------------------------------------------------------------
# device arithmetic harness (tests/devemu): the device headers' parts compiled for sm_90a and run one case per thread
# ------------------------------------------------------------------------------------------
_dev = None
# (source, object, extra flags): the field unit once with the product's out-of-line multiplications and once inlined
# (the Makefile's `make EXTRA=` build), whose entry points end in _inl
DEVEMU_UNITS = [("field.cu", "field.o", ["-DNMSM_MUL_NOINLINE"]), ("field.cu", "field_inl.o", []),
                ("tower.cu", "tower.o", ["-DNMSM_MUL_NOINLINE"]), ("group.cu", "group.o", ["-DNMSM_MUL_NOINLINE"])]


def _nvcc():
    import shutil

    return shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")


def devemu():
    """ctypes handle of tests/devemu/libdevemu.so, (re)built with nvcc for sm_90a when a source or header is newer.  The
    translation units compile in parallel; ptxas reports (-Xptxas -v) go to tests/devemu/build/*.log."""
    global _dev
    if _dev is not None:
        return _dev
    d = os.path.join(ROOT, "tests", "devemu")
    so = os.path.join(d, "libdevemu.so")
    csrc = os.path.join(ROOT, "noble-curves_b200", "csrc")
    deps = [os.path.join(d, f) for f in os.listdir(d) if f.endswith((".cu", ".cuh"))]
    deps += [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(so) or any(os.path.getmtime(x) > os.path.getmtime(so) for x in deps):
        bdir = os.path.join(d, "build")
        os.makedirs(bdir, exist_ok=True)
        nvcc = _nvcc()
        flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
                 "-I", csrc]
        procs = []
        for src, obj, extra in DEVEMU_UNITS:
            log = open(os.path.join(bdir, obj[:-2] + ".log"), "w")
            cmd = [nvcc] + flags + extra + ["-c", os.path.join(d, src), "-o", os.path.join(bdir, obj)]
            procs.append((subprocess.Popen(cmd, stdout=log, stderr=subprocess.STDOUT), log, obj))
        failed = []
        for proc, log, obj in procs:
            if proc.wait() != 0:
                failed.append(obj)
            log.close()
        if failed:
            msgs = [open(os.path.join(bdir, o[:-2] + ".log")).read()[-4000:] for o in failed]
            raise RuntimeError("devemu build failed: %s\n%s" % (failed, "\n".join(msgs)))
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", so]
                              + [os.path.join(bdir, obj) for _, obj, _ in DEVEMU_UNITS])
    _dev = ctypes.CDLL(so)
    return _dev


def u32(b: bytes):
    return np.frombuffer(b, dtype=np.uint32).copy()


def emu_msm(name, pts_b: bytes, scalars_b: bytes, n: int, forced_c=0, forced_L=0, table_c=0, groups=1):
    """table_c != 0: the fixed-base table route (levels 2^(c*j)*P, one bucket window).  groups: window groups the
    pipeline is split into (engine.cuh submit_msm), top windows first."""
    lib = hostemu()
    cb = FP_BYTES[name] * PARTS[name]
    pts = u32(pts_b) if n else np.zeros(4, np.uint32)
    sc = u32(scalars_b) if n else np.zeros(8, np.uint32)
    out = np.zeros(2 * cb // 4, np.uint32)
    inf = np.zeros(1, np.uint32)
    err = np.zeros(2, np.uint32)
    plan = np.zeros(4, np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    if table_c:
        rc = lib.emu_msm_table(CURVE_IDS[name], p(pts), p(sc), n, table_c, forced_L, p(out), p(inf), p(err), p(plan))
    elif groups != 1:
        rc = lib.emu_msm_groups(CURVE_IDS[name], p(pts), p(sc), n, forced_c, forced_L, groups, p(out), p(inf), p(err), p(plan))
    else:
        rc = lib.emu_msm(CURVE_IDS[name], p(pts), p(sc), n, forced_c, forced_L, p(out), p(inf), p(err), p(plan))
    assert rc == 0, rc
    x, y = unpack_point(name, out.tobytes())
    return (x, y, int(inf[0])), (int(err[0]), int(err[1])), tuple(int(v) for v in plan)


def emu_point_table(name, point_b: bytes, scalars_b: bytes, n: int, allow_zero: bool, table_bits=8):
    """nmsm_point_table_* bodies with a table_bits-wide table; returns ([(x, y, inf) or None if rejected], err)."""
    lib = hostemu()
    cb = FP_BYTES[name] * PARTS[name]
    pt, sc = u32(point_b), u32(scalars_b)
    out = np.zeros(n * 2 * cb // 4, np.uint32)
    inf = np.zeros(n, np.uint32)
    err = np.zeros(2, np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = lib.emu_point_table(CURVE_IDS[name], table_bits, p(pt), p(sc), n, 1 if allow_zero else 0, p(out), p(inf), p(err))
    assert rc == 0
    ob = out.tobytes()
    res = []
    for i in range(n):
        if inf[i] == 9:
            res.append(None)
        else:
            x, y = unpack_point(name, ob[i * 2 * cb:(i + 1) * 2 * cb])
            res.append((x, y, int(inf[i])))
    return res, (int(err[0]), int(err[1]))


def emu_torsion(name, pts_b: bytes, n: int):
    lib = hostemu()
    pts = u32(pts_b)
    ok = np.zeros(n, np.uint8)
    err = np.zeros(2, np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    assert lib.emu_torsion(CURVE_IDS[name], p(pts), n, p(ok), p(err)) == 0
    return [int(v) for v in ok], (int(err[0]), int(err[1]))


def emu_mul_batch(name, pts_b: bytes, scalars_b: bytes, n: int, allow_zero: bool):
    lib = hostemu()
    cb = FP_BYTES[name] * PARTS[name]
    pts, sc = u32(pts_b), u32(scalars_b)
    out = np.zeros(n * 2 * cb // 4, np.uint32)
    inf = np.zeros(n, np.uint32)
    err = np.zeros(2, np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = lib.emu_mul_batch(CURVE_IDS[name], p(pts), p(sc), n, 1 if allow_zero else 0, p(out), p(inf), p(err))
    assert rc == 0
    ob = out.tobytes()
    res = []
    for i in range(n):
        x, y = unpack_point(name, ob[i * 2 * cb:(i + 1) * 2 * cb])
        res.append((x, y, int(inf[i])))
    return res, (int(err[0]), int(err[1]))
