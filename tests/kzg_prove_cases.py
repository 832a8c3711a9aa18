"""EIP-4844 prover inputs shared by the CPU (hostemu) and GPU tests: the z cases of compute_kzg_proof, the expected
values from the oracle's scalar prover, and the host build of the prover bodies (tests/hostemu/kzg_prove_emu.cpp).
The seeded tau, blobs and corruptions are kzg_cases'."""
import ctypes
import os
import random
import subprocess

import kzg_cases as C
from oracle import hash_to_g1_ref as H
from oracle import kzg_ref as K
import kzg_prove_ref as KP

R = K.BLS_MODULUS
BRP = K.BRP_ROOTS_OF_UNITY
DOMAIN_INDICES = (0, 1, 2048, 4095)


def z_cases(seed: int = 1):
    """(name, z): random z, z on the bit-reversed domain at DOMAIN_INDICES, and z = 0"""
    rnd = random.Random(seed)
    return ([("random%d" % k, rnd.randrange(R)) for k in range(2)] + [("brp%d" % k, BRP[k]) for k in DOMAIN_INDICES]
            + [("zero", 0)])


def f_tau(blob: bytes, tau: int = C.TAU) -> int:
    return K.evaluate_polynomial_in_evaluation_form(K.blob_to_polynomial(blob), tau)


def expected_proof(blob: bytes, z: int, tau: int = C.TAU):
    """(proof, y) of compute_kzg_proof by the oracle's scalar prover: [(f(tau) - y) / (tau - z)] G1"""
    y = K.evaluate_polynomial_in_evaluation_form(K.blob_to_polynomial(blob), z)
    return K.prove_value(f_tau(blob, tau), z, y, tau), y


def lincomb_scalar(values, setup_scalars) -> int:
    """sum_i values[i] L_brp(i)(tau): the discrete log of g1_lincomb(bit_reversal_permutation(setup), values)"""
    return sum(v * s for v, s in zip(values, KP.bit_reversal_permutation(setup_scalars))) % R


# ---- host build of the prover bodies (tests/hostemu/kzg_prove_emu.cpp) ----------------------------------------------
_emu = None


def emu():
    """ctypes handle of tests/hostemu/libkzgproveemu.so, (re)built with g++ when the source or a device header is
    newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "kzg_prove_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libkzgproveemu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def emu_quotient(blob: bytes, z: int, y: int):
    """(q as ints, ok) of the quotient body for one blob evaluated at z with value y"""
    buf = ctypes.create_string_buffer(blob, len(blob))
    ok = ctypes.create_string_buffer(b"\x01", 1)
    assert emu().emu_kzg_quotient(buf, C.be(z), C.be(y), 1, ok) == 0
    raw = buf.raw
    return [int.from_bytes(raw[32 * i:32 * i + 32], "big") for i in range(K.FIELD_ELEMENTS_PER_BLOB)], ok.raw[0] == 1


def emu_compress(points):
    """kzg_g1_compress of affine points (None: the identity)"""
    n = len(points)
    xy = b"".join(H.g1_packed(p) if p is not None else bytes(96) for p in points)
    inf = bytes(1 if p is None else 0 for p in points)
    out = ctypes.create_string_buffer(48 * n)
    assert emu().emu_g1_compress(xy, inf, n, out) == 0
    return [out.raw[48 * i:48 * i + 48] for i in range(n)]


def emu_lincomb(points48, rows, lanes: int):
    """[(commitment, ok)] of the comb body over compressed points (table order) for each row of scalars"""
    npts, n = len(points48), len(rows)
    scalars = b"".join(C.be(s) for row in rows for s in row)
    out, ok = ctypes.create_string_buffer(48 * n), ctypes.create_string_buffer(n)
    assert emu().emu_kzg_lincomb(b"".join(points48), npts, scalars, n, lanes, out, ok) == 0
    return [(out.raw[48 * i:48 * i + 48], ok.raw[i] == 1) for i in range(n)]
