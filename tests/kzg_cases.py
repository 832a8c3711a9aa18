"""EIP-4844 KZG inputs shared by the CPU (hostemu) and GPU tests: a seeded tau and its setup point, seeded blobs with
honest commitments and proofs from the oracle's test prover, honest point-evaluation items, the corruptions, tiling
helpers, and the host build of the device bodies (tests/hostemu/kzg_emu.cpp)."""
import ctypes
import hashlib
import os
import random
import subprocess

from oracle import hash_to_g1_ref as H
from oracle import kzg_ref as K

R = K.BLS_MODULUS
TAU = random.Random(4844).randrange(2, R)
SETUP = K.setup_g2(TAU)
OTHER_SETUP = K.setup_g2(TAU + 1)
ZERO_BLOB = bytes(K.BYTES_PER_BLOB)
IDENTITY = K.G1_POINT_AT_INFINITY


def be(v: int) -> bytes:
    return v.to_bytes(32, "big")


def random_blob(seed: int) -> bytes:
    rnd = random.Random(seed)
    return b"".join(be(rnd.randrange(R)) for _ in range(K.FIELD_ELEMENTS_PER_BLOB))


def blob_with(blob: bytes, index: int, value: int) -> bytes:
    return blob[:32 * index] + be(value) + blob[32 * index + 32:]


_BLOB_MEMO = {}


def blob_item(seed: int):
    """(blob, commitment, proof, z, y) for a seeded random blob under TAU"""
    if seed not in _BLOB_MEMO:
        blob = random_blob(seed)
        _BLOB_MEMO[seed] = (blob,) + K.blob_commit_and_prove(blob, TAU)
    return _BLOB_MEMO[seed]


def proof_item(rnd):
    """(commitment, z, y, proof) of a random polynomial value f(tau) opened at a random z"""
    f_tau, z = rnd.randrange(R), rnd.randrange(R)
    y = rnd.randrange(R)
    return K.commit_value(f_tau), z, y, K.prove_value(f_tau, z, y, TAU)


def proof_items(count: int, distinct: int = 32, seed: int = 1):
    """count honest (commitment, z, y, proof) items: `distinct` of them tiled"""
    rnd = random.Random(seed)
    base = [proof_item(rnd) for _ in range(min(count, distinct))]
    return [base[k % len(base)] for k in range(count)]


def versioned_hash(commitment: bytes) -> bytes:
    return K.kzg_to_versioned_hash(commitment)


def precompile_input(item) -> bytes:
    c, z, y, pi = item
    return versioned_hash(c) + be(z) + be(y) + c + pi


def pack_proofs(items):
    cs, zs, ys, pis = zip(*items)
    return b"".join(cs), b"".join(be(z) for z in zs), b"".join(be(y) for y in ys), b"".join(pis)


# ---- corrupted encodings ----------------------------------------------------------------------------------------
def off_curve_g1() -> bytes:
    """a compressed encoding whose x has no y on E1"""
    x = 1
    while H.sqrt((x ** 3 + 4) % H.P) is not None:
        x += 1
    b = bytearray(x.to_bytes(48, "big"))
    b[0] |= 0x80
    return bytes(b)


def small_order_g1() -> bytes:
    """(0, 2): a point of order 3 on E1, outside G1"""
    b = bytearray(48)
    b[0] = 0x80
    return bytes(b)


NON_CANONICAL_IDENTITY = b"\xc0" + bytes(46) + b"\x01"


def uncompressed_flag(enc: bytes) -> bytes:
    return bytes([enc[0] & 0x7F]) + enc[1:]


# ---- host build of the device bodies (tests/hostemu/kzg_emu.cpp) ----------------------------------------------------
_emu = None


def kzg_emu():
    """ctypes handle of tests/hostemu/libkzgemu.so, (re)built with g++ when the source or a device header is newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "kzg_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libkzgemu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def emu_challenge(blobs, commitments):
    n = len(blobs)
    out = ctypes.create_string_buffer(32 * n)
    assert kzg_emu().emu_kzg_challenge(b"".join(blobs), b"".join(commitments), n, out) == 0
    return [int.from_bytes(out.raw[32 * k:32 * k + 32], "big") for k in range(n)]


def emu_roots():
    out = (ctypes.c_uint32 * (8 * K.FIELD_ELEMENTS_PER_BLOB))()
    assert kzg_emu().emu_kzg_roots(out) == 0
    raw = bytes(out)
    return [int.from_bytes(raw[32 * i:32 * i + 32], "little") for i in range(K.FIELD_ELEMENTS_PER_BLOB)]


def emu_eval(blobs, zs):
    """[(y, ok)] of the eval body for each blob at its z"""
    n = len(blobs)
    ys, ok = ctypes.create_string_buffer(32 * n), ctypes.create_string_buffer(n)
    assert kzg_emu().emu_kzg_eval(b"".join(blobs), b"".join(be(z) for z in zs), n, ys, ok) == 0
    return [(int.from_bytes(ys.raw[32 * k:32 * k + 32], "big"), ok.raw[k] == 1) for k in range(n)]


def emu_fr_inv(a: int) -> int:
    out = ctypes.create_string_buffer(32)
    kzg_emu().emu_fr_inv(a.to_bytes(32, "little"), out)
    return int.from_bytes(out.raw, "little")


def emu_prepare(items, setup=SETUP, vhs=None):
    """(pairs, pre_ok) from the prepare body: pairs[i] = ((Q, pi) as G1 packings, (-G2, setup) as G2 packings)"""
    n = len(items)
    c, z, y, pi = pack_proofs(items)
    g1 = ctypes.create_string_buffer(192 * n)
    g2 = ctypes.create_string_buffer(384 * n)
    pre = ctypes.create_string_buffer(n)
    rc = kzg_emu().emu_kzg_prepare(c, z, y, pi, b"".join(vhs) if vhs is not None else None, None, n, setup, g1, g2,
                                   pre)
    assert rc == 0
    return [(g1.raw[192 * k:192 * k + 192], g2.raw[384 * k:384 * k + 384]) for k in range(n)], list(pre.raw)


def emu_verify(items, setup=SETUP, vhs=None):
    """serial verdicts of the whole proof check (prepare, Miller loops, final exponentiations)"""
    n = len(items)
    c, z, y, pi = pack_proofs(items)
    out = ctypes.create_string_buffer(n)
    rc = kzg_emu().emu_kzg_verify(c, z, y, pi, b"".join(vhs) if vhs is not None else None, n, setup, out)
    assert rc == 0, rc
    return [b == 1 for b in out.raw]


def sha256(b: bytes) -> bytes:
    return hashlib.sha256(b).digest()
