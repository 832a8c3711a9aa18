"""ECDSA verification for NIST P-256 (secp256r1): the oracle nmsm_p256_verify_batch is checked against, and Ethereum's
P256VERIFY precompile (EIP-7951, RIP-7212) stated from the EIP.

Restates noble-curves v2 `p256.verify(signature, message, publicKey, {prehash, lowS})` (nist.ts over weierstrass.ts
`ecdsa().verify`) with format 'compact', on noble_ref's Weierstrass arithmetic, which handles a != 0 with noble's
complete formulas.  Test infrastructure only.
"""
from __future__ import annotations

import hashlib

from .ecdsa_ref import SECP256K1_MAX_RAW_MSG
from .noble_ref import Field, weierstrass

# NIST P-256 / secp256r1 (noble-curves src/nist.ts p256; SEC 2 v2 §2.4.2, FIPS 186-5): a = -3
P256_CURVE = dict(
    p=0xFFFFFFFF00000001000000000000000000000000FFFFFFFFFFFFFFFFFFFFFFFF,
    n=0xFFFFFFFF00000000FFFFFFFFFFFFFFFFBCE6FAADA7179E84F3B9CAC2FC632551,
    h=1,
    a=0xFFFFFFFF00000001000000000000000000000000FFFFFFFFFFFFFFFFFFFFFFFC,
    b=0x5AC635D8AA3A93E7B3EBBD55769886BC651D06B0CC53B0F63BCE3C3E27D2604B,
    Gx=0x6B17D1F2E12C4247F8BCE6E563A440F277037D812DEB33A0F4A13945D898C296,
    Gy=0x4FE342E2FE1A7F9B8EE7EB4A7C0F9E162BCE33576B315ECECBB6406837BF51F5,
)
# the Point class of p256 (no endomorphism); base-point window W = 6 as weierstrass.ts:1018
P256 = weierstrass(P256_CURVE, Field(P256_CURVE["p"]), Field(P256_CURVE["n"]))
P256.wnaf.setWindowSize(P256.BASE, 6)


def p256_decode_sec1(b: bytes):
    """weierstrass.ts `pointFromBytes` for P-256 -> (x, y); raises ValueError.  y^2 = x^3 - 3x + b."""
    P, A, B = P256_CURVE["p"], P256_CURVE["a"], P256_CURVE["b"]
    head, tail = b[0], b[1:]
    if len(b) == 33 and head in (2, 3):
        x = int.from_bytes(tail, "big")
        if not (0 <= x < P):
            raise ValueError("bad point: is not on curve, wrong x")
        y2 = (x * x * x + A * x + B) % P
        y = pow(y2, (P + 1) // 4, P)  # p = 3 mod 4
        if (y * y) % P != y2:
            raise ValueError("bad point: is not on curve, sqrt error")
        if ((head & 1) == 1) != ((y & 1) == 1):
            y = (-y) % P
        return x, y
    if len(b) == 65 and head == 4:
        x, y = int.from_bytes(tail[:32], "big"), int.from_bytes(tail[32:], "big")
        if not (0 <= x < P and 0 <= y < P) or (y * y - x * x * x - A * x - B) % P:
            raise ValueError("bad point: is not on curve")
        return x, y
    raise ValueError("bad point: got length %d" % len(b))


def p256_ecdsa_verify(sig: bytes, msg: bytes, pk: bytes, prehash: bool = True, lowS: bool = False) -> bool:
    """p256.verify (noble-curves nist.ts), the rules of secp256k1_ecdsa_verify on P-256.  noble creates p256 with
    lowS: false, so that is the default here (OpenSSL does not test s either)."""
    if not all(isinstance(b, (bytes, bytearray)) for b in (sig, msg, pk)):
        raise TypeError("Uint8Array expected")
    if len(sig) != 64:
        raise ValueError("compact signature expected 64 bytes")
    Pt = P256
    N = P256_CURVE["n"]
    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
    if not (1 <= r < N and 1 <= s < N):  # Signature constructor: aInRange('r'/'s', 1, n)
        return False
    try:
        x, y = p256_decode_sec1(bytes(pk))  # Point.fromBytes
    except (ValueError, IndexError):
        return False
    Q = Pt.fromAffine({"x": x, "y": y})
    if lowS and s > (N >> 1):  # hasHighS
        return False
    m = hashlib.sha256(bytes(msg)).digest() if prehash else bytes(msg)
    if len(m) > SECP256K1_MAX_RAW_MSG:  # bits2int throws; the bound is the same on every curve
        return False
    h = int.from_bytes(m, "big")
    delta = len(m) * 8 - 256
    if delta > 0:
        h >>= delta
    h %= N  # bits2int_modN
    w = pow(s, -1, N)
    u1, u2 = (h * w) % N, (r * w) % N
    R = Pt.BASE.multiplyUnsafe(u1).add(Q.multiplyUnsafe(u2))
    if R.is0():
        return False
    return R.toAffine()["x"] % N == r


def p256verify_precompile(inp: bytes) -> bool:
    """Ethereum's P256VERIFY precompile (EIP-7951; RIP-7212 on rollups), stated from the EIP: True iff it returns the
    32-byte word 1, False iff it returns empty output.  input = h || r || s || qx || qy, 32 bytes each, big-endian."""
    P, N, A, B = P256_CURVE["p"], P256_CURVE["n"], P256_CURVE["a"], P256_CURVE["b"]
    if len(inp) != 160:
        return False
    h, r, s, qx, qy = (int.from_bytes(inp[32 * k:32 * (k + 1)], "big") for k in range(5))
    if not (0 < r < N and 0 < s < N):
        return False
    if not (0 <= qx < P and 0 <= qy < P):
        return False
    if (qx, qy) == (0, 0) or (qy * qy - qx * qx * qx - A * qx - B) % P:  # Q on the curve, not the point at infinity
        return False
    Pt = P256
    Q = Pt.fromAffine({"x": qx, "y": qy})
    si = pow(s, -1, N)
    u1, u2 = h * si % N, r * si % N  # the hash is used as given, modulo n
    R = Pt.BASE.multiplyUnsafe(u1).add(Q.multiplyUnsafe(u2))
    if R.is0():
        return False
    return R.toAffine()["x"] % N == r
