"""ECDSA verification for NIST P-384 (secp384r1): the oracle nmsm_p384_verify_batch is checked against.

Restates noble-curves v2 `p384.verify(signature, message, publicKey, {prehash, lowS})` (nist.ts over weierstrass.ts
`ecdsa().verify`) with format 'compact', on noble_ref's Weierstrass arithmetic (a = -3 with noble's complete
formulas), in plain integers.  noble's p384 hashes with SHA-384 and is created with lowS: false.  Test infrastructure
only.
"""
from __future__ import annotations

import hashlib

from .ecdsa_ref import SECP256K1_MAX_RAW_MSG
from .noble_ref import Field, weierstrass

# NIST P-384 / secp384r1 (noble-curves src/nist.ts p384; SEC 2 v2 §2.5.1, FIPS 186-5): a = -3
P384_CURVE = dict(
    p=2**384 - 2**128 - 2**96 + 2**32 - 1,
    n=0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFC7634D81F4372DDF581A0DB248B0A77AECEC196ACCC52973,
    h=1,
    a=2**384 - 2**128 - 2**96 + 2**32 - 1 - 3,
    b=0xB3312FA7E23EE7E4988E056BE3F82D19181D9C6EFE8141120314088F5013875AC656398D8A2ED19D2A85C8EDD3EC2AEF,
    Gx=0xAA87CA22BE8B05378EB1C71EF320AD746E1D3B628BA79B9859F741E082542A385502F25DBF55296C3A545E3872760AB7,
    Gy=0x3617DE4A96262C6F5D9E98BF9292DC29F8F41DBD289A147CE9DA3113B5F0B8C00A60B1CE1D7E819D7A431D7C90EA0E5F,
)
FIELD_BYTES = 48  # p, n and the signature halves
# the Point class of p384 (no endomorphism); base-point window W = 6 as weierstrass.ts:1018
P384 = weierstrass(P384_CURVE, Field(P384_CURVE["p"]), Field(P384_CURVE["n"]))
P384.wnaf.setWindowSize(P384.BASE, 6)


def p384_decode_sec1(b: bytes):
    """weierstrass.ts `pointFromBytes` for P-384 -> (x, y); raises ValueError.  49-byte 02/03 || x, or 97-byte
    04 || x || y; y^2 = x^3 - 3x + b."""
    P, A, B = P384_CURVE["p"], P384_CURVE["a"], P384_CURVE["b"]
    head, tail = b[0], b[1:]
    if len(b) == 1 + FIELD_BYTES and head in (2, 3):
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
    if len(b) == 1 + 2 * FIELD_BYTES and head == 4:
        x, y = int.from_bytes(tail[:FIELD_BYTES], "big"), int.from_bytes(tail[FIELD_BYTES:], "big")
        if not (0 <= x < P and 0 <= y < P) or (y * y - x * x * x - A * x - B) % P:
            raise ValueError("bad point: is not on curve")
        return x, y
    raise ValueError("bad point: got length %d" % len(b))


def bits2int_modn(m: bytes) -> int:
    """bits2int_modN for P-384: the big-endian integer of the first min(len, 48) bytes, mod n (nBitLength = 384)."""
    h = int.from_bytes(m, "big")
    delta = len(m) * 8 - 384
    if delta > 0:
        h >>= delta
    return h % P384_CURVE["n"]


def p384_ecdsa_verify(sig: bytes, msg: bytes, pk: bytes, prehash: bool = True, lowS: bool = False) -> bool:
    """p384.verify (noble-curves nist.ts), the rules of p256_ecdsa_verify at 48-byte width with SHA-384 as the prehash.
    noble creates p384 with lowS: false, so that is the default here (OpenSSL does not test s either)."""
    if not all(isinstance(b, (bytes, bytearray)) for b in (sig, msg, pk)):
        raise TypeError("Uint8Array expected")
    if len(sig) != 2 * FIELD_BYTES:
        raise ValueError("compact signature expected 96 bytes")
    Pt = P384
    N = P384_CURVE["n"]
    r, s = int.from_bytes(sig[:FIELD_BYTES], "big"), int.from_bytes(sig[FIELD_BYTES:], "big")
    if not (1 <= r < N and 1 <= s < N):  # Signature constructor: aInRange('r'/'s', 1, n)
        return False
    try:
        x, y = p384_decode_sec1(bytes(pk))  # Point.fromBytes
    except (ValueError, IndexError):
        return False
    Q = Pt.fromAffine({"x": x, "y": y})
    if lowS and s > (N >> 1):  # hasHighS
        return False
    m = hashlib.sha384(bytes(msg)).digest() if prehash else bytes(msg)
    if len(m) > SECP256K1_MAX_RAW_MSG:  # bits2int throws; the bound is the same on every curve
        return False
    h = bits2int_modn(m)
    w = pow(s, -1, N)
    u1, u2 = (h * w) % N, (r * w) % N
    R = Pt.BASE.multiplyUnsafe(u1).add(Q.multiplyUnsafe(u2))
    if R.is0():
        return False
    return R.toAffine()["x"] % N == r
