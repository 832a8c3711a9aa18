"""ECDSA verification for secp256k1 (next-row f5): the oracle nmsm_secp256k1_verify_batch is checked against.

Restates noble-curves v2 weierstrass.ts `ecdsa().verify(signature, message, publicKey, {prehash, lowS})` with format
'compact' on top of noble_ref's secp256k1 arithmetic and SEC1 decoder.  Test infrastructure only.
"""
from __future__ import annotations

import hashlib

from .noble_ref import CURVES, SECP256K1_CURVE, secp256k1_decode_sec1

SECP256K1_MAX_RAW_MSG = 8192  # weierstrass.ts bits2int: "input is too large"


def secp256k1_ecdsa_verify(sig: bytes, msg: bytes, pk: bytes, prehash: bool = True, lowS: bool = True) -> bool:
    """A signature that is not 64 bytes (or non-bytes arguments) throws before the reference's `try`; inside it every
    failure is a False verdict."""
    if not all(isinstance(b, (bytes, bytearray)) for b in (sig, msg, pk)):
        raise TypeError("Uint8Array expected")
    if len(sig) != 64:
        raise ValueError("compact signature expected 64 bytes")
    Pt = CURVES["secp256k1"]
    N = SECP256K1_CURVE["n"]
    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
    if not (1 <= r < N and 1 <= s < N):  # Signature constructor: aInRange('r'/'s', 1, n)
        return False
    try:
        x, y = secp256k1_decode_sec1(bytes(pk))  # Point.fromBytes
    except (ValueError, IndexError):
        return False
    Q = Pt.fromAffine({"x": x, "y": y})
    if lowS and s > (N >> 1):  # hasHighS
        return False
    m = hashlib.sha256(bytes(msg)).digest() if prehash else bytes(msg)
    if len(m) > SECP256K1_MAX_RAW_MSG:  # bits2int throws
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
