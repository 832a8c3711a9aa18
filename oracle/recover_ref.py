"""secp256k1 ECDSA public-key recovery and Ethereum's ecrecover (next-row f9): the oracle nmsm_secp256k1_recover_batch
and nmsm_secp256k1_ecrecover_batch are checked against.

Restates noble-curves v2 weierstrass.ts `Signature.recoverPublicKey` (reached through
secp256k1.recoverPublicKey(signature, message, {prehash}) with the 65-byte 'recovered' format rec || r || s) on top of
noble_ref's secp256k1 arithmetic and SEC1 decoder, and the ECREC precompile of the Yellow Paper (appendix E).  Where
the reference throws, this returns None (recovery) or b"" (ecrecover).  Test infrastructure only.
"""
from __future__ import annotations

import hashlib

from .ecdsa_ref import SECP256K1_MAX_RAW_MSG
from .keccak_ref import keccak256
from .noble_ref import CURVES, SECP256K1_CURVE, secp256k1_decode_sec1

N = SECP256K1_CURVE["n"]
P = SECP256K1_CURVE["p"]


def secp256k1_recover_public_key(sig65: bytes, msg: bytes, prehash: bool = True):
    """The recovered key as affine (x, y), or None where the reference throws inside recovery.  Non-bytes arguments
    and a signature that is not 65 bytes raise, as they do before the reference's parsing."""
    if not all(isinstance(b, (bytes, bytearray)) for b in (sig65, msg)):
        raise TypeError("Uint8Array expected")
    if len(sig65) != 65:
        raise ValueError("recovered signature expected 65 bytes")
    rec = sig65[0]
    r, s = int.from_bytes(sig65[1:33], "big"), int.from_bytes(sig65[33:], "big")
    if rec not in (0, 1, 2, 3) or not (1 <= r < N and 1 <= s < N):
        return None
    x = r + N if rec & 2 else r
    if x >= P:  # "recovery id 2 or 3 invalid"
        return None
    try:
        rx, ry = secp256k1_decode_sec1(bytes([2 + (rec & 1)]) + x.to_bytes(32, "big"))
    except (ValueError, IndexError):
        return None
    Pt = CURVES["secp256k1"]
    R = Pt.fromAffine({"x": rx, "y": ry})
    m = hashlib.sha256(bytes(msg)).digest() if prehash else bytes(msg)
    if len(m) > SECP256K1_MAX_RAW_MSG:  # bits2int throws
        return None
    h = int.from_bytes(m, "big")
    if len(m) > 32:
        h >>= 8 * len(m) - 256
    h %= N  # bits2int_modN
    ir = pow(r, -1, N)
    u1, u2 = (-h * ir) % N, (s * ir) % N
    Q = Pt.BASE.multiplyUnsafe(u1).add(R.multiplyUnsafe(u2))
    if Q.is0():
        return None
    a = Q.toAffine()
    return a["x"], a["y"]


def eth_address(x: int, y: int) -> bytes:
    """The 20-byte Ethereum address of the key (x, y): the last 20 bytes of keccak256(x || y), big-endian."""
    return keccak256(x.to_bytes(32, "big") + y.to_bytes(32, "big"))[12:]


def eth_ecrecover(input_bytes: bytes) -> bytes:
    """ECREC: the call data right-padded with zeros to 128 bytes (or its first 128) as h || v || r || s.  Returns the
    32-byte word 12 zero bytes || address, or b"" (empty output) for v not 27 / 28, r or s outside [1, n) or a failed
    recovery."""
    data = bytes(input_bytes[:128]).ljust(128, b"\0")
    v = int.from_bytes(data[32:64], "big")
    if v not in (27, 28):
        return b""
    key = secp256k1_recover_public_key(bytes([v - 27]) + data[64:128], data[:32], prehash=False)
    if key is None:
        return b""
    return bytes(12) + eth_address(*key)
