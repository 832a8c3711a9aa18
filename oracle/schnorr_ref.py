"""BIP340 Schnorr signatures for secp256k1 (next-row f6): the oracle nmsm_secp256k1_schnorr_verify_batch is checked
against, and the signer that makes its test inputs.

Restates noble-curves v2 secp256k1.ts `schnorr.verify(signature, message, publicKey)` and `schnorr.sign` (BIP340) on
top of noble_ref's secp256k1 arithmetic.  Test infrastructure only.
"""
from __future__ import annotations

import hashlib

from .noble_ref import CURVES, SECP256K1_CURVE

P = SECP256K1_CURVE["p"]
N = SECP256K1_CURVE["n"]


def tagged_hash(tag: str, data: bytes) -> bytes:
    t = hashlib.sha256(tag.encode()).digest()
    return hashlib.sha256(t + t + data).digest()


def lift_x(x: int):
    """The point with x coordinate x and even y, or None (x >= p, or x^3 + 7 not a square)."""
    if not 0 <= x < P:
        return None
    c = (pow(x, 3, P) + 7) % P
    y = pow(c, (P + 1) // 4, P)
    if y * y % P != c:
        return None
    return CURVES["secp256k1"].fromAffine({"x": x, "y": y if y % 2 == 0 else P - y})


def challenge(r32: bytes, pk32: bytes, msg: bytes) -> int:
    return int.from_bytes(tagged_hash("BIP0340/challenge", r32 + pk32 + msg), "big") % N


def secp256k1_schnorr_verify(sig: bytes, msg: bytes, pk: bytes) -> bool:
    """Non-bytes arguments, a signature that is not 64 bytes and a key that is not 32 bytes throw before the reference's
    `try`; inside it every failure is a False verdict."""
    if not all(isinstance(b, (bytes, bytearray)) for b in (sig, msg, pk)):
        raise TypeError("Uint8Array expected")
    if len(sig) != 64:
        raise ValueError('"signature" expected 64 bytes')
    if len(pk) != 32:
        raise ValueError('"publicKey" expected 32 bytes')
    sig, msg, pk = bytes(sig), bytes(msg), bytes(pk)
    Pt = lift_x(int.from_bytes(pk, "big"))
    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
    if Pt is None or not (1 <= r < P) or not (1 <= s < N):  # noble: inRange(r, 1, p), inRange(s, 1, n)
        return False
    e = challenge(sig[:32], pk, msg)
    R = CURVES["secp256k1"].BASE.multiplyUnsafe(s).add(Pt.multiplyUnsafe((N - e) % N))
    if R.is0():
        return False
    a = R.toAffine()
    return a["y"] % 2 == 0 and a["x"] == r


def public_key(sk: int) -> bytes:
    """x-only public key of the secret key sk (1 <= sk < n)."""
    return CURVES["secp256k1"].BASE.multiply(sk).toAffine()["x"].to_bytes(32, "big")


def schnorr_sign(sk: int, msg: bytes, aux: bytes) -> bytes:
    """BIP340 signing: d and k normalised to even-y points, nonce from the aux and nonce tagged hashes."""
    assert 1 <= sk < N and len(aux) == 32
    G = CURVES["secp256k1"].BASE
    Pa = G.multiply(sk).toAffine()
    d = sk if Pa["y"] % 2 == 0 else N - sk
    px = Pa["x"].to_bytes(32, "big")
    t = (d ^ int.from_bytes(tagged_hash("BIP0340/aux", aux), "big")).to_bytes(32, "big")
    k0 = int.from_bytes(tagged_hash("BIP0340/nonce", t + px + bytes(msg)), "big") % N
    assert k0 != 0
    Ra = G.multiply(k0).toAffine()
    k = k0 if Ra["y"] % 2 == 0 else N - k0
    rx = Ra["x"].to_bytes(32, "big")
    e = challenge(rx, px, bytes(msg))
    return rx + ((k + e * d) % N).to_bytes(32, "big")
