"""ed25519 inputs shared by the CPU (hostemu) and GPU tests of per-signature verification (nmsm_ed25519_verify_each):
signing from the curve equations with chosen r and a and torsion parts, the golden sets (RFC 8032-style vectors, the
ZIP-215 cases, the strict edge cases), the edge set of the verify contract (oracle.noble_ref.ed25519_verify), and
OpenSSL-signed batches through the `cryptography` package."""
import ctypes
import hashlib
import os
import random
import struct
import subprocess

import torsion_cases as TC
from conftest import load_golden
from oracle import noble_ref as R

ED = R.CURVES["ed25519"]
L = ED.Fn.ORDER
P = R.ED25519_CURVE["p"]
MODES = (True, False)  # zip215
MSG_LENS = (0, 47, 48, 175, 176, 1000)  # 64 + |M| on either side of the SHA-512 block boundaries 112 and 240


def le32(x: int) -> bytes:
    return x.to_bytes(32, "little")


def challenge(r32: bytes, pk: bytes, msg: bytes) -> int:
    return int.from_bytes(hashlib.sha512(r32 + pk + msg).digest(), "little") % L


def sign_with(a: int, r: int, msg: bytes, T_R=None, T_A=None, r_bytes=None, a_bytes=None):
    """(sig, msg, pk) with R = r B + T_R, A = a B + T_A and s = r + k a mod l, k = SHA-512(R || A || M) over the
    encodings used (r_bytes / a_bytes: a chosen encoding of the same point, e.g. a non-canonical one)."""
    Rp = ED.BASE.multiply(r) if r else ED.ZERO
    Ap = ED.BASE.multiply(a) if a else ED.ZERO
    if T_R is not None:
        Rp = Rp.add(T_R)
    if T_A is not None:
        Ap = Ap.add(T_A)
    rb = r_bytes if r_bytes is not None else Rp.toBytes()
    ab = a_bytes if a_bytes is not None else Ap.toBytes()
    s = (r + challenge(rb, ab, msg) * a) % L
    return rb + le32(s), msg, ab


def small_order():
    """The eight points of order dividing 8: j * T8 for j = 0..7, the identity first."""
    T8 = next(T for T, q in TC.small_points("ed25519") if q == 8)
    out = [ED.ZERO]
    for _ in range(7):
        out.append(out[-1].add(T8))
    return out


# ---- golden sets -------------------------------------------------------------------------------------------------
def rfc_vectors():
    """[(name, sig, msg, pk)]: the 128 RFC 8032-style vectors, each also with one bit of s and of the message flipped."""
    out = []
    for j, v in enumerate(load_golden("ed25519.json")["vectors"]):
        sig, msg, pk = bytes.fromhex(v["sig"]), bytes.fromhex(v["msg"]), bytes.fromhex(v["pk"])
        out.append(("rfc-%d" % j, sig, msg, pk))
        out.append(("rfc-%d-s^1" % j, sig[:32] + bytes([sig[32] ^ 1]) + sig[33:], msg, pk))
        bad_msg = bytes([msg[0] ^ 0x80]) + msg[1:] if msg else b"\x01"
        out.append(("rfc-%d-msg^" % j, sig, bad_msg, pk))
    return out


def zip215_cases():
    """[(name, sig, msg, pk)]: the 196 ZIP-215 cases (small-order and non-canonical R and A, message "Zcash")."""
    return [("zip215-%d" % j, bytes.fromhex(v["sig_bytes"]), b"Zcash", bytes.fromhex(v["vk_bytes"]))
            for j, v in enumerate(load_golden("ed25519.json")["zip215"])]


def strict_edge_cases():
    """[(name, sig, msg, pk)]: the 12 edge cases of the strict decoding rules."""
    return [("edge-%d" % j, bytes.fromhex(v["signature"]), bytes.fromhex(v["message"]), bytes.fromhex(v["pub_key"]))
            for j, v in enumerate(load_golden("ed25519.json")["edge_cases"])]


# ---- constructed cases -------------------------------------------------------------------------------------------
def constructed_cases(seed: int = 19):
    """[(name, sig, msg, pk)]: the branches of the contract the golden sets do not pin down one by one."""
    rnd = random.Random(seed)
    out = []
    a, r = rnd.randrange(1, L), rnd.randrange(1, L)
    sig, msg, pk = sign_with(a, r, b"constructed")
    out.append(("valid", sig, msg, pk))
    # s range: l and above is false; 0 and l - 1 are in range (made valid through a small-order A)
    for name, s in (("l", L), ("l+1", L + 1), ("2^253", 2**253), ("2^256-1", 2**256 - 1)):
        out.append(("s=" + name, sig[:32] + le32(s), msg, pk))
    ident = ED.ZERO.toBytes()
    T8 = TC.small_points("ed25519")[-1][0]
    out.append(("s=0", T8.toBytes() + le32(0), b"s = 0", ident))  # [8](T + k O - 0 B) = O
    out.append(("s=l-1", ED.BASE.negate().toBytes() + le32(L - 1), b"s = l - 1", ident))  # [8](-B - (l-1) B) = O
    out.append(("s=l-ident", T8.toBytes() + le32(L), b"s = l", ident))
    # 8-torsion parts on R and on A: the cofactored equation accepts
    for j, T in enumerate(small_order()):
        out.append(("tors-R-%d" % j,) + sign_with(rnd.randrange(1, L), rnd.randrange(1, L), b"R + T", T_R=T))
        out.append(("tors-A-%d" % j,) + sign_with(rnd.randrange(1, L), rnd.randrange(1, L), b"A + T", T_A=T))
        out.append(("tors-RA-%d" % j,) + sign_with(rnd.randrange(1, L), rnd.randrange(1, L), b"R+T, A+T'", T_R=T,
                                                   T_A=small_order()[(j + 3) % 8]))
    # A of small order (the identity included): ZIP-215 accepts when the equation holds, strict rejects
    for j, T in enumerate(small_order()):
        r = rnd.randrange(1, L)
        out.append(("small-A-%d" % j, ED.BASE.multiply(r).toBytes() + le32(r), b"small A", T.toBytes()))
    # the hash is over the raw bytes: R = O encoded with y = p + 1
    a = rnd.randrange(1, L)
    raw_o = le32(P + 1)
    out.append(("raw-R",) + sign_with(a, 0, b"raw bytes", r_bytes=raw_o))
    sig, msg, pk = sign_with(a, 0, b"raw bytes", r_bytes=ident)
    out.append(("raw-R-canonical-k", raw_o + sig[32:], msg, pk))  # k over the canonical encoding: rejected
    # the identity as x = 0 with the sign bit set
    ident_neg = ident[:31] + bytes([ident[31] | 0x80])
    out.append(("x0-sign-R",) + sign_with(rnd.randrange(1, L), 0, b"x = 0, sign", r_bytes=ident_neg))
    r = rnd.randrange(1, L)
    out.append(("x0-sign-A", ED.BASE.multiply(r).toBytes() + le32(r), b"x = 0, sign", ident_neg))
    # message lengths around the SHA-512 block boundaries
    for ln in MSG_LENS:
        m = bytes(rnd.randrange(256) for _ in range(ln))
        out.append(("msg-%d" % ln,) + sign_with(rnd.randrange(1, L), rnd.randrange(1, L), m))
    return out


def all_cases():
    return rfc_vectors() + zip215_cases() + strict_edge_cases() + constructed_cases()


# ---- OpenSSL (cryptography) ----------------------------------------------------------------------------------------
def openssl_sign(n: int, seed: int, msg_len=None):
    """n fresh keys and signatures from OpenSSL: [(sig, msg, pk)]; msg_len: fixed length (default: random 0..99)."""
    from cryptography.hazmat.primitives import serialization
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey

    rnd = random.Random(seed)
    raw = serialization.Encoding.Raw, serialization.PublicFormat.Raw
    out = []
    for _ in range(n):
        sk = Ed25519PrivateKey.from_private_bytes(rnd.randbytes(32))
        m = rnd.randbytes(msg_len if msg_len is not None else rnd.randrange(0, 100))
        out.append((sk.sign(m), m, sk.public_key().public_bytes(*raw)))
    return out


def openssl_verify(sig: bytes, msg: bytes, pk: bytes) -> bool:
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PublicKey

    try:
        Ed25519PublicKey.from_public_bytes(pk).verify(sig, msg)
        return True
    except (InvalidSignature, ValueError):
        return False


def corrupt(items, seed: int):
    """Scatter invalid items among valid ones: a flipped message bit, s + 1, s + l, a flipped byte of R, another key.
    About one item in three is touched.  Returns [(sig, msg, pk)] and the expected verdicts."""
    rnd = random.Random(seed)
    out, want = [], []
    for j, (sig, msg, pk) in enumerate(items):
        kind = rnd.randrange(15)
        s = int.from_bytes(sig[32:], "little")
        if kind == 0 and msg:
            msg = bytes([msg[0] ^ 1]) + msg[1:]
        elif kind in (0, 1):
            sig = sig[:32] + le32((s + 1) % L)
        elif kind == 2:
            sig = sig[:32] + le32(s + L)
        elif kind == 3:
            sig = bytes([sig[0] ^ 0x10]) + sig[1:]
        elif kind == 4:
            pk = items[(j + 1) % len(items)][2] if items[(j + 1) % len(items)][2] != pk else ED.BASE.toBytes()
        out.append((sig, msg, pk))
        want.append(kind > 4)
    return out, want


def pack(sigs, msgs, pks):
    """The packed arrays of nmsm_ed25519_verify_each: sigs, pks, msgs, msg_off."""
    off = [0]
    for m in msgs:
        off.append(off[-1] + len(m))
    return b"".join(sigs), b"".join(pks), b"".join(msgs), struct.pack("<%dQ" % len(off), *off)


# ---- host build of the verification bodies (tests/hostemu/ed25519_verify_emu.cpp) --------------------------------
_emu = None


def ed25519_emu():
    """ctypes handle of tests/hostemu/libed25519verifyemu.so, (re)built with g++ when the source or a device header is
    newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "ed25519_verify_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libed25519verifyemu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def emu_verify(items, zip215: bool = True):
    """[(sig, msg, pk)] -> verdicts of the serial host bodies."""
    sigs, pks, msgs, msg_off = pack([i[0] for i in items], [i[1] for i in items], [i[2] for i in items])
    out = ctypes.create_string_buffer(max(len(items), 1))
    cp = lambda b: ctypes.c_char_p(b or b"\0")  # noqa: E731
    rc = ed25519_emu().emu_ed25519_verify_each(cp(sigs), cp(pks), cp(msgs), cp(msg_off), len(items),
                                               0 if zip215 else 1, out)
    assert rc == 0
    return [b == 1 for b in out.raw[:len(items)]]
