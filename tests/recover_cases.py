"""secp256k1 public-key recovery and ecrecover inputs shared by the CPU (hostemu) and GPU tests: a signer that knows
the recovery id, the edge sets of the recovery contract (oracle.recover_ref) and of the ecrecover precompile,
signatures constructed to reach Q = O and the doubling path, and batches with scattered failures."""
import ctypes
import hashlib
import os
import random
import struct
import subprocess

import ecdsa_cases as E
from oracle import recover_ref as RR

PT, N, P = E.PT, E.N, E.P
be32 = E.be32
KEY1_ADDRESS = bytes.fromhex("7E5F4552091A69125d5DfCb7b8C2659029395Bdf")  # the address of private key 1


def key_of(d: int):
    a = PT.BASE.multiply(d % N).toAffine()
    return a["x"], a["y"]


def sig65(rec: int, r: int, s: int) -> bytes:
    return bytes([rec]) + be32(r % 2**256) + be32(s % 2**256)


def sign_rec(d: int, h: int, rnd: random.Random, low_s: bool = True, high_s: bool = False) -> bytes:
    """rec || r || s for the message representative h: rec = parity of y(k G) + 2 (x(k G) >= n); negating s (low_s
    normalisation, or high_s forcing s > n/2) negates k G and flips the parity bit."""
    while True:
        k = rnd.randrange(1, N)
        a = PT.BASE.multiply(k).toAffine()
        r = a["x"] % N
        s = pow(k, -1, N) * (h + r * d) % N
        if not (r and s):
            continue
        rec = (a["y"] & 1) | (2 if a["x"] >= N else 0)
        if (low_s and s > N >> 1) or (high_s and s <= N >> 1):
            s, rec = N - s, rec ^ 1
        return sig65(rec, r, s)


def _rec_of(sig: bytes) -> int:
    return sig[0]


def _r_s(sig: bytes):
    return int.from_bytes(sig[1:33], "big"), int.from_bytes(sig[33:], "big")


def _formula_key(rec_point, r: int, s: int, h: int):
    """Q = r^-1 (s R - h G) from the parts of a constructed signature"""
    ir = pow(r, -1, N)
    Q = rec_point.multiply(s * ir % N).add(PT.BASE.multiply(h * ir % N).negate())
    return None if Q.is0() else (Q.toAffine()["x"], Q.toAffine()["y"])


def edge_cases(seed: int = 11):
    """[(name, sig65, msg, prehash, want)]: want = the affine key known from how the item was built, None = fails."""
    rnd = random.Random(seed)
    d = rnd.randrange(1, N)
    Q = key_of(d)
    out = []
    for prehash, tag in ((True, "prehash"), (False, "raw")):  # both recovery ids, both message modes
        need = {0, 1}
        while need:
            m = bytes(rnd.randrange(256) for _ in range(32 if not prehash else 20))
            h = E.bits2int_modn(hashlib.sha256(m).digest() if prehash else m)
            sig = sign_rec(d, h, rnd)
            if _rec_of(sig) in need:
                need.discard(_rec_of(sig))
                out.append(("rec%d-%s" % (_rec_of(sig), tag), sig, m, prehash, Q))
    for ln in (0, 31, 32, 33, 64, 10000):
        m = bytes(rnd.randrange(256) for _ in range(ln))
        out.append(("msg-%d" % ln, sign_rec(d, E.bits2int_modn(hashlib.sha256(m).digest()), rnd), m, True, Q))
    for ln in (8192, 8193):
        m = bytes(rnd.randrange(256) for _ in range(ln))
        out.append(("raw-%d" % ln, sign_rec(d, E.bits2int_modn(m), rnd), m, False, Q if ln == 8192 else None))
    for name, hv in (("h=0", 0), ("h=n", N), ("h=n+5", N + 5)):
        m = be32(hv)
        out.append((name, sign_rec(d, hv % N, rnd), m, False, Q))
    m = b"high s"
    good = sign_rec(d, E.bits2int_modn(hashlib.sha256(m).digest()), rnd, low_s=False, high_s=True)
    out.append(("high-s", good, m, True, Q))
    r0, s0 = _r_s(good)
    # rec 2 / 3 on R = (n + t, y): both parities recover, to two different keys
    t = 1
    while not E._is_square(((N + t) ** 3 + 7) % P):
        t += 1
    xr = N + t
    yr = pow((xr**3 + 7) % P, (P + 1) // 4, P)
    for rec in (2, 3):
        y = yr if (yr & 1) == (rec & 1) else P - yr
        s, h = rnd.randrange(1, N), rnd.randrange(0, N)
        out.append(("rec%d-x=n+t" % rec, sig65(rec, t, s), be32(h), False,
                    _formula_key(PT.fromAffine({"x": xr, "y": y}), t, s, h)))
    for rec in (2, 3):  # r + n >= p for a random r (r + n >= 2^256 too), and r + n = p exactly
        out.append(("rec%d-r+n>=p" % rec, sig65(rec, r0, s0), m, True, None))
        out.append(("rec%d-x=p" % rec, sig65(rec, P - N, s0), m, True, None))
    for rec in (4, 27, 255):
        out.append(("rec=%d" % rec, sig65(rec, r0, s0), m, True, None))
    for v in (0, N, N + 1, 2**256 - 1):
        out.append(("r=%x" % v, sig65(_rec_of(good), v, s0), m, True, None))
        out.append(("s=%x" % v, sig65(_rec_of(good), r0, v), m, True, None))
    xn = 1
    while E._is_square((xn**3 + 7) % P):
        xn += 1
    out.append(("r-no-sqrt", sig65(0, xn, s0), m, True, None))
    out += constructed_cases(seed + 1)
    return out


def constructed_cases(seed: int = 12):
    """R = k G with h = s k (Q = O, fails) and with h = -s k (u1 G = u2 R: the complete addition doubles); msg = the
    raw 32-byte h."""
    rnd = random.Random(seed)
    out = []
    for name, sign in (("Q=O", 1), ("u1G=u2R", -1)):
        while True:
            k = rnd.randrange(1, N)
            a = PT.BASE.multiply(k).toAffine()
            if a["x"] < N:
                break
        r, s = a["x"], rnd.randrange(1, N)
        h = sign * s * k % N
        want = None if sign == 1 else key_of(2 * s * k * pow(r, -1, N))
        out.append((name, sig65(a["y"] & 1, r, s), be32(h), False, want))
    return out


def ecrecover_cases(seed: int = 13):
    """[(name, input128, want)]: want = the precompile's output word, b"" for empty output."""
    rnd = random.Random(seed)
    d = rnd.randrange(1, N)
    word = bytes(12) + RR.eth_address(*key_of(d))
    out = []
    need = {0, 1}
    base = None
    while need:
        h = be32(rnd.randrange(2**256))
        sig = sign_rec(d, E.bits2int_modn(h), rnd)
        if _rec_of(sig) in need:
            need.discard(_rec_of(sig))
            out.append(("v=%d" % (27 + _rec_of(sig)), h + be32(27 + _rec_of(sig)) + sig[1:], word))
            if base is None:
                base = (h, sig)
    h, sig = base
    for v in (0, 1, 29, 27 + 2**8, 27 + 2**248):
        out.append(("v=%x" % v, h + be32(v) + sig[1:], b""))
    r, s = _r_s(sig)
    v = be32(27 + _rec_of(sig))
    for name, rr, ss in (("r=0", 0, s), ("r=n", N, s), ("s=0", r, 0), ("s=n", r, N)):
        out.append((name, h + v + be32(rr) + be32(ss), b""))
    while True:
        hs = be32(rnd.randrange(2**256))
        sig = sign_rec(d, E.bits2int_modn(hs), rnd, low_s=False, high_s=True)
        if _rec_of(sig) < 2:
            out.append(("high-s", hs + be32(27 + _rec_of(sig)) + sig[1:], word))
            break
    while True:
        h1 = be32(rnd.randrange(2**256))
        sig = sign_rec(1, E.bits2int_modn(h1), rnd)
        if _rec_of(sig) < 2:
            out.append(("key-1", h1 + be32(27 + _rec_of(sig)) + sig[1:], bytes(12) + KEY1_ADDRESS))
            break
    return out


def signed_batch(n: int, seed: int, keys: int = 8, msg_len=None):
    """n signatures (prehash) by `keys` oracle-signer keys: [(sig65, msg, key)]; msg_len: fixed message length
    (default: random 0..79)."""
    rnd = random.Random(seed)
    ds = [rnd.randrange(1, N) for _ in range(keys)]
    pubs = [key_of(d) for d in ds]
    out = []
    for _ in range(n):
        j = rnd.randrange(keys)
        m = bytes(rnd.randrange(256) for _ in range(msg_len if msg_len is not None else rnd.randrange(0, 80)))
        out.append((sign_rec(ds[j], E.bits2int_modn(hashlib.sha256(m).digest()), rnd), m, pubs[j]))
    return out


def corrupt(items, seed: int):
    """Scatter failures among valid items: rec -> 4, r -> 0, s -> n, rec -> rec + 2 (r + n >= p); plus flipped
    message bytes, which recover a different key.  Returns [(sig65, msg)], the verdicts known from construction, and
    per item the signer's key where it must come back (None where the key is unknown or the item fails)."""
    rnd = random.Random(seed)
    out, ok, keys = [], [], []
    for sig, msg, key in items:
        kind = rnd.randrange(12)
        r, s = _r_s(sig)
        if kind == 0:
            sig = sig65(4, r, s)
        elif kind == 1:
            sig = sig65(sig[0], 0, s)
        elif kind == 2:
            sig = sig65(sig[0], r, N)
        elif kind == 3:
            sig = sig65(sig[0] | 2, r, s)
        elif kind == 4:
            msg = bytes([msg[0] ^ 1]) + msg[1:] if msg else b"\x00"
        out.append((sig, msg))
        ok.append(kind > 3)
        keys.append(key if kind > 4 else None)
    return out, ok, keys


def pack(sigs, msgs):
    """The packed arrays of nmsm_secp256k1_recover_batch: sigs65, msgs, msg_off."""
    off = [0]
    for m in msgs:
        off.append(off[-1] + len(m))
    return b"".join(sigs), b"".join(msgs), struct.pack("<%dQ" % len(off), *off)


def xy_bytes(key) -> bytes:
    """A key in the library's affine packing (little-endian x || y); 64 zero bytes for None"""
    if key is None:
        return bytes(64)
    return key[0].to_bytes(32, "little") + key[1].to_bytes(32, "little")


def key_from_xy(xy: bytes):
    return int.from_bytes(xy[:32], "little"), int.from_bytes(xy[32:], "little")


# ---- host build of the recovery bodies (tests/hostemu/recover_emu.cpp) ------------------------------------------
_emu = None


def recover_emu():
    """ctypes handle of tests/hostemu/librecoveremu.so, (re)built with g++ when the source or a device header is newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "recover_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "librecoveremu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def emu_keccak256_64(data: bytes) -> bytes:
    assert len(data) == 64
    out = ctypes.create_string_buffer(32)
    recover_emu().emu_keccak256_64(ctypes.c_char_p(data), out)
    return out.raw


def emu_recover(sigs, msgs, prehash: bool):
    """(n x 64 B keys, n verdict bytes) from the host build of the recovery bodies"""
    s, m, off = pack(sigs, msgs)
    n = len(sigs)
    xy, ok = ctypes.create_string_buffer(max(64 * n, 1)), ctypes.create_string_buffer(max(n, 1))
    rc = recover_emu().emu_recover_batch(ctypes.c_char_p(s or b"\0"), ctypes.c_char_p(m or b"\0"), ctypes.c_char_p(off),
                                         ctypes.c_uint32(n), ctypes.c_int(1 if prehash else 0), xy, ok)
    assert rc == 0
    return xy.raw[:64 * n], ok.raw[:n]


def emu_ecrecover(inputs):
    n = len(inputs)
    words, ok = ctypes.create_string_buffer(max(32 * n, 1)), ctypes.create_string_buffer(max(n, 1))
    rc = recover_emu().emu_ecrecover_batch(ctypes.c_char_p(b"".join(inputs) or b"\0"), ctypes.c_uint32(n), words, ok)
    assert rc == 0
    return words.raw[:32 * n], ok.raw[:n]
