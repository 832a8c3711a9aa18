"""BLS12-381 pairing inputs shared by the CPU (hostemu) and GPU tests: packing, random points in and outside the
subgroups, pairing checks whose verdict is known by bilinearity, the verification edge set of the contract
(oracle.bls_pairing_ref.bls_verify), and the host build of the device bodies (tests/hostemu/pairing_emu.cpp)."""
import ctypes
import os
import random
import struct
import subprocess

from oracle import bls_pairing_ref as B

P, N = B.P, B.N
G1, G2 = B.G1, B.G2
F2 = B.F2


# ---- packing: the C ABI's affine layout, 48-byte little-endian coordinates, (0, 0) for the identity ---------------
def g1_bytes(p) -> bytes:
    return p[0].to_bytes(48, "little") + p[1].to_bytes(48, "little")


def g2_bytes(q) -> bytes:
    return b"".join(c.to_bytes(48, "little") for c in (q[0][0], q[0][1], q[1][0], q[1][1]))


def offsets(counts) -> bytes:
    offs = [0]
    for c in counts:
        offs.append(offs[-1] + c)
    return struct.pack("<%dQ" % len(offs), *offs)


def pack_checks(checks):
    """checks: lists of (g1 affine, g2 affine) -> (g1 bytes, g2 bytes, offset bytes)"""
    return (b"".join(g1_bytes(p) for c in checks for p, _ in c), b"".join(g2_bytes(q) for c in checks for _, q in c),
            offsets([len(c) for c in checks]))


ID1, ID2 = (0, 0), ((0, 0), (0, 0))


# ---- points -------------------------------------------------------------------------------------------------------
def g1_mul(k):
    return B.affine(G1.BASE.multiply(k % N)) if k % N else ID1


def g2_mul(k):
    return B.affine(G2.BASE.multiply(k % N)) if k % N else ID2


def g1_off_subgroup(rnd):
    """an on-curve point of E(Fp) outside G1"""
    while True:
        x = rnd.randrange(P)
        y2 = (x ** 3 + 4) % P
        y = pow(y2, (P + 1) // 4, P)
        if y * y % P == y2 and y:
            pt = G1.fromAffine({"x": x, "y": y})
            if not B.torsion_free(pt):
                return (x, y)


def g2_off_subgroup(rnd):
    """an on-curve point of the twist E'(Fp2) outside G2"""
    while True:
        x = (rnd.randrange(P), rnd.randrange(P))
        rhs = F2.add(F2.mul(F2.sqr(x), x), (4, 4))
        try:
            y = F2.sqrt(rhs)
        except ValueError:
            continue
        pt = G2.fromAffine({"x": x, "y": y})
        if not B.torsion_free(pt):
            return (x, y)


def true_check(rnd, k):
    """k pairs whose pairing product is 1 by bilinearity: (a_i G1, b_i G2) for i < k - 1 and (-(sum a_i b_i) G1, G2)"""
    a = [rnd.randrange(1, N) for _ in range(k - 1)]
    b = [rnd.randrange(1, N) for _ in range(k - 1)]
    s = sum(x * y for x, y in zip(a, b)) % N
    return [(g1_mul(x), g2_mul(y)) for x, y in zip(a, b)] + [(g1_mul(-s), g2_mul(1))]


def false_check(rnd, k):
    """true_check with the last G1 scalar changed by 1"""
    a = [rnd.randrange(1, N) for _ in range(k - 1)]
    b = [rnd.randrange(1, N) for _ in range(k - 1)]
    s = sum(x * y for x, y in zip(a, b)) % N
    return [(g1_mul(x), g2_mul(y)) for x, y in zip(a, b)] + [(g1_mul(-s + 1), g2_mul(1))]


# ---- signatures -----------------------------------------------------------------------------------------------------
def keypair_item(rnd):
    """(sig96, H affine, pk48) of a valid signature: H = h G2 stands for a hashed message, sig = sk H"""
    sk, h = rnd.randrange(1, N), rnd.randrange(1, N)
    H = G2.BASE.multiply(h)
    return B.sign(sk, H), B.affine(H), B.public_key(sk)


def _set_x_g1(x: int, flags: int = 0x80) -> bytes:
    b = bytearray(x.to_bytes(48, "big"))
    b[0] |= flags
    return bytes(b)


def _set_x_g2(x0: int, x1: int, flags: int = 0x80) -> bytes:
    b = bytearray(x1.to_bytes(48, "big") + x0.to_bytes(48, "big"))
    b[0] |= flags
    return bytes(b)


def _nonsquare_g1_x():
    x = 1
    while True:
        y2 = (x ** 3 + 4) % P
        if pow(y2, (P - 1) // 2, P) == P - 1:
            return x
        x += 1


def _nonsquare_g2_x():
    x = 1
    while True:
        try:
            F2.sqrt(F2.add(F2.mul(F2.sqr((x, 1)), (x, 1)), (4, 4)))
        except ValueError:
            return (x, 1)
        x += 1


def edge_cases(seed=11):
    """(name, sig96, H, pk48) covering every branch of the verify contract"""
    rnd = random.Random(seed)
    v1, v2 = keypair_item(rnd), keypair_item(rnd)
    sig, H, pk = v1
    out = [("valid", *v1), ("valid-2", *v2),
           ("wrong-key", sig, H, v2[2]), ("wrong-message", sig, v2[1], pk), ("swapped-sig", v2[0], H, pk)]
    out.append(("sig-uncompressed-flag", bytes([sig[0] & 0x7F]) + sig[1:], H, pk))
    out.append(("pk-uncompressed-flag", sig, H, bytes([pk[0] & 0x7F]) + pk[1:]))
    out.append(("sig-flags-e0", bytes([sig[0] | 0xE0]) + sig[1:], H, pk))
    out.append(("pk-flags-e0", sig, H, bytes([pk[0] | 0xE0]) + pk[1:]))
    out.append(("pk-x>=p", sig, H, _set_x_g1(P)))
    out.append(("sig-x.c1>=p", _set_x_g2(1, P), H, pk))
    out.append(("sig-x.c0>=p", _set_x_g2(P + 1, 0), H, pk))
    out.append(("pk-nonsquare", sig, H, _set_x_g1(_nonsquare_g1_x())))
    x = _nonsquare_g2_x()
    out.append(("sig-nonsquare", _set_x_g2(x[0], x[1]), H, pk))
    out.append(("pk-identity", sig, H, bytes([0xC0]) + bytes(47)))
    out.append(("sig-identity", bytes([0xC0]) + bytes(95), H, pk))
    out.append(("pk-identity-noncanonical", sig, H, bytes([0xC0]) + bytes(46) + b"\x01"))
    out.append(("H-identity", sig, ID2, pk))
    p1 = g1_off_subgroup(rnd)
    out.append(("pk-off-subgroup", sig, H, B.g1_encode(G1.fromAffine({"x": p1[0], "y": p1[1]}))))
    q1 = g2_off_subgroup(rnd)
    out.append(("sig-off-subgroup", B.g2_encode(G2.fromAffine({"x": q1[0], "y": q1[1]})), H, pk))
    return out


# ---- host build of the device bodies (tests/hostemu/pairing_emu.cpp) -------------------------------------------
_emu = None


def pairing_emu():
    """ctypes handle of tests/hostemu/libpairingemu.so, (re)built with g++ when the source or a device header is newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "pairing_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libpairingemu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def _words(b: bytes):
    return (ctypes.c_uint32 * (len(b) // 4)).from_buffer_copy(b)


def f12_bytes(a) -> bytes:
    return b"".join(c.to_bytes(48, "little") for c in B.flat(a))


def f12_from(buf) -> tuple:
    raw = bytes(buf)
    return B.unflat([int.from_bytes(raw[48 * k:48 * k + 48], "little") for k in range(12)])


def emu_fp12(op: int, a, b=B.O12):
    out = (ctypes.c_uint32 * 144)()
    assert pairing_emu().emu_fp12(op, _words(f12_bytes(a)), _words(f12_bytes(b)), out) == 0
    return f12_from(out)


def emu_pairing(pairs):
    g1 = b"".join(g1_bytes(p) for p, _ in pairs) or bytes(96)
    g2 = b"".join(g2_bytes(q) for _, q in pairs) or bytes(192)
    out = (ctypes.c_uint32 * 144)()
    pairing_emu().emu_pairing(_words(g1), _words(g2), len(pairs), out)
    return f12_from(out)


def emu_pairing_check(checks, chunk=1 << 16):
    g1, g2, off = pack_checks(checks)
    out = ctypes.create_string_buffer(max(len(checks), 1))
    err = (ctypes.c_uint32 * 2)()
    pairing_emu().emu_pairing_check(_words(g1 or bytes(4)), _words(g2 or bytes(4)), ctypes.c_char_p(off),
                                    ctypes.c_uint64(len(checks)), ctypes.c_uint64(chunk), out, err)
    bad = lambda e: None if e == 0xFFFFFFFF else e  # noqa: E731
    return [b == 1 for b in out.raw[:len(checks)]], (bad(err[0]), bad(err[1]))


def emu_verify(items, chunk=1 << 16):
    """items: (sig96, H affine, pk48) -> (verdicts, smallest bad message index or None)"""
    sigs = b"".join(i[0] for i in items)
    pks = b"".join(i[2] for i in items)
    hs = b"".join(g2_bytes(i[1]) for i in items)
    out = ctypes.create_string_buffer(max(len(items), 1))
    err = (ctypes.c_uint32 * 1)()
    rc = pairing_emu().emu_bls_verify(ctypes.c_char_p(sigs), ctypes.c_char_p(pks), _words(hs), len(items),
                                      ctypes.c_uint64(chunk), out, err)
    assert rc == 0
    return [b == 1 for b in out.raw[:len(items)]], (None if err[0] == 0xFFFFFFFF else err[0])
