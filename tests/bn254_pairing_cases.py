"""bn254 pairing inputs shared by the CPU (hostemu) and GPU tests: packing (the C ABI's and EIP-197's), random points in
and outside G2, pairing checks whose verdict is known by bilinearity, and the host build of the device bodies
(tests/hostemu/bn254_pairing_emu.cpp)."""
import ctypes
import os
import random
import struct
import subprocess

from oracle import bn254_pairing_ref as B

P, N = B.P, B.N
G1, G2 = B.G1, B.G2
F2 = B.F2
B2 = (19485874751759354771024239261021720505790618469301721065564631296452457478373,
      266929791119991161246907387137283842545076965332900288569378510910307636690)  # the twist's b = 3 / (9 + u)


# ---- packing: the C ABI's affine layout, 32-byte little-endian coordinates, (0, 0) for the identity ---------------
def g1_bytes(p) -> bytes:
    return p[0].to_bytes(32, "little") + p[1].to_bytes(32, "little")


def g2_bytes(q) -> bytes:
    return b"".join(c.to_bytes(32, "little") for c in (q[0][0], q[0][1], q[1][0], q[1][1]))


def offsets(counts) -> bytes:
    offs = [0]
    for c in counts:
        offs.append(offs[-1] + c)
    return struct.pack("<%dQ" % len(offs), *offs)


def pack_checks(checks):
    """checks: lists of (g1 affine, g2 affine) -> (g1 bytes, g2 bytes, offset bytes)"""
    return (b"".join(g1_bytes(p) for c in checks for p, _ in c), b"".join(g2_bytes(q) for c in checks for _, q in c),
            offsets([len(c) for c in checks]))


def eip197_bytes(pairs) -> bytes:
    """EIP-197 input: per pair G1 x, y then G2 x.c1, x.c0, y.c1, y.c0, each 32 B big-endian; zeros for the identity"""
    return b"".join(c.to_bytes(32, "big") for p, q in pairs for c in (p[0], p[1], q[0][1], q[0][0], q[1][1], q[1][0]))


ID1, ID2 = (0, 0), ((0, 0), (0, 0))


# ---- points -------------------------------------------------------------------------------------------------------
def g1_mul(k):
    return B.affine(G1.BASE.multiply(k % N)) if k % N else ID1


def g2_mul(k):
    return B.affine(G2.BASE.multiply(k % N)) if k % N else ID2


def g1_neg(p):
    return (p[0], (-p[1]) % P) if p != ID1 else ID1


def g2_off_subgroup(rnd):
    """an on-curve point of the twist E'(Fp2) outside G2"""
    while True:
        x = (rnd.randrange(P), rnd.randrange(P))
        rhs = F2.add(F2.mul(F2.sqr(x), x), B2)
        try:
            y = F2.sqrt(rhs)
        except ValueError:
            continue
        if not B.torsion_free(G2.fromAffine({"x": x, "y": y})):
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


def groth16_check(rnd, perturb=False):
    """The Groth16 verification shape e(A, B) e(-alpha, beta) e(-L, gamma) e(-C, delta) == 1 with scalars chosen by
    bilinearity: a b = al be + l ga + c de.  perturb changes the proof's C scalar by 1."""
    al, be, ga, de, l, c, b = (rnd.randrange(1, N) for _ in range(7))
    a = (al * be + l * ga + c * de) * pow(b, -1, N) % N
    if perturb:
        c += 1
    return [(g1_mul(a), g2_mul(b)), (g1_mul(-al), g2_mul(be)), (g1_mul(-l), g2_mul(ga)), (g1_mul(-c), g2_mul(de))]


# ---- host build of the device bodies (tests/hostemu/bn254_pairing_emu.cpp) -------------------------------------
_emu = None


def pairing_emu():
    """ctypes handle of tests/hostemu/libbn254pairingemu.so, (re)built with g++ when the source or a device header is
    newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "bn254_pairing_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libbn254pairingemu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def _words(b: bytes):
    return (ctypes.c_uint32 * (len(b) // 4)).from_buffer_copy(b)


def f12_bytes(a) -> bytes:
    return b"".join(c.to_bytes(32, "little") for c in B.flat(a))


def f12_from(buf) -> tuple:
    raw = bytes(buf)
    return B.unflat([int.from_bytes(raw[32 * k:32 * k + 32], "little") for k in range(12)])


def emu_fp12(op: int, a, b=B.O12):
    out = (ctypes.c_uint32 * 96)()
    assert pairing_emu().emu_fp12(op, _words(f12_bytes(a)), _words(f12_bytes(b)), out) == 0
    return f12_from(out)


def emu_pairing(pairs):
    g1 = b"".join(g1_bytes(p) for p, _ in pairs) or bytes(64)
    g2 = b"".join(g2_bytes(q) for _, q in pairs) or bytes(128)
    out = (ctypes.c_uint32 * 96)()
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


def random_pool(seed=5):
    """true and false checks of 1, 2, 3, 4 and 8 pairs"""
    rnd = random.Random(seed)
    out = {}
    for k in (2, 3, 4, 8):
        out[k] = (true_check(rnd, k), false_check(rnd, k))
    g = (g1_mul(3), g2_mul(5))
    out[1] = ([(g[0], ID2)], [g])  # one pair: only an identity pair gives 1
    return out
