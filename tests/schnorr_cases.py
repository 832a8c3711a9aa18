"""secp256k1 BIP340 Schnorr inputs shared by the CPU (hostemu) and GPU tests: the two known-answer rows of BIP340's
test vectors, the edge set of the verify contract (oracle.schnorr_ref.secp256k1_schnorr_verify), signatures constructed
to reach the rare branches of the check, and batches from the oracle signer with scattered invalid items."""
import ctypes
import os
import random
import struct
import subprocess

import ecdsa_cases as E
from oracle import schnorr_ref as SR

N = SR.N
P = SR.P

# (sk, aux, msg, pk, sig): rows 0 and 1 of BIP340's test-vectors.csv
KAT = [
    (3, bytes(32), bytes(32),
     bytes.fromhex("F9308A019258C31049344F85F89D5229B531C845836F99B08601F113BCE036F9"),
     bytes.fromhex("E907831F80848D1069A5371B402410364BDF1C5F8307B0084C55F1CE2DCA8215"
                   "25F66A4A85EA8B71E482A74F382D2CE5EBEEE8FDB2172F477DF4900D310536C0")),
    (0xB7E151628AED2A6ABF7158809CF4F3C762E7160F38B4DA56A784D9045190CFEF, bytes(31) + b"\x01",
     bytes.fromhex("243F6A8885A308D313198A2E03707344A4093822299F31D0082EFA98EC4E6C89"),
     bytes.fromhex("DFF1D77F2A671C5F36183726DB2341BE58FEAE1DA2DECED843240F7B502BA659"),
     bytes.fromhex("6896BD60EEAE296DB48A229FF71DFE071BDE413E6D43F917DC8DCF8C78DE3341"
                   "8906D11AC976ABCCB20B091292BFF4EA897EFCB639EA871CFA95F6DE339E4B0A")),
]

be32 = E.be32


def _rand_bytes(rnd: random.Random, n: int) -> bytes:
    return bytes(rnd.randrange(256) for _ in range(n))


def _even_d(sk: int) -> int:
    """The secret d with d G = lift_x(x(sk G)) (BIP340 negates sk when sk G has an odd y)."""
    return sk if E.PT.BASE.multiply(sk).toAffine()["y"] % 2 == 0 else N - sk


def sign(sk: int, msg: bytes, rnd: random.Random) -> tuple:
    """(sig, msg, pk) from the oracle signer with fresh aux randomness."""
    return SR.schnorr_sign(sk, msg, _rand_bytes(rnd, 32)), msg, SR.public_key(sk)


def edge_cases(seed: int = 17):
    """[(name, sig, msg, pk)]: the edge set the host bodies and the GPU are compared with the oracle on."""
    rnd = random.Random(seed)
    sk = rnd.randrange(1, N)
    pk = SR.public_key(sk)
    msg = b"edge set"
    good = SR.schnorr_sign(sk, msg, _rand_bytes(rnd, 32))
    r0, s0 = good[:32], good[32:]
    out = [("valid", good, msg, pk)]
    for k, (_, _, m, kpk, ksig) in enumerate(KAT):
        out.append(("kat-%d" % k, ksig, m, kpk))
    xn = 1  # the smallest x >= 1 with x^3 + 7 not a square (x = 0 has none either: 7 is not a square mod p)
    while SR.lift_x(xn) is not None:
        xn += 1
    for name, x in (("0", 0), ("p", P), ("p+1", P + 1), ("2^256-1", 2**256 - 1), ("no-sqrt", xn)):
        out.append(("key-x=" + name, good, msg, be32(x)))
    for name, r in (("0", 0), ("p-1", P - 1), ("p", P), ("2^256-1", 2**256 - 1), ("n", N), ("n+1", N + 1)):
        out.append(("r=" + name, be32(r) + s0, msg, pk))
    for name, s in (("0", 0), ("n", N), ("2^256-1", 2**256 - 1), ("n-s", N - int.from_bytes(s0, "big"))):
        out.append(("s=" + name, r0 + be32(s), msg, pk))
    for ln in (0, 32, 55, 56, 119, 120, 10000):
        m = _rand_bytes(rnd, ln)
        out.append(("msg-%d" % ln,) + sign(sk, m, rnd))
    out += constructed_cases(seed + 1)
    return out


def constructed_cases(seed: int = 18):
    """Signatures that reach the rare branches of the check: R = O, an odd y(R) with x(R) == r, and s G == u P (the
    complete addition doubles)."""
    rnd = random.Random(seed)
    sk = rnd.randrange(1, N)
    d = _even_d(sk)
    pk = SR.public_key(sk)
    out = []
    # R = s G - e P = O: s = e d for a chosen r
    msg = b"R = O"
    r32 = be32(E.PT.BASE.multiply(rnd.randrange(1, N)).toAffine()["x"])
    s = SR.challenge(r32, pk, msg) * d % N
    out.append(("R=O", r32 + be32(s), msg, pk))
    # odd y(R): k G with an odd y, used without BIP340's negation of k
    msg = b"odd y"
    while True:
        k = rnd.randrange(1, N)
        Ra = E.PT.BASE.multiply(k).toAffine()
        if Ra["y"] % 2:
            break
    r32 = be32(Ra["x"])
    s = (k + SR.challenge(r32, pk, msg) * d) % N
    out.append(("odd-y", r32 + be32(s), msg, pk))
    # s G == u P with u = n - e: s = u d, R = 2 s G
    msg = b"sG = uP"
    r32 = be32(E.PT.BASE.multiply(rnd.randrange(1, N)).toAffine()["x"])
    u = (N - SR.challenge(r32, pk, msg)) % N
    out.append(("sG=uP", r32 + be32(u * d % N), msg, pk))
    return out


def signed_batch(n: int, seed: int, msg_len=None):
    """n fresh keys signed by the oracle signer: [(sig, msg, pk)]; msg_len: fixed length (default: random 0..79)."""
    rnd = random.Random(seed)
    out = []
    for _ in range(n):
        m = _rand_bytes(rnd, msg_len if msg_len is not None else rnd.randrange(0, 80))
        out.append(sign(rnd.randrange(1, N), m, rnd))
    return out


def corrupt(items, seed: int):
    """Scatter invalid items among valid ones: flipped message byte, flipped r byte, s -> n - s, key x -> x + 1.
    About one item in four is touched.  Returns [(sig, msg, pk)] and the expected verdicts."""
    rnd = random.Random(seed)
    out, want = [], []
    for sig, msg, pk in items:
        kind = rnd.randrange(16)
        if kind == 0 and msg:
            msg = bytes([msg[0] ^ 1]) + msg[1:]
        elif kind in (0, 1):
            sig = bytes([sig[0] ^ 0x80]) + sig[1:]
        elif kind == 2:
            sig = sig[:32] + be32(N - int.from_bytes(sig[32:], "big"))
        elif kind == 3:
            pk = be32(int.from_bytes(pk, "big") + 1)
        out.append((sig, msg, pk))
        want.append(kind > 3)
    return out, want


def pack(sigs, msgs, pks):
    """The packed arrays of nmsm_secp256k1_schnorr_verify_batch: sigs, pks, msgs, msg_off."""
    off = [0]
    for m in msgs:
        off.append(off[-1] + len(m))
    return b"".join(sigs), b"".join(pks), b"".join(msgs), struct.pack("<%dQ" % len(off), *off)


# ---- host build of the verification bodies (tests/hostemu/schnorr_emu.cpp) --------------------------------------
_emu = None


def schnorr_emu():
    """ctypes handle of tests/hostemu/libschnorremu.so, (re)built with g++ when the source or a device header is newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "schnorr_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libschnorremu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def emu_challenge(r32: bytes, pk32: bytes, msg: bytes) -> bytes:
    out = ctypes.create_string_buffer(32)
    schnorr_emu().emu_bip340_challenge(ctypes.c_char_p(r32), ctypes.c_char_p(pk32), ctypes.c_char_p(msg or b"\0"),
                                       ctypes.c_uint64(len(msg)), out)
    return out.raw


def emu_verify(items):
    sigs, pks, msgs, msg_off = pack([i[0] for i in items], [i[1] for i in items], [i[2] for i in items])
    out = ctypes.create_string_buffer(max(len(items), 1))
    cp = lambda b: ctypes.c_char_p(b or b"\0")  # noqa: E731
    rc = schnorr_emu().emu_schnorr_verify_batch(cp(sigs), cp(pks), cp(msgs), cp(msg_off), len(items), out)
    assert rc == 0
    return [b == 1 for b in out.raw[:len(items)]]
