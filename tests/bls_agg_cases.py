"""BLS12-381 aggregate-verification inputs shared by the CPU (hostemu) and GPU tests: key packing, the edge set of the
contract (oracle.bls_aggregate_ref.aggregate_verify, rules 1-5), packing of checks into the C ABI's arrays, and the
host build of the device bodies (tests/hostemu/bls_agg_emu.cpp)."""
import ctypes
import os
import random
import struct
import subprocess

import bls_cases as BC
from oracle import bls_aggregate_ref as A
from oracle import bls_pairing_ref as B

P, N = B.P, B.N
ID1 = (0, 0)
DST = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_"


def key_bytes(k) -> bytes:
    """an affine G1 key in the C ABI's 96-byte packing"""
    return k[0].to_bytes(48, "little") + k[1].to_bytes(48, "little")


def neg(k):
    return ID1 if k == ID1 else (k[0], (-k[1]) % P)


def sign_agg(sks, msg: bytes, dst: bytes = DST) -> bytes:
    """(sum sks) H(msg), encoded: an aggregate of the signatures of sks over msg (the identity if the sum is 0 mod N)"""
    h = A.hashed(msg, dst)
    s = sum(sks) % N
    if s == 0 or h == BC.ID2:
        return bytes([0xC0]) + bytes(95)
    return B.g2_encode(B.G2.fromAffine({"x": h[0], "y": h[1]}).multiply(s))


def sign_groups(groups_sks, dst: bytes = DST) -> bytes:
    """one aggregate signature over [(msg, [sk])]: sum over groups of (sum sks) H(msg)"""
    acc = B.G2.ZERO
    for msg, sks in groups_sks:
        h = A.hashed(msg, dst)
        s = sum(sks) % N
        if s:
            acc = acc.add(B.G2.fromAffine({"x": h[0], "y": h[1]}).multiply(s))
    return B.g2_encode(acc)


def pack(checks):
    """checks: [(sig96, [(msg, [affine keys])])] -> the C ABI's (sigs96, group_off, msgs, msg_off, keys_xy, key_off)
    as bytes, u64 little-endian offsets"""
    sigs, goff, msgs, moff, keys, koff = [], [0], [], [0], [], [0]
    for sig, groups in checks:
        sigs.append(sig)
        for msg, ks in groups:
            msgs.append(msg)
            moff.append(moff[-1] + len(msg))
            keys.extend(key_bytes(k) for k in ks)
            koff.append(len(keys))
        goff.append(len(moff) - 1)
    u64 = lambda v: struct.pack("<%dQ" % len(v), *v)  # noqa: E731
    return b"".join(sigs), u64(goff), b"".join(msgs), u64(moff), b"".join(keys), u64(koff)


def oracle(checks, dst: bytes = DST):
    return [A.aggregate_verify(sig, groups, dst) for sig, groups in checks]


def edge_checks(seed=5):
    """(name, check) for every rule of the contract in order, with the verdict the oracle gives"""
    rnd = random.Random(seed)
    sks = [rnd.randrange(1, N) for _ in range(5)]
    pks = [BC.g1_mul(k) for k in sks]
    m1, m2 = b"attestation-1", b"attestation-2"
    good = sign_agg(sks[:3], m1)
    out = [("valid-3", (good, [(m1, pks[:3])])),
           ("valid-1", (sign_agg(sks[:1], m1), [(m1, pks[:1])])),
           ("valid-two-groups", (sign_groups([(m1, sks[:2]), (m2, sks[2:4])]), [(m1, pks[:2]), (m2, pks[2:4])]))]
    # rule 1: the signature encodings of the verify edge set, each over the good check's keys
    for name, sig, _, _ in BC.edge_cases():
        if name.startswith("sig-"):
            out.append((name, (sig, [(m1, pks[:3])])))
    # rule 2: an empty check and an empty group
    out.append(("empty-check", (good, [])))
    out.append(("empty-group", (good, [(m1, pks[:3]), (m2, [])])))
    # rule 3: an identity key, also next to keys that would verify without it
    out.append(("identity-key", (good, [(m1, pks[:3] + [ID1])])))
    # rule 4: P and -P sum to the identity
    out.append(("p-and-minus-p", (sign_agg([sks[0], sks[1], -sks[1]], m1), [(m1, [pks[0], pks[1], neg(pks[1])])])))
    out.append(("sum-identity", (sign_agg([sks[0]], m1), [(m1, [pks[0], neg(pks[0])])])))
    # a repeated key: the doubling branch of the additions
    out.append(("duplicate-key", (sign_agg([sks[0], sks[0], sks[1]], m1), [(m1, [pks[0], pks[0], pks[1]])])))
    # rule 5: a wrong message and a swapped key
    out.append(("wrong-message", (good, [(m2, pks[:3])])))
    out.append(("swapped-key", (good, [(m1, pks[:2] + [pks[3]])])))
    # a key outside G1 (the caller's subgroup check is skipped on purpose): whatever the formulas give
    out.append(("key-off-subgroup", (good, [(m1, pks[:3] + [BC.g1_off_subgroup(rnd)])])))
    return out


# ---- host build of the device bodies (tests/hostemu/bls_agg_emu.cpp) ------------------------------------------------
_emu = None


def agg_emu():
    """ctypes handle of tests/hostemu/libblsaggemu.so, (re)built with g++ when the source or a device header is newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "bls_agg_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libblsaggemu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def emu_aggregate(checks, tile, chunk, cap=1 << 20, dst: bytes = DST):
    """(verdicts, smallest bad key index or None, internal pair errors) from bls_agg_serial"""
    sigs, goff, msgs, moff, keys, koff = pack(checks)
    n = len(checks)
    out = ctypes.create_string_buffer(max(n, 1))
    err = (ctypes.c_uint32 * 3)()
    keys_w = (ctypes.c_uint32 * max(len(keys) // 4, 1)).from_buffer_copy(keys or bytes(4))
    rc = agg_emu().emu_bls_aggregate(ctypes.c_char_p(sigs or b"\0"), ctypes.c_char_p(goff), ctypes.c_uint64(n),
                                     ctypes.c_char_p(msgs or b"\0"), ctypes.c_char_p(moff), keys_w,
                                     ctypes.c_char_p(koff), ctypes.c_char_p(dst), ctypes.c_uint32(len(dst)),
                                     ctypes.c_uint64(tile), ctypes.c_uint64(cap), ctypes.c_uint64(chunk), out, err)
    assert rc == 0
    bad = lambda e: None if e == 0xFFFFFFFF else e  # noqa: E731
    return [b == 1 for b in out.raw[:n]], bad(err[0]), (bad(err[1]), bad(err[2]))
