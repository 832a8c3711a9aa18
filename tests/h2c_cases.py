"""Hash-to-G2 inputs and helpers shared by the CPU (hostemu) and GPU tests: the RFC 9380 known answers, messages whose
lengths cross the SHA-256 padding edges, hand-picked field elements for the SWU map's special branches, the oracle over
many messages in parallel, and the host build of the device bodies (tests/hostemu/h2c_emu.cpp)."""
import ctypes
import os
import random
import struct
import subprocess

from oracle import hash_to_curve_ref as H

P = H.P

# RFC 9380 J.10.1 (DST = H.DST_QUUX): msg -> (x.c0, x.c1, y.c0, y.c1)
KATS = {
    b"": (0x0141EBFBDCA40EB85B87142E130AB689C673CF60F1A3E98D69335266F30D9B8D4AC44C1038E9DCDD5393FAF5C41FB78A,
          0x05CB8437535E20ECFFAEF7752BADDF98034139C38452458BAEEFAB379BA13DFF5BF5DD71B72418717047F5B0F37DA03D,
          0x0503921D7F6A12805E72940B963C0CF3471C7B2A524950CA195D11062EE75EC076DAF2D4BC358C4B190C0C98064FDD92,
          0x12424AC32561493F3FE3C260708A12B7C620E7BE00099A974E259DDC7D1F6395C3C811CDD19F1E8DBF3E9ECFDCBAB8D6),
    b"abc": (0x02C2D18E033B960562AAE3CAB37A27CE00D80CCD5BA4B7FE0E7A210245129DBEC7780CCC7954725F4168AFF2787776E6,
             0x139CDDBCCDC5E91B9623EFD38C49F81A6F83F175E80B06FC374DE9EB4B41DFE4CA3A230ED250FBE3A2ACF73A41177FD8,
             0x1787327B68159716A37440985269CF584BCB1E621D3A7202BE6EA05C4CFE244AEB197642555A0645FB87BF7466B2BA48,
             0x00AA65DAE3C8D732D10ECD2C50F8A1BAF3001578F71C694E03866E9F3D49AC1E1CE70DD94A733534F106D4CEC0EDDD16),
}
# RFC 9380 K.1: expand_message_xmd(SHA-256), msg "", len_in_bytes 0x20
XMD_KAT = (b"QUUX-V01-CS02-with-expander-SHA256-128", b"", 0x20,
           bytes.fromhex("68a985b87eb6b46952128911f2a4412bbc302a9d759667f87f7a21d803f07235"))

EDGE_LENGTHS = (0, 1, 31, 32, 55, 56, 57, 63, 64, 65, 119, 120, 121, 127, 128, 255, 256, 300)


def kat_packed(coords) -> bytes:
    return b"".join(v.to_bytes(48, "little") for v in coords)


def random_messages(n: int, seed: int, max_len: int = 300):
    """n messages with lengths 0..max_len, every edge length of EDGE_LENGTHS (<= max_len) among them"""
    rnd = random.Random(seed)
    lens = [ln for ln in EDGE_LENGTHS if ln <= max_len]
    lens += [rnd.randrange(max_len + 1) for _ in range(n - len(lens))]
    rnd.shuffle(lens)
    return [bytes(rnd.randrange(256) for _ in range(ln)) for ln in lens[:n]]


def pack_messages(msgs):
    offs = [0]
    for m in msgs:
        offs.append(offs[-1] + len(m))
    return b"".join(msgs), struct.pack("<%dQ" % len(offs), *offs)


def _oracle_chunk(args):
    msgs, dst = args
    return [H.g2_packed(H.hash_to_g2(m, dst)) for m in msgs]


def oracle_packed(msgs, dst, workers=None):
    """[the oracle's hash_to_g2(m, dst) in the G2 packing], computed on all CPUs"""
    from concurrent.futures import ProcessPoolExecutor

    msgs = list(msgs)
    workers = workers or min(32, os.cpu_count() or 1)
    if workers == 1 or len(msgs) < 64:
        return _oracle_chunk((msgs, dst))
    step = -(-len(msgs) // (4 * workers))
    chunks = [(msgs[k:k + step], dst) for k in range(0, len(msgs), step)]
    with ProcessPoolExecutor(workers) as ex:
        return [b for part in ex.map(_oracle_chunk, chunks) for b in part]


def sqrt_minus_inv_z():
    """u with Z u^2 = -1, the second root of tv1 = Z^2 u^4 + Z u^2 = 0 besides u = 0 (None if -1/Z is not a square)"""
    return H.sqrt(H.neg(H.inv(H.Z_SSWU)))


def u_nonsquare_gx1(seed=11):
    """a u in Fp2 whose g(x1) is not a square, so the map takes x2 = Z u^2 x1"""
    rnd = random.Random(seed)
    while True:
        u = (rnd.randrange(P), rnd.randrange(P))
        zu2 = H.mul(H.Z_SSWU, H.mul(u, u))
        tv1 = H.add(H.mul(zu2, zu2), zu2)
        x1 = H.mul(H.mul(H.neg(H.B_ISO), H.inv(H.A_ISO)), H.add(H.ONE2, H.inv(tv1)))
        if H.sqrt(H.g_iso(x1)) is None:
            return u


def u_square_gx1(seed=12):
    rnd = random.Random(seed)
    while True:
        u = (rnd.randrange(P), rnd.randrange(P))
        zu2 = H.mul(H.Z_SSWU, H.mul(u, u))
        tv1 = H.add(H.mul(zu2, zu2), zu2)
        x1 = H.mul(H.mul(H.neg(H.B_ISO), H.inv(H.A_ISO)), H.add(H.ONE2, H.inv(tv1)))
        if H.sqrt(H.g_iso(x1)) is not None:
            return u


def special_us():
    """(name, u) for the map's branches: tv1 = 0 (u = 0 and, when it exists, Z u^2 = -1), g(x1) square and not,
    sgn0 decided by c1 (c0 = 0), and p - 1 limbs"""
    out = [("u=0", (0, 0)), ("gx1-nonsquare", u_nonsquare_gx1()), ("gx1-square", u_square_gx1()),
           ("c0=0", (0, 5)), ("c0=0-odd", (0, P - 6)), ("u=1", (1, 0)), ("u=p-1", (P - 1, P - 1))]
    r = sqrt_minus_inv_z()
    if r is not None:
        out.append(("Zu^2=-1", r))
    return out


def f2_words(a) -> bytes:
    return a[0].to_bytes(48, "little") + a[1].to_bytes(48, "little")


def point_from_packed(b: bytes):
    v = [int.from_bytes(b[48 * k:48 * k + 48], "little") for k in range(4)]
    return None if not any(v) else ((v[0], v[1]), (v[2], v[3]))


def e2_non_subgroup_points(count, seed=21):
    """points of E2(Fp2) outside G2 (random x with x^3 + 4(1 + u) a square)"""
    rnd = random.Random(seed)
    out = []
    while len(out) < count:
        x = (rnd.randrange(P), rnd.randrange(P))
        y = H.sqrt(H.add(H.mul(H.mul(x, x), x), H.B_E2))
        if y is not None:
            out.append((x, y))
    return out


# ---- host build of the device bodies (tests/hostemu/h2c_emu.cpp) ----------------------------------------------------
_emu = None


def h2c_emu():
    """ctypes handle of tests/hostemu/libh2cemu.so, (re)built with g++ when the source or a device header is newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "h2c_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libh2cemu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def emu_hash(msgs, dst: bytes):
    """[hash_to_g2(m, dst) in the G2 packing] from the host build of k_bls_hash_to_g2's bodies (dst <= 255 bytes)"""
    m, off = pack_messages(msgs)
    n = len(msgs)
    out = ctypes.create_string_buffer(max(192 * n, 1))
    rc = h2c_emu().emu_h2c_hash(ctypes.c_char_p(m or b"\0"), ctypes.c_char_p(off), ctypes.c_uint32(n),
                                ctypes.c_char_p(dst), ctypes.c_uint32(len(dst)), out)
    assert rc == 0
    return [out.raw[192 * k:192 * k + 192] for k in range(n)]


def emu_reduce512(e: int) -> int:
    out = ctypes.create_string_buffer(48)
    h2c_emu().emu_h2c_reduce512(ctypes.c_char_p(e.to_bytes(64, "little")), out)
    return int.from_bytes(out.raw, "little")


def emu_hash_to_field(msg: bytes, dst: bytes):
    out = ctypes.create_string_buffer(192)
    h2c_emu().emu_h2c_hash_to_field(ctypes.c_char_p(msg or b"\0"), ctypes.c_uint64(len(msg)), ctypes.c_char_p(dst),
                                    ctypes.c_uint32(len(dst)), out)
    v = [int.from_bytes(out.raw[48 * k:48 * k + 48], "little") for k in range(4)]
    return [(v[0], v[1]), (v[2], v[3])]


def emu_sswu(u):
    out = ctypes.create_string_buffer(192)
    h2c_emu().emu_h2c_sswu(ctypes.c_char_p(f2_words(u)), out)
    v = [int.from_bytes(out.raw[48 * k:48 * k + 48], "little") for k in range(4)]
    return (v[0], v[1]), (v[2], v[3])


def emu_iso_map(pt):
    out = ctypes.create_string_buffer(192)
    h2c_emu().emu_h2c_iso_map(ctypes.c_char_p(f2_words(pt[0]) + f2_words(pt[1])), out)
    return point_from_packed(out.raw)


def emu_clear_cofactor(pt):
    out = ctypes.create_string_buffer(192)
    h2c_emu().emu_h2c_clear_cofactor(ctypes.c_char_p(H.g2_packed(pt)), out)
    return point_from_packed(out.raw)
