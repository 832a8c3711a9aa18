"""Hash-to-G1 and short-signature inputs shared by the CPU (hostemu) and GPU tests: the RFC 9380 J.9.1 known answers,
field elements for the SWU map's special branches, points of E1 outside G1, the short-signature edge set, signed
batches, the oracle over many messages in parallel, and the host build of the device bodies (tests/hostemu/h2g1_emu.cpp).
Message packing and the message generator are h2c_cases'."""
import ctypes
import os
import random
import subprocess

import bls_cases as BC
from h2c_cases import EDGE_LENGTHS, pack_messages, random_messages  # noqa: F401  (re-exported for the tests)
from oracle import bls_pairing_ref as B
from oracle import hash_to_g1_ref as H

P, N = H.P, H.N

# RFC 9380 J.9.1 (DST = H.DST_QUUX): msg -> (x, y)
KATS = {
    b"": (0x052926ADD2207B76CA4FA57A8734416C8DC95E24501772C814278700EED6D1E4E8CF62D9C09DB0FAC349612B759E79A1,
          0x08BA738453BFED09CB546DBB0783DBB3A5F1F566ED67BB6BE0E8C67E2E81A4CC68EE29813BB7994998F3EAE0C9C6A265),
    b"abc": (0x03567BC5EF9C690C2AB2ECDF6A96EF1C139CC0B2F284DCA0A9A7943388A49A3AEE664BA5379A7655D3C68900BE2F6903,
             0x0B9C15F3FE6E5CF4211F346271D7B01C8F3B28BE689C8429C85B67AF215533311F0B8DFAAA154FA6B88176C229F2885D),
}


def kat_packed(coords) -> bytes:
    return b"".join(v.to_bytes(48, "little") for v in coords)


def point_from_packed(b: bytes):
    x, y = int.from_bytes(b[:48], "little"), int.from_bytes(b[48:96], "little")
    return None if x == 0 and y == 0 else (x, y)


def _oracle_chunk(args):
    msgs, dst = args
    return [H.g1_packed(H.hash_to_g1(m, dst)) for m in msgs]


def oracle_packed(msgs, dst, workers=None):
    """[the oracle's hash_to_g1(m, dst) in the G1 packing], computed on all CPUs"""
    from concurrent.futures import ProcessPoolExecutor

    msgs = list(msgs)
    workers = workers or min(32, os.cpu_count() or 1)
    if workers == 1 or len(msgs) < 64:
        return _oracle_chunk((msgs, dst))
    step = -(-len(msgs) // (4 * workers))
    chunks = [(msgs[k:k + step], dst) for k in range(0, len(msgs), step)]
    with ProcessPoolExecutor(workers) as ex:
        return [b for part in ex.map(_oracle_chunk, chunks) for b in part]


# ---- the SWU map's branches and points outside G1 ---------------------------------------------------------------
def _x1(u):
    zu2 = H.Z_SSWU * u * u % P
    tv1 = (zu2 * zu2 + zu2) % P
    return H.B_ISO * H.inv(H.Z_SSWU * H.A_ISO) % P if tv1 == 0 else -H.B_ISO * H.inv(H.A_ISO) * (1 + H.inv(tv1)) % P


def u_gx1(square: bool, seed: int):
    """a u whose g(x1) is (not) a square"""
    rnd = random.Random(seed)
    while True:
        u = rnd.randrange(P)
        if (H.sqrt(H.g_iso(_x1(u))) is not None) == square:
            return u


def special_us():
    """(name, u) for the map's branches: tv1 = 0 (u = 0 and Z u^2 = -1, i.e. u = +-sqrt(-1/11)), g(x1) square and not,
    and the ends of the field"""
    r = H.sqrt(-H.inv(H.Z_SSWU) % P)
    assert r is not None  # -1 and 11 are both non-residues
    return [("u=0", 0), ("u=sqrt(-1/Z)", r), ("u=-sqrt(-1/Z)", P - r), ("gx1-nonsquare", u_gx1(False, 11)),
            ("gx1-square", u_gx1(True, 12)), ("u=1", 1), ("u=p-1", P - 1)]


def e1_non_subgroup_points(count, seed=21):
    """points of E1(Fp) outside G1 (random x with x^3 + 4 a square)"""
    rnd = random.Random(seed)
    out = []
    while len(out) < count:
        x = rnd.randrange(P)
        y = H.sqrt((x ** 3 + 4) % P)
        if y is not None and not H.in_g1((x, y)):
            out.append((x, y))
    return out


# ---- short signatures ---------------------------------------------------------------------------------------------
def signed(rnd, msg: bytes, dst: bytes = H.DST_G1_NUL, sk=None):
    """(sig48, pk96) of sk H(msg) under dst, sk random unless given"""
    sk = sk or rnd.randrange(1, N)
    return H.sign(sk, H.hash_to_g1(msg, dst)), H.public_key(sk)


def _set_x_g1(x: int, flags: int = 0x80) -> bytes:
    b = bytearray(x.to_bytes(48, "big"))
    b[0] |= flags
    return bytes(b)


def _set_x_g2(x0: int, x1: int, flags: int = 0x80) -> bytes:
    b = bytearray(x1.to_bytes(48, "big") + x0.to_bytes(48, "big"))
    b[0] |= flags
    return bytes(b)


def edge_cases(seed=5):
    """(name, sig48, msg, pk96) covering every branch of the short-verify contract; messages are verified under
    DST_G1_NUL"""
    rnd = random.Random(seed)
    m1, m2 = b"edge message one", b"edge message two"
    sig, pk = signed(rnd, m1)
    sig2, pk2 = signed(rnd, m2)
    out = [("valid", sig, m1, pk), ("valid-2", sig2, m2, pk2), ("valid-empty-message", *_swap(signed(rnd, b""), b""))]
    out += [("wrong-message", sig, m2, pk), ("wrong-key", sig, m1, pk2), ("swapped-sig", sig2, m1, pk)]
    out.append(("wrong-tag", *_swap(signed(rnd, m1, H.DST_G1_POP), m1)))
    out.append(("negated-sig", bytes([sig[0] ^ 0x20]) + sig[1:], m1, pk))  # the sort bit picks -y
    out.append(("sig-identity", bytes([0xC0]) + bytes(47), m1, pk))
    out.append(("pk-identity", sig, m1, bytes([0xC0]) + bytes(95)))
    out.append(("sig-identity-noncanonical", bytes([0xC0]) + bytes(46) + b"\x01", m1, pk))
    q = BC.g1_off_subgroup(rnd)
    out.append(("sig-off-subgroup", H.g1_encode(q), m1, pk))
    q2 = BC.g2_off_subgroup(rnd)
    out.append(("pk-off-subgroup", sig, m1, B.g2_encode(B.G2.fromAffine({"x": q2[0], "y": q2[1]}))))
    out.append(("sig-x>=p", _set_x_g1(P), m1, pk))
    out.append(("sig-x=2^381-1", _set_x_g1(2 ** 381 - 1), m1, pk))
    out.append(("pk-x.c1>=p", sig, m1, _set_x_g2(1, P)))
    out.append(("pk-x.c0>=p", sig, m1, _set_x_g2(P + 1, 0)))
    out.append(("sig-nonsquare", _set_x_g1(BC._nonsquare_g1_x()), m1, pk))
    xn = BC._nonsquare_g2_x()
    out.append(("pk-nonsquare", sig, m1, _set_x_g2(xn[0], xn[1])))
    out.append(("sig-uncompressed-flag", bytes([sig[0] & 0x7F]) + sig[1:], m1, pk))
    out.append(("pk-uncompressed-flag", sig, m1, bytes([pk[0] & 0x7F]) + pk[1:]))
    out.append(("sig-flags-e0", bytes([sig[0] | 0xE0]) + sig[1:], m1, pk))
    out.append(("pk-flags-e0", sig, m1, bytes([pk[0] | 0xE0]) + pk[1:]))
    # a long-signature pair (sig in G2, key in G1) cut and padded into the short sizes
    lsig, _, lpk = BC.keypair_item(rnd)
    out.append(("long-pair-in-short-slots", lsig[:48], m1, lpk + bytes(48)))
    return out


def _swap(sig_pk, msg):
    return sig_pk[0], msg, sig_pk[1]


def signed_triples(count: int, seed: int, keys: int = 16):
    """count valid (sig48, msg, pk96) under DST_G1_NUL with `keys` distinct keys; messages of 0..80 bytes"""
    rnd = random.Random(seed)
    sks = [rnd.randrange(1, N) for _ in range(keys)]
    pks = [H.public_key(sk) for sk in sks]
    out = []
    for k in range(count):
        msg = bytes(rnd.randrange(256) for _ in range(rnd.randrange(81)))
        sk = sks[k % keys]
        out.append((H.sign(sk, H.hash_to_g1(msg, H.DST_G1_NUL)), msg, pks[k % keys]))
    return out


# ---- host build of the device bodies (tests/hostemu/h2g1_emu.cpp) ---------------------------------------------------
_emu = None


def h2g1_emu():
    """ctypes handle of tests/hostemu/libh2g1emu.so, (re)built with g++ when the source or a device header is newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "h2g1_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libh2g1emu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu


def emu_hash(msgs, dst: bytes):
    """[hash_to_g1(m, dst) in the G1 packing] from the host build of k_bls_hash_to_g1's bodies (dst <= 255 bytes)"""
    m, off = pack_messages(msgs)
    n = len(msgs)
    out = ctypes.create_string_buffer(max(96 * n, 1))
    rc = h2g1_emu().emu_h2g1_hash(ctypes.c_char_p(m or b"\0"), ctypes.c_char_p(off), ctypes.c_uint32(n),
                                  ctypes.c_char_p(dst), ctypes.c_uint32(len(dst)), out)
    assert rc == 0
    return [out.raw[96 * k:96 * k + 96] for k in range(n)]


def emu_hash_to_field(msg: bytes, dst: bytes):
    out = ctypes.create_string_buffer(96)
    h2g1_emu().emu_h2g1_hash_to_field(ctypes.c_char_p(msg or b"\0"), ctypes.c_uint64(len(msg)), ctypes.c_char_p(dst),
                                      ctypes.c_uint32(len(dst)), out)
    return [int.from_bytes(out.raw[48 * k:48 * k + 48], "little") for k in range(2)]


def emu_sswu(u: int):
    out = ctypes.create_string_buffer(96)
    h2g1_emu().emu_h2g1_sswu(ctypes.c_char_p(u.to_bytes(48, "little")), out)
    return int.from_bytes(out.raw[:48], "little"), int.from_bytes(out.raw[48:], "little")


def emu_iso_map(pt):
    out = ctypes.create_string_buffer(96)
    h2g1_emu().emu_h2g1_iso_map(ctypes.c_char_p(H.g1_packed(pt)), out)
    return point_from_packed(out.raw)


def emu_clear_cofactor(pt):
    out = ctypes.create_string_buffer(96)
    h2g1_emu().emu_h2g1_clear_cofactor(ctypes.c_char_p(H.g1_packed(pt)), out)
    return point_from_packed(out.raw)


def emu_short_verify(items, chunk=1 << 16):
    """items: (sig48, H affine or None, pk96) -> (verdicts, smallest bad message index or None)"""
    sigs = b"".join(i[0] for i in items)
    pks = b"".join(i[2] for i in items)
    hs = b"".join(H.g1_packed(i[1]) for i in items)
    out = ctypes.create_string_buffer(max(len(items), 1))
    err = (ctypes.c_uint32 * 1)()
    rc = h2g1_emu().emu_short_verify(ctypes.c_char_p(sigs), ctypes.c_char_p(pks), ctypes.c_char_p(hs), len(items),
                                     ctypes.c_uint64(chunk), out, err)
    assert rc == 0
    return [b == 1 for b in out.raw[:len(items)]], (None if err[0] == 0xFFFFFFFF else err[0])
