"""P-384 (secp384r1) ECDSA inputs shared by the CPU (hostemu) and GPU tests: signing from the curve equations, the edge
set of the verify contract (oracle.p384_ref.p384_ecdsa_verify), signatures constructed to reach the rare branches of
the check, and OpenSSL-signed batches through the `cryptography` package."""
import hashlib
import os
import random
import subprocess

from ecdsa_cases import FLAGS, pack  # noqa: F401  (re-exported)
from oracle import p384_ref as PR

PT = PR.P384
N = PR.P384_CURVE["n"]
P = PR.P384_CURVE["p"]
A = PR.P384_CURVE["a"]
B = PR.P384_CURVE["b"]
bits2int_modn = PR.bits2int_modn


def be48(x: int) -> bytes:
    return x.to_bytes(48, "big")


def compressed(Q) -> bytes:
    a = Q.toAffine()
    return bytes([2 + (a["y"] & 1)]) + be48(a["x"])


def uncompressed(Q) -> bytes:
    a = Q.toAffine()
    return b"\x04" + be48(a["x"]) + be48(a["y"])


def sig_for(r: int, s: int) -> bytes:
    return be48(r) + be48(s)


def rhs(x: int) -> int:
    return (x * x * x + A * x + B) % P


def is_square(v: int) -> bool:
    return pow(v, (P - 1) // 2, P) in (0, 1)


def lift_x(x: int):
    """The point with abscissa x and even y (x^3 - 3x + b must be a square)."""
    y = pow(rhs(x), (P + 1) // 4, P)
    assert y * y % P == rhs(x)
    return PT.fromAffine({"x": x, "y": y if y % 2 == 0 else P - y})


def sign_h(d: int, h: int, rnd: random.Random) -> bytes:
    """r || s for the message representative h, normalised to s <= n/2."""
    while True:
        k = rnd.randrange(1, N)
        r = PT.BASE.multiply(k).toAffine()["x"] % N
        s = pow(k, -1, N) * (h + r * d) % N
        if r and s:
            return sig_for(r, min(s, N - s))


def _sig_with_s(d: int, s: int, rnd: random.Random):
    """A signature with the given s that verifies with prehash = false (msg = the 48-byte h)."""
    while True:
        k = rnd.randrange(1, N)
        r = PT.BASE.multiply(k).toAffine()["x"] % N
        h = (s * k - r * d) % N
        if r:
            return sig_for(r, s), be48(h)


def edge_cases(seed: int = 7):
    """[(name, sig, msg, pk)]: every item is checked under all four (prehash, lowS) combinations."""
    rnd = random.Random(seed)
    d = rnd.randrange(1, N)
    Q = PT.BASE.multiply(d)
    pk, pk97 = compressed(Q), uncompressed(Q)
    msg = b"edge set"
    good = sign_h(d, bits2int_modn(hashlib.sha384(msg).digest()), rnd)
    r0, s0 = int.from_bytes(good[:48], "big"), int.from_bytes(good[48:], "big")
    out = [("valid", good, msg, pk), ("valid-97", good, msg, pk97),
           ("valid-negated-s", sig_for(r0, N - s0), msg, pk), ("valid-negated-s-97", sig_for(r0, N - s0), msg, pk97)]
    for v in (0, N, N + 1, 2**384 - 1):
        out.append(("r=%x" % v, sig_for(v, s0), msg, pk))
        out.append(("s=%x" % v, sig_for(r0, v), msg, pk))
    for s in (N >> 1, (N >> 1) + 1):
        sig, m = _sig_with_s(d, s, rnd)
        out.append(("s=%x" % s, sig, m, pk))
    x = Q.toAffine()["x"]
    y = Q.toAffine()["y"]
    bad_keys = {
        "04-on-49": b"\x04" + be48(x), "02-on-97": b"\x02" + be48(x) + be48(y),
        "00": b"\x00" + be48(x), "01": b"\x01" + be48(x), "05": b"\x05" + be48(x), "05-on-97": b"\x05" + pk97[1:],
        "len0": b"", "len48": be48(x), "len50": pk + b"\x00", "len96": be48(x) + be48(y), "len98": pk97 + b"\x00",
        "x=p": b"\x02" + be48(P), "x=p+1": b"\x03" + be48(P + 1), "x=2^384-1": b"\x02" + be48(2**384 - 1),
        "x>=p-97": b"\x04" + be48(P) + be48(y), "y=p-97": b"\x04" + be48(x) + be48(P),
        "off-curve-97": b"\x04" + be48(x) + be48((y + 1) % P), "zero-97": b"\x04" + bytes(96),
        "zero-49": b"\x02" + bytes(48), "wrong-parity-49": bytes([2 + 1 - (y & 1)]) + be48(x),
    }
    xn = 1
    while is_square(rhs(xn)):
        xn += 1
    bad_keys["no-sqrt-49"] = b"\x02" + be48(xn)
    for name, k in bad_keys.items():
        out.append(("key-" + name, good, msg, k))
    # empty message: prehash signs sha384(b""), raw signs h = 0 (u1 = 0)
    out.append(("empty-prehash", sign_h(d, bits2int_modn(hashlib.sha384(b"").digest()), rnd), b"", pk))
    out.append(("empty-raw", sign_h(d, 0, rnd), b"", pk))
    # raw messages around bits2int's 48 bytes and its 8192-byte limit
    for ln in (47, 48, 49, 8192, 8193):
        m = bytes(rnd.randrange(256) for _ in range(ln))
        out.append(("raw-%d" % ln, sign_h(d, bits2int_modn(m), rnd), m, pk))
    # prehashed messages around SHA-384's 128-byte block and its 16-byte length field (111 + 1 + 16 = 128)
    for ln in (111, 112, 127, 128, 239):
        m = bytes(rnd.randrange(256) for _ in range(ln))
        out.append(("prehash-%d" % ln, sign_h(d, bits2int_modn(hashlib.sha384(m).digest()), rnd), m, pk))
    for name, hv in (("h=n", N), ("h=n+5", N + 5), ("h=2^384-1", 2**384 - 1)):
        m = be48(hv)
        out.append((name, sign_h(d, bits2int_modn(m), rnd), m, pk))
    out += constructed_cases(seed + 1)
    return out


def constructed_cases(seed: int = 8):
    """Signatures that verify (or not) through the rare branches of the check; msg = the raw 48-byte h.  Each is built
    from the R it must produce as Q = u2^-1 (R - u1 G)."""
    rnd = random.Random(seed)
    out = []
    # R.x >= n: x = n + t for the smallest t >= 1 with x^3 - 3x + b a square (x < p because p - n > 2^189)
    t = 1
    while not is_square(rhs(N + t)):
        t += 1
    Rp = lift_x(N + t)
    u1, u2 = rnd.randrange(1, N), rnd.randrange(1, N)
    iu2 = pow(u2, -1, N)
    Q = Rp.subtract(PT.BASE.multiply(u1)).multiply(iu2)
    for name, r in (("Rx>=n", t), ("Rx>=n-r=x", N + t)):  # r = x >= n is out of range: rejected before the check
        s = r * iu2 % N
        h = u1 * s % N
        out.append((name, sig_for(r, s), be48(h), compressed(Q)))
    # R = O: Q = -(u1 / u2) G
    u1, u2 = rnd.randrange(1, N), rnd.randrange(1, N)
    iu2 = pow(u2, -1, N)
    Q = PT.BASE.multiply((-u1 * iu2) % N)
    r = rnd.randrange(1, N)
    s = r * iu2 % N
    out.append(("R=O", sig_for(r, s), be48(u1 * s % N), compressed(Q)))
    # u1 G == u2 Q: the complete addition doubles
    d = rnd.randrange(1, N)
    u2 = rnd.randrange(1, N)
    u1 = u2 * d % N
    Q = PT.BASE.multiply(d)
    r = PT.BASE.multiply(2 * u1 % N).toAffine()["x"] % N
    s = r * pow(u2, -1, N) % N
    out.append(("u1G=u2Q", sig_for(r, s), be48(u1 * s % N), uncompressed(Q)))
    # u1 = 0 (h = 0): R = u2 Q alone
    d = rnd.randrange(1, N)
    Q = PT.BASE.multiply(d)
    u2 = rnd.randrange(1, N)
    r = Q.multiply(u2).toAffine()["x"] % N
    s = r * pow(u2, -1, N) % N
    out.append(("u1=0", sig_for(r, s), be48(0), compressed(Q)))
    return out


# ---- OpenSSL (cryptography) ------------------------------------------------------------------------------------
def openssl_sign(n: int, seed: int, compressed_ratio: float = 0.5, prehash: bool = True, msg_len=None):
    """n fresh P-384 keys and signatures from OpenSSL: [(sig96, msg, pk)].  prehash = False signs 48-byte digests as
    given (utils.Prehashed); msg_len: fixed message length (default: random lengths 0..159 with prehash)."""
    ec, hashes, serialization, utils = _crypto()
    rnd = random.Random(seed)
    out = []
    for _ in range(n):
        k = ec.generate_private_key(ec.SECP384R1())
        ln = 48 if not prehash else (msg_len if msg_len is not None else rnd.randrange(0, 160))
        msg = bytes(rnd.randrange(256) for _ in range(ln))
        algo = ec.ECDSA(hashes.SHA384()) if prehash else ec.ECDSA(utils.Prehashed(hashes.SHA384()))
        r, s = utils.decode_dss_signature(k.sign(msg, algo))
        fmt = serialization.PublicFormat.CompressedPoint if rnd.random() < compressed_ratio \
            else serialization.PublicFormat.UncompressedPoint
        pk = k.public_key().public_bytes(serialization.Encoding.X962, fmt)
        out.append((sig_for(r, s), msg, pk))
    return out


def openssl_verify(sig: bytes, msg: bytes, pk: bytes, prehash: bool = True, lowS: bool = False) -> bool:
    """OpenSSL's verdict, with the reference's lowS rule on top when asked for (OpenSSL accepts high s)."""
    ec, hashes, _, utils = _crypto()
    from cryptography.exceptions import InvalidSignature

    r, s = int.from_bytes(sig[:48], "big"), int.from_bytes(sig[48:], "big")
    if not (1 <= r < N and 1 <= s < N) or (lowS and s > N >> 1):
        return False
    try:
        pub = ec.EllipticCurvePublicKey.from_encoded_point(ec.SECP384R1(), pk)
    except ValueError:
        return False
    algo = ec.ECDSA(hashes.SHA384()) if prehash else ec.ECDSA(utils.Prehashed(hashes.SHA384()))
    try:
        pub.verify(utils.encode_dss_signature(r, s), msg, algo)
        return True
    except InvalidSignature:
        return False


def _crypto():
    from cryptography.hazmat.primitives import hashes, serialization
    from cryptography.hazmat.primitives.asymmetric import ec, utils

    return ec, hashes, serialization, utils


def corrupt(items, seed: int):
    """Scatter invalid items among valid ones: flipped message byte, flipped r byte, s -> n - s (high/low swap),
    broken key prefix.  Returns a new list; about one item in four is touched."""
    rnd = random.Random(seed)
    out = []
    for sig, msg, pk in items:
        kind = rnd.randrange(8)
        if kind == 0 and msg:
            msg = bytes([msg[0] ^ 1]) + msg[1:]
        elif kind == 1:
            sig = bytes([sig[0] ^ 0x80]) + sig[1:]
        elif kind == 2:
            s = int.from_bytes(sig[48:], "big")
            sig = sig[:48] + be48(N - s)
        elif kind == 3:
            pk = b"\x05" + pk[1:]
        out.append((sig, msg, pk))
    return out


# ---- host build of the verification bodies (tests/hostemu/p384_emu.cpp) -----------------------------------------
_emu = None


def p384_emu():
    """ctypes handle of tests/hostemu/libp384emu.so, (re)built with g++ when the source or a device header is newer."""
    global _emu
    if _emu is not None:
        return _emu
    import ctypes

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "p384_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libp384emu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu
