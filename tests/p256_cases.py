"""P-256 (secp256r1) ECDSA inputs shared by the CPU (hostemu) and GPU tests: signing from the curve equations, the edge
set of the verify contract (oracle.p256_ref.p256_ecdsa_verify), signatures constructed to reach the rare branches of
the check, OpenSSL-signed batches through the `cryptography` package, and P256VERIFY precompile inputs (EIP-7951)."""
import ctypes
import hashlib
import os
import random
import subprocess

from ecdsa_cases import FLAGS, be32, compressed, pack, sig_for, uncompressed  # noqa: F401  (re-exported)
from oracle import p256_ref as PR

PT = PR.P256
N = PR.P256_CURVE["n"]
P = PR.P256_CURVE["p"]
A = PR.P256_CURVE["a"]
B = PR.P256_CURVE["b"]


def rhs(x: int) -> int:
    return (x * x * x + A * x + B) % P


def is_square(v: int) -> bool:
    return pow(v, (P - 1) // 2, P) in (0, 1)


def lift_x(x: int):
    """The point with abscissa x and even y (x^3 - 3x + b must be a square)."""
    y = pow(rhs(x), (P + 1) // 4, P)
    assert y * y % P == rhs(x)
    return PT.fromAffine({"x": x, "y": y if y % 2 == 0 else P - y})


def bits2int_modn(m: bytes) -> int:
    h = int.from_bytes(m, "big")
    if len(m) > 32:
        h >>= 8 * len(m) - 256
    return h % N


def sign_h(d: int, h: int, rnd: random.Random) -> bytes:
    """r || s for the message representative h, normalised to s <= n/2."""
    while True:
        k = rnd.randrange(1, N)
        r = PT.BASE.multiply(k).toAffine()["x"] % N
        s = pow(k, -1, N) * (h + r * d) % N
        if r and s:
            return be32(r) + be32(min(s, N - s))


def _sig_with_s(d: int, s: int, rnd: random.Random):
    """A signature with the given s that verifies with prehash = false (msg = the 32-byte h)."""
    while True:
        k = rnd.randrange(1, N)
        r = PT.BASE.multiply(k).toAffine()["x"] % N
        h = (s * k - r * d) % N
        if r:
            return sig_for(r, s), be32(h)


def edge_cases(seed: int = 7):
    """[(name, sig, msg, pk)]: every item is checked under all four (prehash, lowS) combinations."""
    rnd = random.Random(seed)
    d = rnd.randrange(1, N)
    Q = PT.BASE.multiply(d)
    pk, pk65 = compressed(Q), uncompressed(Q)
    msg = b"edge set"
    good = sign_h(d, bits2int_modn(hashlib.sha256(msg).digest()), rnd)
    r0, s0 = int.from_bytes(good[:32], "big"), int.from_bytes(good[32:], "big")
    out = [("valid", good, msg, pk), ("valid-65", good, msg, pk65),
           ("valid-negated-s", sig_for(r0, N - s0), msg, pk), ("valid-negated-s-65", sig_for(r0, N - s0), msg, pk65)]
    for v in (0, N, N + 1, 2**256 - 1):
        out.append(("r=%x" % v, sig_for(v % 2**256, s0), msg, pk))
        out.append(("s=%x" % v, sig_for(r0, v % 2**256), msg, pk))
    for s in (N >> 1, (N >> 1) + 1):
        sig, m = _sig_with_s(d, s, rnd)
        out.append(("s=%x" % s, sig, m, pk))
    x = Q.toAffine()["x"]
    y = Q.toAffine()["y"]
    bad_keys = {
        "04-on-33": b"\x04" + be32(x), "02-on-65": b"\x02" + be32(x) + be32(y), "05": b"\x05" + be32(x),
        "len0": b"", "len32": be32(x), "len64": be32(x) + be32(y), "len66": pk65 + b"\x00",
        "x=p": b"\x02" + be32(P), "x=p+1": b"\x03" + be32(P + 1), "x>=p-65": b"\x04" + be32(P) + be32(y),
        "y=p-65": b"\x04" + be32(x) + be32(P),
        "off-curve-65": b"\x04" + be32(x) + be32((y + 1) % P), "zero-65": b"\x04" + bytes(64),
        "wrong-parity-33": bytes([2 + 1 - (y & 1)]) + be32(x),
    }
    xn = 1
    while is_square(rhs(xn)):
        xn += 1
    bad_keys["no-sqrt-33"] = b"\x02" + be32(xn)
    for name, k in bad_keys.items():
        out.append(("key-" + name, good, msg, k))
    # empty message: prehash signs sha256(b""), raw signs h = 0 (u1 = 0)
    out.append(("empty-prehash", sign_h(d, bits2int_modn(hashlib.sha256(b"").digest()), rnd), b"", pk))
    out.append(("empty-raw", sign_h(d, 0, rnd), b"", pk))
    for ln in (31, 32, 33, 64, 8192, 8193):
        m = bytes(rnd.randrange(256) for _ in range(ln))
        out.append(("raw-%d" % ln, sign_h(d, bits2int_modn(m), rnd), m, pk))
    for name, hv in (("h=n", N), ("h=n+5", N + 5), ("h=2^256-1", 2**256 - 1)):
        m = be32(hv)
        out.append((name, sign_h(d, bits2int_modn(m), rnd), m, pk))
    out += constructed_cases(seed + 1)
    return out


def constructed_cases(seed: int = 8):
    """Signatures that verify (or not) through the rare branches of the check; msg = the raw 32-byte h.  Each is built
    from the R it must produce as Q = u2^-1 (R - u1 G)."""
    rnd = random.Random(seed)
    out = []
    # R.x >= n: x = n + t for the smallest t >= 1 with x^3 - 3x + b a square (x < p because p - n > 2^127)
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
        out.append((name, sig_for(r, s), be32(h), compressed(Q)))
    # R = O: Q = -(u1 / u2) G
    u1, u2 = rnd.randrange(1, N), rnd.randrange(1, N)
    iu2 = pow(u2, -1, N)
    Q = PT.BASE.multiply((-u1 * iu2) % N)
    r = rnd.randrange(1, N)
    s = r * iu2 % N
    out.append(("R=O", sig_for(r, s), be32(u1 * s % N), compressed(Q)))
    # u1 G == u2 Q: the complete addition doubles
    d = rnd.randrange(1, N)
    u2 = rnd.randrange(1, N)
    u1 = u2 * d % N
    Q = PT.BASE.multiply(d)
    r = PT.BASE.multiply(2 * u1 % N).toAffine()["x"] % N
    s = r * pow(u2, -1, N) % N
    out.append(("u1G=u2Q", sig_for(r, s), be32(u1 * s % N), uncompressed(Q)))
    # u1 = 0 (h = 0): R = u2 Q alone
    d = rnd.randrange(1, N)
    Q = PT.BASE.multiply(d)
    u2 = rnd.randrange(1, N)
    r = Q.multiply(u2).toAffine()["x"] % N
    s = r * pow(u2, -1, N) % N
    out.append(("u1=0", sig_for(r, s), be32(0), compressed(Q)))
    return out


# ---- P256VERIFY (EIP-7951) -------------------------------------------------------------------------------------
def precompile_input(h: bytes, r: int, s: int, qx: int, qy: int) -> bytes:
    return h + be32(r) + be32(s) + be32(qx) + be32(qy)


def precompile_cases(seed: int = 11):
    """[(name, input)]: valid inputs, every field out of range, bad keys and wrong lengths."""
    rnd = random.Random(seed)
    d = rnd.randrange(1, N)
    Q = PT.BASE.multiply(d).toAffine()
    qx, qy = Q["x"], Q["y"]
    h = hashlib.sha256(b"precompile").digest()
    sig = sign_h(d, bits2int_modn(h), rnd)
    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
    hn = be32(N + 3)  # a hash >= n is used modulo n
    sig_hn = sign_h(d, 3, rnd)
    out = [("valid", precompile_input(h, r, s, qx, qy)), ("valid-high-s", precompile_input(h, r, N - s, qx, qy)),
           ("valid-h>=n", precompile_input(hn, int.from_bytes(sig_hn[:32], "big"), int.from_bytes(sig_hn[32:], "big"),
                                           qx, qy)),
           ("wrong-hash", precompile_input(bytes([h[0] ^ 1]) + h[1:], r, s, qx, qy)),
           ("negated-key", precompile_input(h, r, s, qx, P - qy))]
    for v in (0, N, N + 1, 2**256 - 1):
        out.append(("r=%x" % v, precompile_input(h, v, s, qx, qy)))
        out.append(("s=%x" % v, precompile_input(h, r, v, qx, qy)))
    out += [("qx=p", precompile_input(h, r, s, P, qy)), ("qy=p", precompile_input(h, r, s, qx, P)),
            ("qx=qx+p", precompile_input(h, r, s, qx + P, qy) if qx + P < 2**256 else precompile_input(h, r, s, P + 1, qy)),
            ("qy=qy+p", precompile_input(h, r, s, qx, qy + P) if qy + P < 2**256 else precompile_input(h, r, s, qx, P + 1)),
            ("q=(0,0)", precompile_input(h, r, s, 0, 0)), ("off-curve", precompile_input(h, r, s, qx, (qy + 1) % P))]
    good = out[0][1]
    out += [("len0", b""), ("len159", good[:159]), ("len161", good + b"\x00")]
    # R = O and R.x >= n through the constructed signatures (their 32-byte h is the hash)
    for name, sg, m, pk in constructed_cases(seed + 1):
        x, y = _decode(pk)
        out.append(("constructed-" + name, precompile_input(m, int.from_bytes(sg[:32], "big"),
                                                            int.from_bytes(sg[32:], "big"), x, y)))
    return out


def _decode(pk: bytes):
    return PR.p256_decode_sec1(pk)


# ---- OpenSSL (cryptography) ------------------------------------------------------------------------------------
def openssl_sign(n: int, seed: int, compressed_ratio: float = 0.5, prehash: bool = True, msg_len=None):
    """n fresh P-256 keys and signatures from OpenSSL: [(sig64, msg, pk)].  prehash = False signs 32-byte digests as
    given (utils.Prehashed); msg_len: fixed message length (default: random lengths 0..79 with prehash)."""
    ec, hashes, serialization, utils = _crypto()
    rnd = random.Random(seed)
    out = []
    for _ in range(n):
        k = ec.generate_private_key(ec.SECP256R1())
        ln = 32 if not prehash else (msg_len if msg_len is not None else rnd.randrange(0, 80))
        msg = bytes(rnd.randrange(256) for _ in range(ln))
        algo = ec.ECDSA(hashes.SHA256()) if prehash else ec.ECDSA(utils.Prehashed(hashes.SHA256()))
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

    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
    if not (1 <= r < N and 1 <= s < N) or (lowS and s > N >> 1):
        return False
    try:
        pub = ec.EllipticCurvePublicKey.from_encoded_point(ec.SECP256R1(), pk)
    except ValueError:
        return False
    algo = ec.ECDSA(hashes.SHA256()) if prehash else ec.ECDSA(utils.Prehashed(hashes.SHA256()))
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
            s = int.from_bytes(sig[32:], "big")
            sig = sig[:32] + be32(N - s)
        elif kind == 3:
            pk = b"\x05" + pk[1:]
        out.append((sig, msg, pk))
    return out


# ---- host build of the verification bodies (tests/hostemu/p256_emu.cpp) -----------------------------------------
_emu = None


def p256_emu():
    """ctypes handle of tests/hostemu/libp256emu.so, (re)built with g++ when the source or a device header is newer."""
    global _emu
    if _emu is not None:
        return _emu
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "hostemu", "p256_emu.cpp")
    so = os.path.join(root, "tests", "hostemu", "libp256emu.so")
    csrc = os.path.join(root, "noble-curves_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", csrc, src, "-o", so])
    _emu = ctypes.CDLL(so)
    return _emu
