"""Hash to BLS12-381 G2, suite BLS12381G2_XMD:SHA-256_SSWU_RO_ (RFC 9380 §8.8.2; next-row f10): the oracle
nmsm_bls12_381_hash_to_g2_batch and nmsm_bls12_381_verify_msg_batch are checked against.

A plain Python-int restatement of noble-curves' bls12_381.G2.hashToCurve(msg, { DST }) (abstract/hash-to-curve.ts,
bls12-381.ts): expand_message_xmd with hashlib's SHA-256 (§5.3.1, oversize tags per §5.3.3), hash_to_field (§5.2),
the simplified SWU map on E2' (§6.6.2), the 3-isogeny to E2 (§E.3), and clear_cofactor as the scalar multiplication
by h_eff (§8.8.2), not the psi method the device uses.  Points are affine ((x0, x1), (y0, y1)) tuples, None for the
identity.  Test infrastructure only.
"""
from __future__ import annotations

import hashlib

P = 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB
R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
X = -0xD201000000010000  # the BLS parameter
H2 = 0x5D543A95414E7F1091D50792876A202CD91DE4547085ABAA68A205B2E5A7DDFA628F1CB4D9E82EF21537E293A6691AE1616EC6E786F0C70CF1C38E31C7238E5
H_EFF = 0xBC69F08F2EE75B3584C6A0EA91B352888E2A8E9145AD7689986FF031508FFE1329C2F178731DB956D82BF015D1212B02EC0EC69D7477C1AE954CBC06689F6A359894C0ADEBBF6B4E8020005AAA95551
assert H_EFF == 3 * (X * X - 1) * H2

DST_G2_NUL = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_"  # noble's default for long signatures
DST_G2_POP = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_"  # Ethereum consensus
DST_QUUX = b"QUUX-V01-CS02-with-BLS12381G2_XMD:SHA-256_SSWU_RO_"  # RFC 9380 J.10.1


# ---- Fp2 = Fp[u] / (u^2 + 1) ------------------------------------------------------------------------------------
def f2(a0, a1=0):
    return (a0 % P, a1 % P)


def add(a, b):
    return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)


def sub(a, b):
    return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)


def mul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def neg(a):
    return ((-a[0]) % P, (-a[1]) % P)


def inv(a):
    t = pow(a[0] * a[0] + a[1] * a[1], P - 2, P)
    return (a[0] * t % P, (-a[1]) * t % P)


ZERO2, ONE2 = (0, 0), (1, 0)


def sqrt(a):
    """A square root of a in Fp2, or None (p = 3 mod 4: through the norm)"""
    if a == ZERO2:
        return a
    a0, a1 = a
    nrm = (a0 * a0 + a1 * a1) % P
    n = pow(nrm, (P + 1) // 4, P)
    if n * n % P != nrm:
        return None
    half = (P + 1) // 2
    for s in (n, P - n):
        t = (a0 + s) * half % P
        r0 = pow(t, (P + 1) // 4, P)
        if r0 and r0 * r0 % P == t:
            r = (r0, a1 * pow(2 * r0, P - 2, P) % P)
            if mul(r, r) == a:
                return r
    r = (0, pow(-a0 % P, (P + 1) // 4, P))  # a1 = 0 and a0 a non-residue: sqrt(-a0) u
    return r if mul(r, r) == a else None


def sgn0(a):
    """§4.1 for m = 2: sign_0 OR (zero_0 AND sign_1)"""
    return (a[0] & 1) | (int(a[0] == 0) & (a[1] & 1))


# ---- expand_message_xmd and hash_to_field -----------------------------------------------------------------------
def dst_prime_tag(dst: bytes) -> bytes:
    """§5.3.3: a tag longer than 255 bytes is replaced by SHA-256("H2C-OVERSIZE-DST-" || DST)"""
    if len(dst) > 255:
        return hashlib.sha256(b"H2C-OVERSIZE-DST-" + dst).digest()
    return dst


def expand_message_xmd(msg: bytes, dst: bytes, len_in_bytes: int) -> bytes:
    """§5.3.1 with SHA-256 (b_in_bytes = 32, s_in_bytes = 64)"""
    dst = dst_prime_tag(dst)
    ell = (len_in_bytes + 31) // 32
    if ell > 255 or len_in_bytes > 65535:
        raise ValueError("len_in_bytes too large")
    dst_prime = dst + bytes([len(dst)])
    b0 = hashlib.sha256(bytes(64) + msg + len_in_bytes.to_bytes(2, "big") + b"\0" + dst_prime).digest()
    bs = [hashlib.sha256(b0 + b"\1" + dst_prime).digest()]
    for i in range(2, ell + 1):
        bs.append(hashlib.sha256(bytes(x ^ y for x, y in zip(b0, bs[-1])) + bytes([i]) + dst_prime).digest())
    return b"".join(bs)[:len_in_bytes]


def hash_to_field(msg: bytes, dst: bytes):
    """count = 2, m = 2, L = 64: [u0, u1] with u_i = e_{2i} + e_{2i+1} u"""
    uniform = expand_message_xmd(msg, dst, 256)
    e = [int.from_bytes(uniform[64 * k:64 * k + 64], "big") % P for k in range(4)]
    return [(e[0], e[1]), (e[2], e[3])]


# ---- simplified SWU on E2' and the 3-isogeny ----------------------------------------------------------------------
A_ISO, B_ISO, Z_SSWU = f2(0, 240), f2(1012, 1012), f2(-2, -1)


def g_iso(x):
    return add(add(mul(mul(x, x), x), mul(A_ISO, x)), B_ISO)


def map_to_curve_sswu(u):
    """§6.6.2 straight from its definition: the point (x, y) of E2': y^2 = x^3 + A' x + B'"""
    zu2 = mul(Z_SSWU, mul(u, u))
    tv1 = add(mul(zu2, zu2), zu2)
    if tv1 == ZERO2:
        x1 = mul(B_ISO, inv(mul(Z_SSWU, A_ISO)))
    else:
        x1 = mul(mul(neg(B_ISO), inv(A_ISO)), add(ONE2, inv(tv1)))
    x, y = x1, sqrt(g_iso(x1))
    if y is None:
        x = mul(zu2, x1)
        y = sqrt(g_iso(x))
    assert y is not None and mul(y, y) == g_iso(x)
    if sgn0(u) != sgn0(y):
        y = neg(y)
    return x, y


_C = 0x5C759507E8E333EBB5B7A9A47D7ED8532C52D39FD3A042A88B58423C50AE15D5C2638E343D9C71C6238AAAAAAAA97D6
ISO_XNUM = [f2(_C, _C),
            f2(0, 0x11560BF17BAA99BC32126FCED787C88F984F87ADF7AE0C7F9A208C6B4F20A4181472AAA9CB8D555526A9FFFFFFFFC71A),
            f2(0x11560BF17BAA99BC32126FCED787C88F984F87ADF7AE0C7F9A208C6B4F20A4181472AAA9CB8D555526A9FFFFFFFFC71E,
               0x8AB05F8BDD54CDE190937E76BC3E447CC27C3D6FBD7063FCD104635A790520C0A395554E5C6AAAA9354FFFFFFFFE38D),
            f2(0x171D6541FA38CCFAED6DEA691F5FB614CB14B4E7F4E810AA22D6108F142B85757098E38D0F671C7188E2AAAAAAAA5ED1)]
ISO_XDEN = [f2(0, -72), f2(12, -12), ONE2]
_D = 0x1530477C7AB4113B59A4C18B076D11930F7DA5D4A07F649BF54439D87D27E500FC8C25EBF8C92F6812CFC71C71C6D706
ISO_YNUM = [f2(_D, _D),
            f2(0, 0x5C759507E8E333EBB5B7A9A47D7ED8532C52D39FD3A042A88B58423C50AE15D5C2638E343D9C71C6238AAAAAAAA97BE),
            f2(0x11560BF17BAA99BC32126FCED787C88F984F87ADF7AE0C7F9A208C6B4F20A4181472AAA9CB8D555526A9FFFFFFFFC71C,
               0x8AB05F8BDD54CDE190937E76BC3E447CC27C3D6FBD7063FCD104635A790520C0A395554E5C6AAAA9354FFFFFFFFE38F),
            f2(0x124C9AD43B6CF79BFBF7043DE3811AD0761B0F37A1E26286B0E977C69AA274524E79097A56DC4BD9E1B371C71C718B10)]
ISO_YDEN = [f2(-432, -432), f2(0, -216), f2(18, -18), ONE2]


def _poly(coeffs, x):
    r = ZERO2
    for c in reversed(coeffs):
        r = add(mul(r, x), c)
    return r


def iso_map(pt):
    """§E.3: E2' -> E2; a point of the isogeny's kernel maps to the identity (None)"""
    x, y = pt
    xd, yd = _poly(ISO_XDEN, x), _poly(ISO_YDEN, x)
    if xd == ZERO2 or yd == ZERO2:
        return None
    return mul(_poly(ISO_XNUM, x), inv(xd)), mul(y, mul(_poly(ISO_YNUM, x), inv(yd)))


# ---- E2: y^2 = x^3 + 4 (1 + u) -----------------------------------------------------------------------------------
B_E2 = f2(4, 4)


def on_e2(pt) -> bool:
    return pt is None or mul(pt[1], pt[1]) == add(mul(mul(pt[0], pt[0]), pt[0]), B_E2)


def point_add(p1, p2):
    """the affine group law of E2, complete (identity None, P + P, P + (-P))"""
    if p1 is None:
        return p2
    if p2 is None:
        return p1
    if p1[0] == p2[0]:
        if p1[1] != p2[1] or p1[1] == ZERO2:
            return None
        lam = mul(mul(f2(3), mul(p1[0], p1[0])), inv(add(p1[1], p1[1])))
    else:
        lam = mul(sub(p2[1], p1[1]), inv(sub(p2[0], p1[0])))
    x3 = sub(sub(mul(lam, lam), p1[0]), p2[0])
    return x3, sub(mul(lam, sub(p1[0], x3)), p1[1])


def scalar_mul(k: int, pt):
    """k pt for k >= 0 by double-and-add in Jacobian coordinates (one inversion at the end)"""
    if pt is None or k == 0:
        return None
    X1, Y1, Z1 = pt[0], pt[1], ONE2
    acc = None  # (X, Y, Z)

    def dbl(q):
        X, Y, Z = q
        if Y == ZERO2:
            return None
        A, B = mul(X, X), mul(Y, Y)
        C = mul(B, B)
        D = sub(mul(add(X, B), add(X, B)), add(A, C))
        D = add(D, D)
        E = add(add(A, A), A)
        X3 = sub(mul(E, E), add(D, D))
        C8 = add(C, C)
        C8 = add(C8, C8)
        C8 = add(C8, C8)
        return X3, sub(mul(E, sub(D, X3)), C8), mul(add(Y, Y), Z)

    def madd(q):  # q + (X1, Y1) with Z1 = 1
        if q is None:
            return (X1, Y1, Z1)
        X, Y, Z = q
        ZZ = mul(Z, Z)
        U2, S2 = mul(X1, ZZ), mul(Y1, mul(ZZ, Z))
        H, Rr = sub(U2, X), sub(S2, Y)
        if H == ZERO2:
            return dbl(q) if Rr == ZERO2 else None
        HH = mul(H, H)
        HHH = mul(HH, H)
        V = mul(X, HH)
        X3 = sub(sub(mul(Rr, Rr), HHH), add(V, V))
        return X3, sub(mul(Rr, sub(V, X3)), mul(Y, HHH)), mul(Z, H)

    for bit in bin(k)[2:]:
        if acc is not None:
            acc = dbl(acc)
        if bit == "1":
            acc = madd(acc)
    if acc is None:
        return None
    zi = inv(acc[2])
    zi2 = mul(zi, zi)
    return mul(acc[0], zi2), mul(acc[1], mul(zi2, zi))


def clear_cofactor(pt):
    return scalar_mul(H_EFF, pt)


def in_g2(pt) -> bool:
    return scalar_mul(R, pt) is None


def map_to_curve(u):
    """map_to_curve of the suite: iso_map(simplified SWU(u)), a point of E2 (None: the identity)"""
    return iso_map(map_to_curve_sswu(u))


def hash_to_g2(msg: bytes, dst: bytes = DST_G2_NUL):
    """hash_to_curve (§3): clear_cofactor(map_to_curve(u0) + map_to_curve(u1))"""
    if not isinstance(msg, (bytes, bytearray)) or not isinstance(dst, (bytes, bytearray)):
        raise TypeError("bytes expected")
    if len(dst) == 0:
        raise ValueError("DST must be non-empty")
    u0, u1 = hash_to_field(bytes(msg), bytes(dst))
    return clear_cofactor(point_add(map_to_curve(u0), map_to_curve(u1)))


def g2_packed(pt) -> bytes:
    """the G2 packing of include/nmsm.h: x.c0, x.c1, y.c0, y.c1, 48 B little-endian each; the identity is all zero"""
    if pt is None:
        return bytes(192)
    (x0, x1), (y0, y1) = pt
    return b"".join(v.to_bytes(48, "little") for v in (x0, x1, y0, y1))
