"""BLS12-381 pairing and BLS signature verification oracle — TEST INFRASTRUCTURE ONLY, never imported by the product.

Written independently of the device formulas (csrc/fp12.cuh, csrc/pairing.cuh):
- Fp6 = Fp2[v]/(v^3 - xi), xi = 1 + u, and Fp12 = Fp6[w]/(w^2 - v) over noble_ref.Field2, with schoolbook products and
  inversion by exponentiation (a^(p^12 - 2));
- Q on the twist is untwisted into E(Fp12), (x, y) -> (x / w^2, y / w^3), and asserted to satisfy y^2 = x^3 + 4;
- a textbook affine Miller loop over |x| with exact tangent / chord lines evaluated at P (vertical lines, which lie in
  Fp6, are dropped), then conjugated because x < 0;
- the final exponentiation is Python's pow with the exponent M (p^12 - 1) / r, where M = 3 is the multiple the
  device's hard-part chain computes (csrc/pairing.cuh).

Elements of Fp12 are ((a0, a1, a2), (b0, b1, b2)) with Fp2 tuples (c0, c1); `flat` / `unflat` give the 12 integers in
the device's memory order."""
from __future__ import annotations

from oracle import noble_ref as R

P = R.BLS12_381_G1_CURVE["p"]
N = R.BLS12_381_G1_CURVE["n"]
X_ABS = 0xD201000000010000  # the curve parameter is x = -X_ABS
M = 3
FINAL_EXP = M * (P ** 12 - 1) // N
F2 = R.Field2(R.Field(P))
XI = (1, 1)
G1 = R.CURVES["bls12_381_G1"]
G2 = R.CURVES["bls12_381_G2"]

Z2, O2 = (0, 0), (1, 0)
Z6, O6 = (Z2, Z2, Z2), (O2, Z2, Z2)
O12 = (O6, Z6)


def f6_add(a, b):
    return tuple(F2.add(x, y) for x, y in zip(a, b))


def f6_sub(a, b):
    return tuple(F2.sub(x, y) for x, y in zip(a, b))


def f6_neg(a):
    return tuple(F2.neg(x) for x in a)


def f6_mul(a, b):
    """schoolbook: sum a_i b_j v^(i+j), v^3 = xi"""
    acc = [Z2] * 5
    for i in range(3):
        for j in range(3):
            acc[i + j] = F2.add(acc[i + j], F2.mul(a[i], b[j]))
    return (F2.add(acc[0], F2.mul(acc[3], XI)), F2.add(acc[1], F2.mul(acc[4], XI)), acc[2])


def f6_mul_v(a):
    return (F2.mul(a[2], XI), a[0], a[1])


def f12_mul(a, b):
    """schoolbook: (a0 + a1 w)(b0 + b1 w), w^2 = v"""
    return (f6_add(f6_mul(a[0], b[0]), f6_mul_v(f6_mul(a[1], b[1]))),
            f6_add(f6_mul(a[0], b[1]), f6_mul(a[1], b[0])))


def f12_sqr(a):
    return f12_mul(a, a)


def f12_conj(a):
    return (a[0], f6_neg(a[1]))


def f12_pow(a, e: int):
    r = O12
    for bit in bin(e)[2:]:
        r = f12_sqr(r)
        if bit == "1":
            r = f12_mul(r, a)
    return r


def f12_inv(a):
    """solve a * z = 1 as a 12 x 12 linear system over Fp (column k = a * basis_k)"""
    cols = []
    for k in range(12):
        e = [0] * 12
        e[k] = 1
        cols.append(flat(f12_mul(a, unflat(e))))
    m = [[cols[c][r] for c in range(12)] + [1 if r == 0 else 0] for r in range(12)]
    for c in range(12):
        piv = next(r for r in range(c, 12) if m[r][c] % P)
        m[c], m[piv] = m[piv], m[c]
        iv = pow(m[c][c], -1, P)
        m[c] = [v * iv % P for v in m[c]]
        for r in range(12):
            if r != c and m[r][c]:
                t = m[r][c]
                m[r] = [(v - t * w) % P for v, w in zip(m[r], m[c])]
    z = unflat([m[r][12] for r in range(12)])
    assert f12_mul(a, z) == O12
    return z


def f12_frobenius(a, k: int = 1):
    return f12_pow(a, P ** k)


def f12_add(a, b):
    return (f6_add(a[0], b[0]), f6_add(a[1], b[1]))


def f12_sub(a, b):
    return (f6_sub(a[0], b[0]), f6_sub(a[1], b[1]))


def from_fp(c: int):
    return (((c % P, 0), Z2, Z2), Z6)


def from_fp2(c):
    return ((c, Z2, Z2), Z6)


def flat(a):
    return [c for f6 in a for f2 in f6 for c in f2]


def unflat(v):
    v = [int(c) for c in v]
    f2 = [(v[2 * k], v[2 * k + 1]) for k in range(6)]
    return ((f2[0], f2[1], f2[2]), (f2[3], f2[4], f2[5]))


W = (Z6, O6)  # w
W_INV = f12_inv(W)
W_INV2, W_INV3 = f12_sqr(W_INV), f12_mul(f12_sqr(W_INV), W_INV)


def untwist(q):
    """(x', y') on y^2 = x^3 + 4 xi over Fp2 -> (x' / w^2, y' / w^3) on y^2 = x^3 + 4 over Fp12"""
    x = f12_mul(from_fp2(q[0]), W_INV2)
    y = f12_mul(from_fp2(q[1]), W_INV3)
    assert f12_sqr(y) == f12_add(f12_mul(f12_sqr(x), x), from_fp(4)), "untwisted point is not on E(Fp12)"
    return x, y


def miller_loop(p, q):
    """f_{|x|,Q}(P), conjugated.  p = (x, y) ints, q = ((x0, x1), (y0, y1)); neither the identity."""
    xp, yp = from_fp(p[0]), from_fp(p[1])
    Q = untwist(q)
    T = Q
    f = O12
    for bit in bin(X_ABS)[3:]:
        # tangent at T: l = yP - yT - s (xP - xT), s = 3 xT^2 / (2 yT)
        xt, yt = T
        s = f12_mul(f12_mul(from_fp(3), f12_sqr(xt)), f12_inv(f12_add(yt, yt)))
        f = f12_mul(f12_sqr(f), f12_sub(f12_sub(yp, yt), f12_mul(s, f12_sub(xp, xt))))
        x3 = f12_sub(f12_sqr(s), f12_add(xt, xt))
        T = (x3, f12_sub(f12_mul(s, f12_sub(xt, x3)), yt))
        if bit == "1":
            xt, yt = T
            xq, yq = Q
            s = f12_mul(f12_sub(yt, yq), f12_inv(f12_sub(xt, xq)))
            f = f12_mul(f, f12_sub(f12_sub(yp, yt), f12_mul(s, f12_sub(xp, xt))))
            x3 = f12_sub(f12_sub(f12_sqr(s), xt), xq)
            T = (x3, f12_sub(f12_mul(s, f12_sub(xt, x3)), yt))
    return f12_conj(f)


def final_exp(f):
    return f12_pow(f, FINAL_EXP)


def is_identity_g1(p) -> bool:
    return p[0] == 0 and p[1] == 0


def is_identity_g2(q) -> bool:
    return q[0] == Z2 and q[1] == Z2


def pairing_product(pairs):
    """prod e(P_i, Q_i) (times M in the exponent); pairs with an identity point contribute 1"""
    f = O12
    for p, q in pairs:
        if is_identity_g1(p) or is_identity_g2(q):
            continue
        f = f12_mul(f, miller_loop(p, q))
    return final_exp(f)


def pairing(p, q):
    return pairing_product([(p, q)])


def pairing_check(pairs) -> bool:
    return pairing_product(pairs) == O12


def affine(pt):
    a = pt.toAffine()
    return a["x"], a["y"]


def torsion_free(pt) -> bool:
    """n P == O by double-and-add (the predicate of noble's isTorsionFree)"""
    return R.naive_mul(type(pt), pt, N).is0()


def bls_verify(sig96: bytes, H, pk48: bytes) -> bool:
    """noble's bls12_381.verify(signature, message, publicKey) for long signatures, with the message already hashed to
    the G2 point H (affine tuples): pk and sig must decode, be non-identity and lie in their subgroups; H must not be
    the identity; then e(pk, H) e(-G1, sig) == 1."""
    if is_identity_g2(H):
        return False
    try:
        pk = R.bls12_381_g1_decode(pk48)
        sig = R.bls12_381_g2_decode(sig96)
    except ValueError:
        return False
    if len(pk48) != 48 or len(sig96) != 96 or is_identity_g1(pk) or is_identity_g2(sig):
        return False
    if not torsion_free(G1.fromAffine({"x": pk[0], "y": pk[1]})):
        return False
    if not torsion_free(G2.fromAffine({"x": sig[0], "y": sig[1]})):
        return False
    neg_g1 = affine(G1.BASE.negate())
    return pairing_check([(pk, H), (neg_g1, sig)])


# ---- encoders (Zcash-flag compressed, bls12-381.ts:377-468) and a signer for tests ---------------------------------
def g1_encode(pt) -> bytes:
    if pt.is0():
        return bytes([0xC0]) + bytes(47)
    x, y = affine(pt)
    b = bytearray(x.to_bytes(48, "big"))
    b[0] |= 0x80 | (0x20 if (2 * y) // P else 0)
    return bytes(b)


def g2_encode(pt) -> bytes:
    if pt.is0():
        return bytes([0xC0]) + bytes(95)
    (x0, x1), (y0, y1) = affine(pt)
    b = bytearray(x1.to_bytes(48, "big") + x0.to_bytes(48, "big"))
    part = y1 if y1 else y0
    b[0] |= 0x80 | (0x20 if (2 * part) // P else 0)
    return bytes(b)


def public_key(sk: int) -> bytes:
    return g1_encode(G1.BASE.multiply(sk))


def sign(sk: int, H_pt) -> bytes:
    """sk H for a G2 point H (noble's sign with the message already hashed)"""
    return g2_encode(H_pt.multiply(sk))
