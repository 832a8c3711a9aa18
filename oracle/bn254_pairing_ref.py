"""bn254 pairing oracle — TEST INFRASTRUCTURE ONLY, never imported by the product.

Written independently of the device formulas (csrc/fp12.cuh, csrc/pairing_bn254.cuh) and of the generated constants:
- Fp6 = Fp2[v]/(v^3 - xi), xi = 9 + u, and Fp12 = Fp6[w]/(w^2 - v) over noble_ref.Field2, with schoolbook products and
  inversion by solving a linear system;
- Q on the D-type twist y^2 = x^3 + 3 / xi is untwisted into E(Fp12), (x, y) -> (x w^2, y w^3), and asserted to satisfy
  y^2 = x^3 + 3;
- a textbook affine Miller loop over the bits of 6u + 2 with exact tangent / chord lines evaluated at P (vertical lines,
  which lie in Fp6, are dropped), then the two chords through pi(Q) and -pi^2(Q), where pi is the p-th power of the
  untwisted coordinates;
- the final exponentiation is Python's pow with the exponent M (p^12 - 1) / r, where M = 2u (6u^2 + 3u + 1) is the
  multiple the device's hard-part chain computes (csrc/pairing_bn254.cuh).

Elements of Fp12 are ((a0, a1, a2), (b0, b1, b2)) with Fp2 tuples (c0, c1); `flat` / `unflat` give the 12 integers in
the device's memory order."""
from __future__ import annotations

from oracle import noble_ref as R

P = R.BN254_G1_CURVE["p"]
N = R.BN254_G1_CURVE["n"]
U = 0x44E992B44A6909F1  # the curve parameter (bn254.ts BN_X)
ATE = 6 * U + 2
M = 2 * U * (6 * U * U + 3 * U + 1)
FINAL_EXP = M * (P ** 12 - 1) // N
F2 = R.Field2(R.Field(P))
XI = (9, 1)
G1 = R.CURVES["bn254_G1"]
G2 = R.CURVES["bn254_G2"]

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


def f12_add(a, b):
    return (f6_add(a[0], b[0]), f6_add(a[1], b[1]))


def f12_sub(a, b):
    return (f6_sub(a[0], b[0]), f6_sub(a[1], b[1]))


def f12_pow(a, e: int):
    r = O12
    for bit in bin(e)[2:]:
        r = f12_sqr(r)
        if bit == "1":
            r = f12_mul(r, a)
    return r


def flat(a):
    return [c for f6 in a for f2 in f6 for c in f2]


def unflat(v):
    v = [int(c) for c in v]
    f2 = [(v[2 * k], v[2 * k + 1]) for k in range(6)]
    return ((f2[0], f2[1], f2[2]), (f2[3], f2[4], f2[5]))


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


def from_fp(c: int):
    return (((c % P, 0), Z2, Z2), Z6)


def from_fp2(c):
    return ((c, Z2, Z2), Z6)


W = (Z6, O6)  # w
W2, W3 = f12_sqr(W), f12_mul(f12_sqr(W), W)


def untwist(q):
    """(x', y') on y^2 = x^3 + 3 / xi over Fp2 -> (x' w^2, y' w^3) on y^2 = x^3 + 3 over Fp12"""
    x = f12_mul(from_fp2(q[0]), W2)
    y = f12_mul(from_fp2(q[1]), W3)
    assert f12_sqr(y) == f12_add(f12_mul(f12_sqr(x), x), from_fp(3)), "untwisted point is not on E(Fp12)"
    return x, y


def _line_and_add(f, T, S, xp, yp):
    """f * (line through T and S, or the tangent at T when S == T, at P) and T + S, all affine over Fp12.  When
    S = -T the line is vertical (in Fp6, dropped) and T + S is the identity (None): only the last step can meet it."""
    xt, yt = T
    xs, ys = S
    if T != S and xt == xs:
        assert ys == f12_sub(from_fp(0), yt)
        return f, None
    if T == S:
        s = f12_mul(f12_mul(from_fp(3), f12_sqr(xt)), f12_inv(f12_add(yt, yt)))
    else:
        s = f12_mul(f12_sub(yt, ys), f12_inv(f12_sub(xt, xs)))
    f = f12_mul(f, f12_sub(f12_sub(yp, yt), f12_mul(s, f12_sub(xp, xt))))
    x3 = f12_sub(f12_sub(f12_sqr(s), xt), xs)
    return f, (x3, f12_sub(f12_mul(s, f12_sub(xt, x3)), yt))


def miller_loop(p, q):
    """f_{6u+2,Q}(P) l_{T,pi(Q)}(P) l_{T',-pi^2(Q)}(P).  p = (x, y) ints, q = ((x0, x1), (y0, y1)); neither the
    identity."""
    xp, yp = from_fp(p[0]), from_fp(p[1])
    Q = untwist(q)
    T = Q
    f = O12
    for bit in bin(ATE)[3:]:
        f, T = _line_and_add(f12_sqr(f), T, T, xp, yp)
        if bit == "1":
            f, T = _line_and_add(f, T, Q, xp, yp)
    Q1 = (f12_frobenius(Q[0], 1), f12_frobenius(Q[1], 1))
    Q2 = (f12_frobenius(Q[0], 2), f12_frobenius(Q[1], 2))
    f, T = _line_and_add(f, T, Q1, xp, yp)
    f, _ = _line_and_add(f, T, (Q2[0], f12_sub(from_fp(0), Q2[1])), xp, yp)
    return f


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
