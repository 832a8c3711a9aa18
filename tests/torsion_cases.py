"""Points of small and mixed order on the curves with a cofactor, and the scalars that walk them through the identity.

A point outside the prime-order subgroup is what a subgroup check must reject and what cofactor clearing, isSmallOrder
and the *_ANY MSM ids take as input.  Random points outside the subgroup have a huge order, so a scalar multiplication
of one never meets the identity on the way.  The points here have a torsion part T of small order q: multiplying
P + T runs through O, T and -T, which reaches the exceptional branches of the device formulas (P = +-Q in madd / add,
identity table entries, warps whose results are all O, bucket sums that cancel).

Every expected value of the tests built on these cases comes from mul_any (plain double-and-add over the oracle's
complete add / double) or the oracle itself, never from the library.  Shared by test_torsion_cpu.py (hostemu) and
test_gpu_torsion.py.
"""
import functools
import random

import arith_cases as A
import helpers as H
from oracle import noble_ref as R

r_of = lambda name: R.CURVES[name].Fn.ORDER  # noqa: E731

# group orders #E = h * r of the curves with a cofactor, and small factors q of h with points of order q
_R_BLS = R.BLS12_381_G1_CURVE["n"]
_R_BN = R.BN254_G1_CURVE["n"]
COFACTOR = {
    "ed25519": R.ED25519_CURVE["h"],
    "bls12_381_G1": R.BLS12_381_G1_CURVE["h"],  # 3 * 11^2 * 10177^2 * 859267^2 * 52437899^2
    "bls12_381_G2": R.BLS12_381_G2_CURVE["h"],
    "bn254_G2": 2 * R.BN254_G1_CURVE["p"] - _R_BN,
    "secp256k1": 1,
    "bn254_G1": 1,
}
GROUP_ORDER = {name: COFACTOR[name] * r_of(name) for name in COFACTOR}
SMALL_ORDERS = {
    "ed25519": [2, 4, 8],
    "bls12_381_G1": [3, 11, 10177, 859267, 52437899],
    "bls12_381_G2": [13, 23, 2713, 11953, 262069],
    "bn254_G2": [10069, 5864401, 1875725156269],
}
assert COFACTOR["bn254_G2"] == R.BN254_G2_CURVE["h"]
assert COFACTOR["bls12_381_G1"] == 3 * 11**2 * 10177**2 * 859267**2 * 52437899**2
for _name, _qs in SMALL_ORDERS.items():
    assert all(COFACTOR[_name] % q == 0 for q in _qs), _name
# r = 1 mod every small prime of h1: (r - 1) T = O, the last addition of the subgroup check starts from the identity
assert all(_R_BLS % q == 1 for q in SMALL_ORDERS["bls12_381_G1"])
assert _R_BLS % 13 == 7 and _R_BLS % 23 == 8
assert R.ED25519_CURVE["n"] % 8 == 5

# curve name -> the ids of the C ABI that run it
IDS = {"secp256k1": [0], "ed25519": [1], "bn254_G1": [2], "bn254_G2": [3], "bls12_381_G1": [4, 6],
       "bls12_381_G2": [5, 7]}
NAME_OF_ID = {cid: name for name, ids in IDS.items() for cid in ids}
ID_NAME = {0: "secp256k1", 1: "ed25519", 2: "bn254_G1", 3: "bn254_G2", 4: "bls12_381_G1", 5: "bls12_381_G2",
           6: "bls12_381_G1_any", 7: "bls12_381_G2_any"}
WITH_COFACTOR = ["ed25519", "bn254_G2", "bls12_381_G1", "bls12_381_G2"]


def mul_any(P, k):
    """k * P for any integer k >= 0 by plain double-and-add over the oracle's add / double.  The oracle's multiplyUnsafe
    rejects k >= r, and its wNAF walk should not be the only reference on points outside the subgroup."""
    assert k >= 0
    acc, base = type(P).ZERO, P
    while k:
        if k & 1:
            acc = acc.add(base)
        base = base.double()
        k >>= 1
    return acc


_MEMO = {}


def expected(name, P, k):
    """H.expected_tuple of mul_any(P, k), memoised on (curve, affine P, k): the CPU and GPU tests share the values."""
    key = (name, H.point_bytes(name, P), k)
    if key not in _MEMO:
        _MEMO[key] = H.expected_tuple(name, mul_any(P, k))
    return _MEMO[key]


def expected_sum(name, pts, scalars):
    """sum_i k_i P_i with k_i taken as integers (repeated points are folded first, so tiled sets stay cheap)."""
    folded = {}
    for P, k in zip(pts, scalars):
        b = H.point_bytes(name, P)
        folded[b] = (P, folded.get(b, (P, 0))[1] + k)
    acc = R.CURVES[name].ZERO
    for P, k in folded.values():
        acc = acc.add(mul_any(P, k))
    return H.expected_tuple(name, acc)


def random_point(name, rnd):
    """A uniformly random point of E (or the twist E'): its order is almost surely a large multiple of r."""
    P = R.CURVES[name]
    if name == "ed25519":
        p, d = R.ED25519_CURVE["p"], R.ED25519_CURVE["d"]
        while True:
            y = rnd.randrange(p)
            ok, x = R.ed25519_uv_ratio((y * y - 1) % p, (d * y * y + 1) % p)[:2]
            if ok:
                return P.fromAffine({"x": x, "y": y})
    if name == "bls12_381_G1":
        p = P.Fp.ORDER
        while True:
            x = rnd.randrange(p)
            y2 = (x**3 + 4) % p
            y = pow(y2, (p + 1) // 4, p)
            if y * y % p == y2:
                return P.fromAffine({"x": x, "y": y})
    F2 = P.Fp
    b = R.BLS12_381_G2_CURVE["b"] if name == "bls12_381_G2" else R.BN254_G2_CURVE["b"]
    while True:
        x = (rnd.randrange(F2.Fp.ORDER), rnd.randrange(F2.Fp.ORDER))
        try:
            y = F2.sqrt(F2.add(F2.mul(F2.sqr(x), x), b))
        except ValueError:
            continue
        return P.fromAffine({"x": x, "y": y})


def small_order_point(name, q, rnd):
    """A point T of prime order q: the q-part (#E / q^e) Q of a random point Q (q^e the largest power of q dividing
    #E), retried while it is O, then multiplied by q while that is not O.  #E / q alone would not do: where q^2 divides
    h the q-torsion can be all of Z/q x Z/q (BLS12-381 G1 for q = 11), and (#E / q) Q is then always O."""
    qe = q
    while GROUP_ORDER[name] % (qe * q) == 0:
        qe *= q
    while True:
        T = mul_any(random_point(name, rnd), GROUP_ORDER[name] // qe)
        if not T.is0():
            break
    while not mul_any(T, q).is0():
        T = mul_any(T, q)
    assert mul_any(T, q).is0() and not T.is0()
    return T


def _norm(name, pts):
    return R.normalizeZ(R.CURVES[name], pts)


@functools.lru_cache(maxsize=None)
def points(name):
    """[(kind, point, q)]: kind in subgroup / small / mixed / random / identity; q is the order of the torsion part
    (1 for subgroup points and the identity, 0 where it is not known: random points of E outside the subgroup).
    A few tens of points per curve; the large tests tile them."""
    P = R.CURVES[name]
    r = P.Fn.ORDER
    rnd = random.Random("torsion-" + name)
    sub = [P.BASE.multiplyUnsafe(rnd.randrange(1, r)) for _ in range(3)]
    out = [("subgroup", s, 1) for s in sub]
    if name in ("secp256k1", "bn254_G1"):
        return tuple(_finish(name, out + [("identity", P.ZERO, 1)]))
    if name == "ed25519":
        small = []
        for T in A.ed25519_small_order_points():
            q = next(o for o in (1, 2, 4, 8) if mul_any(T, o).is0())
            small.append((T, q))
    else:
        small = [(small_order_point(name, q, rnd), q) for q in SMALL_ORDERS[name]]
        small.append((small[0][0].negate(), small[0][1]))  # -T next to T
    out += [("small", T, q) for T, q in small]
    for j, (T, q) in enumerate(small[:3]):
        out.append(("mixed", sub[j].add(T), q))
    if name == "bls12_381_G1":
        rand = H.bls_g1_non_subgroup_points(2)
    elif name == "bls12_381_G2":
        rand = H.bls_g2_non_subgroup_points(2)
    else:
        rand = [random_point(name, rnd) for _ in range(2)]
    out += [("random", Q, 0) for Q in rand]
    out.append(("identity", P.ZERO, 1))
    return tuple(_finish(name, out))


def _finish(name, out):
    pts = _norm(name, [p for _, p, _ in out])
    return [(kind, p, q) for (kind, _, q), p in zip(out, pts)]


def scalars_for(name, q, rnd):
    """1, 2, q - 1, q, q + 1, 2q, a random multiple of q, r - 1, r - 2, (r - 1) / 2, h where h < r, random values;
    every one in [1, r)."""
    r, h = r_of(name), COFACTOR[name]
    ks = [1, 2, r - 1, r - 2, (r - 1) // 2, rnd.randrange(1, r), rnd.randrange(1, r)]
    if h < r and h > 1:
        ks.append(h)
    if q > 1:
        ks += [q - 1, q, q + 1, 2 * q, q * rnd.randrange(1, r // q)]
    return list(dict.fromkeys(k for k in ks if 0 < k < r))


@functools.lru_cache(maxsize=None)
def mul_cases(name):
    """[(point, k)] over points(name), with scalars_for the order of each point's torsion part."""
    rnd = random.Random("torsion-scalars-" + name)
    return tuple((p, k) for _, p, q in points(name) for k in scalars_for(name, q, rnd))


def small_points(name):
    return [(p, q) for kind, p, q in points(name) if kind == "small"]


@functools.lru_cache(maxsize=None)
def msm_sets(name):
    """[(label, points, scalars)] for MSMs over points outside the subgroup:
    mixed   every point of points(name), scalars random or multiples of the torsion order;
    cancel  S_a + T and S_b - T with equal scalars, T and -T with equal scalars, T twice with scalars summing to q:
            the torsion parts cancel inside buckets and across windows;
    zero    small-order points only, scalars summing to 0 mod q per point: the sum is O."""
    P = R.CURVES[name]
    r = P.Fn.ORDER
    rnd = random.Random("torsion-msm-" + name)
    pl = points(name)
    sub = [p for kind, p, _ in pl if kind == "subgroup"]
    small = small_points(name)
    pts = [p for _, p, _ in pl]
    sc = []
    for _, _, q in pl:
        sc.append(rnd.choice([q, r - 1, q * rnd.randrange(1, r // q)]) if q > 1 else rnd.randrange(r))
    sets = [("mixed", pts, sc)]
    cp, cs = [], []
    for j, (T, q) in enumerate(small[:3]):
        s = rnd.randrange(1, r)
        a = rnd.randrange(1, q)
        cp += [sub[j].add(T), sub[(j + 1) % len(sub)].add(T.negate()), T, T.negate(), T, T]
        cs += [s, s, s, s, a, q - a]
    sets.append(("cancel", _norm(name, cp), cs))
    zp, zs = [], []
    for T, q in small:
        a, b = rnd.randrange(r), rnd.randrange(r)
        c = (-(a + b)) % q + q * rnd.randrange(r // q - 1)
        zp += [T, T, T]
        zs += [a, b, c]
    assert expected_sum(name, zp, zs)[2] == 1
    sets.append(("zero", zp, zs))
    return tuple(sets)


def table_scalars(name, q, bits, rnd, count=6):
    """Scalars for a fixed-point table with `bits`-bit digits whose digits are multiples of q in [0, 2^(bits-1)] (the
    table entries d * 2^(bits j) * T with q | d are the identity for a point T of order q), some with a negative digit
    2^bits - m q (recoded as -(m q) and a carry), and the edge scalars."""
    r = r_of(name)
    half = 1 << (bits - 1)
    mults = [d for d in range(0, half + 1, q)] or [0]
    top = (r.bit_length() - 1) // bits  # digits below this level keep k < r
    out = [1, 2, r - 1, r - 2]
    for i in range(count):
        ds = [rnd.choice(mults) for _ in range(top)]
        if i % 2 and mults[-1] > 0:
            ds[rnd.randrange(top - 1)] = (1 << bits) - rnd.choice(mults[1:])
        k = sum(d << (bits * j) for j, d in enumerate(ds))
        if 0 < k < r:
            out.append(k)
    if q <= half:
        out += [q, half - half % q, q << bits, (q << bits) + q]
    return list(dict.fromkeys(k for k in out if 0 < k < r))
