"""Case generator for the arithmetic tests of the device headers: the host build (tests/hostemu, test_hostemu_parity.py)
and the device build (tests/devemu, test_gpu_arith.py) take their inputs from here.

Random inputs almost never reach a carry or borrow at a limb boundary or the final conditional subtraction, so besides
seeded random values every list holds the values where those happen: 0, 1, p - 1, the residues next to powers of 2^32,
R mod p and its relatives, limbs of all-ones / all-zeros / top-bit patterns, and operand pairs whose Montgomery product
is a chosen extreme result.  Expected values are Python integers and the oracles; nothing here restates the device
algorithms."""
import random

from oracle import noble_ref as R

# field id -> (label, modulus, 32-bit limbs); the ids of hostemu emu_field / devemu dev_field
FIELDS = {
    0: ("secp256k1 p", R.SECP256K1_CURVE["p"], 8),
    1: ("ed25519 p", R.ED25519_CURVE["p"], 8),
    2: ("bn254 p", R.BN254_G1_CURVE["p"], 8),
    3: ("BLS12-381 p", R.BLS12_381_G1_CURVE["p"], 12),
    4: ("secp256k1 n", R.SECP256K1_CURVE["n"], 8),
    5: ("ed25519 l", R.ED25519_CURVE["n"], 8),
    6: ("bn254 r", R.BN254_G1_CURVE["n"], 8),
    7: ("BLS12-381 r", R.BLS12_381_G1_CURVE["n"], 8),
}

# op numbers of emu_field / dev_field
MUL, ADD, SUB, INV_XGCD, FROM_MONT_IN, TO_CANON, SQR, NEG, DIVSTEPS, INV_WORDS, INV, IN_RANGE = range(12)
LIMB_PATTERNS = (0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF)


def words(values, n):
    """little-endian 32-bit words of each value, n words per value, as one flat list"""
    out = []
    for v in values:
        out += [(v >> (32 * k)) & 0xFFFFFFFF for k in range(n)]
    return out


def ints(ws, n):
    return [sum(int(ws[i * n + k]) << (32 * k) for k in range(n)) for i in range(len(ws) // n)]


def assert_same(what, got, want, operands):
    """got == want element-wise; otherwise name the operation, the number of mismatches and the first failing case
    with its operands in hex"""
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert len(got) == len(want), (what, len(got), len(want))
    if bad:
        i = bad[0]

        def hx(v):
            return repr(v) if not isinstance(v, int) else hex(v)

        ops = ", ".join(hx(o) for o in operands[i]) if isinstance(operands[i], (tuple, list)) else hx(operands[i])
        raise AssertionError("%s: %d of %d cases wrong; first: case %d operands (%s) got %s want %s"
                             % (what, len(bad), len(got), i, ops, hx(got[i]), hx(want[i])))


def field_values(fid, seed=0, randoms=64):
    """Reduced values in [0, p) that sit on the carry edges of an n-limb Montgomery field, then seeded random ones."""
    _, p, n = FIELDS[fid]
    Rm = 1 << (32 * n)
    rnd = random.Random(1000 * fid + seed)
    v = [0, 1, 2, 3, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, p >> 1, (1 << (p.bit_length() - 1)) % p]
    for k in range(1, n + 1):
        v += [(p - (1 << (32 * k))) % p, ((1 << (32 * k)) - 1) % p]
    v += [Rm % p, Rm * Rm % p, (-Rm) % p, pow(Rm, -1, p), 0x55555555555555555555555555555555 % p, pow(3, 200, p)]
    for pat in LIMB_PATTERNS:  # every limb the same pattern
        v.append(sum(pat << (32 * k) for k in range(n)) % p)
    for _ in range(4 * n):  # limbs drawn from the patterns
        v.append(sum(rnd.choice(LIMB_PATTERNS) << (32 * k) for k in range(n)) % p)
    v += [rnd.randrange(p) for _ in range(randoms)]
    out, seen = [], set()
    for x in v:
        if x not in seen:
            seen.add(x)
            out.append(x)
    return out


def mont_targets(fid):
    """t values for b = t R a^-1: the Montgomery product a b / R then lands on 1, p - 1, p - 2 or R mod p"""
    _, p, n = FIELDS[fid]
    return [1, p - 1, p - 2, (1 << (32 * n)) % p]


def binary_pairs(fid, seed=0, per_value=8):
    """(a, b) operand pairs for *, +, -: every edge value against a sample of the others, plus pairs whose Montgomery
    product is each of mont_targets (b = t R a^-1 mod p)."""
    _, p, n = FIELDS[fid]
    Rm = 1 << (32 * n)
    vals = field_values(fid, seed)
    rnd = random.Random(7000 + 1000 * fid + seed)
    edge = vals[:8]
    pairs = []
    for a in vals:
        for b in rnd.sample(vals, per_value) + edge:
            pairs.append((a, b))
    for a in vals:
        if a:
            for t in mont_targets(fid):
                pairs.append((a, t * Rm * pow(a, -1, p) % p))
    return pairs


def inverse_values(fid, seed=0):
    """non-zero x < p for the inversions, including small and sparse ones (few division steps, long runs of zeros)"""
    _, p, n = FIELDS[fid]
    rnd = random.Random(3000 + 1000 * fid + seed)
    v = [x for x in field_values(fid, seed, randoms=200) if x]
    v += [1 << 30, (1 << 30) - 1, 1 << 60, (1 << 255) % p, (1 << (p.bit_length() - 1)) - 1]
    v += [rnd.randrange(1, 1 << k) % p or 1 for k in (8, 31, 61, 64, 90, 200) for _ in range(5)]
    return v


def unreduced_operands(fid):
    """N-limb integers for mul_wide, reduced or not: up to 2^(32N) - 1"""
    _, p, n = FIELDS[fid]
    top = (1 << (32 * n)) - 1
    rnd = random.Random(5000 + fid)
    v = [0, 1, p - 1, p, p + 1, 2 * p - 2, 2 * p - 1, top, top - 1, 1 << (32 * n - 1), (1 << (32 * n - 1)) - 1]
    for pat in LIMB_PATTERNS:
        v.append(sum(pat << (32 * k) for k in range(n)))
    v += [sum(rnd.choice(LIMB_PATTERNS) << (32 * k) for k in range(n)) for _ in range(16)]
    v += [rnd.randrange(top + 1) for _ in range(16)]
    return v


def wide_pairs(fid):
    v = unreduced_operands(fid)
    rnd = random.Random(5100 + fid)
    return [(a, b) for a in v for b in v[:12]] + [(rnd.choice(v), rnd.choice(v)) for _ in range(200)]


def reduce_wide_inputs(fid):
    """2N-limb T < p R / 2, the contract of mont_reduce_wide: its ends, products of the extreme residues, the double-width
    differences of mul_lazy (t1 - t2 + p R / 4) and random values"""
    _, p, n = FIELDS[fid]
    Rm = 1 << (32 * n)
    lim = p * Rm // 2
    rnd = random.Random(5200 + fid)
    v = [0, 1, lim - 1, lim - 2, p * Rm // 4, p * Rm // 4 - 1, (p - 1) ** 2, (2 * p - 2) ** 2 // 2, p * p, p * Rm // 4 + (p - 1) ** 2,
         p * Rm // 4 - (p - 1) ** 2, Rm - 1, Rm, Rm * (p // 2 - 1),(Rm - 1) * (p - 1) // 2 + p // 2]
    for pat in LIMB_PATTERNS:
        v.append(sum(pat << (32 * k) for k in range(2 * n)) % lim)
    v += [rnd.randrange(lim) for _ in range(200)]
    assert all(0 <= x < lim for x in v)
    return v


def fp2_pairs(fid, seed=0, randoms=300):
    """((a0, a1), (b0, b1)) Montgomery words: every slot from {0, 1, p - 1, ...} so that the coordinate sums of mul_lazy
    reach 2p - 2 and its double-width differences their bounds, then mixed and random ones"""
    _, p, n = FIELDS[fid]
    rnd = random.Random(6000 + fid + seed)
    ext = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (1 << (32 * n - 34)) - 1 if n == 12 else p // 3, (1 << (32 * n)) % p]
    cases = [((a0, a1), (b0, b1)) for a0 in ext[:5] for a1 in ext[:5] for b0 in (0, p - 1, 1) for b1 in (0, p - 1, 2)]
    cases += [((rnd.choice(ext), rnd.choice(ext)), (rnd.choice(ext), rnd.choice(ext))) for _ in range(200)]
    vals = field_values(fid, seed)
    cases += [((rnd.choice(vals), rnd.choice(vals)), (rnd.choice(vals), rnd.choice(vals))) for _ in range(200)]
    cases += [((rnd.randrange(p), rnd.randrange(p)), (rnd.randrange(p), rnd.randrange(p))) for _ in range(randoms)]
    return cases


def warp_inverse_batches(specials, rand, seed=0):
    """batches of n in {1, 5, 31, 32, 33, 71} non-zero values drawn by rand(rnd), each with as many of `specials` (1,
    p - 1, R mod p, ...) as it has room for, at spread-out lanes"""
    rnd = random.Random(9000 + seed)
    out = []
    for n in (1, 5, 31, 32, 33, 71):
        b = [rand(rnd) for _ in range(n)]
        for k, v in enumerate(specials[:n]):
            b[(7 * k + 3) % n if n > len(specials) else k] = v
        out.append(b)
    return out


# ---- group law -------------------------------------------------------------------------------------------------
# curve id -> oracle name; the ids of devemu dev_group (= helpers.CURVE_IDS 0..5)
GROUP_CURVES = {0: "secp256k1", 1: "ed25519", 2: "bn254_G1", 3: "bn254_G2", 4: "bls12_381_G1", 5: "bls12_381_G2"}


def _rand_field_elem(F, rnd):
    if hasattr(F, "Fp"):  # Field2
        p = F.Fp.ORDER
        return (rnd.randrange(1, p), rnd.randrange(1, p))
    return rnd.randrange(1, F.ORDER)


def acc_coords(name, pt, lam):
    """the oracle point as a device accumulator with the projective factor lam: SwXyzz (x l^2, y l^3, l^2, l^3) with the
    identity as (0, 1, 0, 0); EdExt (x l, y l, l, x y l)"""
    P = R.CURVES[name]
    F = P.Fp
    a = pt.toAffine()
    x, y = a["x"], a["y"]
    if name == "ed25519":
        return [F.mul(x, lam), F.mul(y, lam), lam, F.mul(F.mul(x, y), lam)]
    if pt.is0():
        return [F.ZERO, F.ONE, F.ZERO, F.ZERO]
    l2 = F.sqr(lam)
    l3 = F.mul(l2, lam)
    return [F.mul(x, l2), F.mul(y, l3), l2, l3]


def ed25519_small_order_points():
    """the torsion part l Q of random points Q: points of order 1, 2, 4 and 8 (plus (0, -1) and the two of order 4)"""
    P = R.CURVES["ed25519"]
    p, d, l = R.ED25519_CURVE["p"], R.ED25519_CURVE["d"], R.ED25519_CURVE["n"]
    rnd = random.Random(17)
    out = [P.fromAffine({"x": 0, "y": p - 1}), P.fromAffine({"x": R.ED25519_SQRT_M1, "y": 0})]
    while len(out) < 6:
        y = rnd.randrange(p)
        ok, x = R.ed25519_uv_ratio((y * y - 1) % p, (d * y * y + 1) % p)[:2]
        if not ok:
            continue
        t = P.fromAffine({"x": x, "y": y}).multiplyUnsafe(l - 1)
        t = t.add(P.fromAffine({"x": x, "y": y}))
        if not t.double().double().is0():  # order 8
            out.append(t)
    return out


def group_cases(cid, count=64, seed=0):
    """(kind, p point, p lambda, q point, q lambda) for dev_group: generic sums, P + P (same and other representative),
    P + (-P), the identity on either side or both, and the curve's special points (small order for ed25519, outside the
    prime-order subgroup for BLS12-381).  The kinds cycle, so consecutive cases (the quads of one warp) differ."""
    import helpers as H

    name = GROUP_CURVES[cid]
    P = R.CURVES[name]
    F = P.Fp
    rnd = random.Random(4000 + 100 * cid + seed)
    n = P.Fn.ORDER
    one = F.ONE
    rp = lambda: P.BASE.multiplyUnsafe(rnd.randrange(1, n))  # noqa: E731
    lam = lambda: _rand_field_elem(F, rnd)  # noqa: E731
    special = []
    if name == "ed25519":
        special = ed25519_small_order_points()
    elif name == "bls12_381_G1":
        special = H.bls_g1_non_subgroup_points(4)
    elif name == "bls12_381_G2":
        special = H.bls_g2_non_subgroup_points(2)
    kinds = ["generic", "same", "same-rep", "opposite", "id-left", "id-right", "id-both", "special"]
    out = []
    for i in range(count):
        kind = kinds[i % len(kinds)]
        a = rp()
        if kind == "generic":
            out.append((kind, a, lam(), rp(), lam()))
        elif kind == "same":
            out.append((kind, a, one, a, one))
        elif kind == "same-rep":
            out.append((kind, a, lam(), a, lam()))
        elif kind == "opposite":
            out.append((kind, a, lam(), a.negate(), lam()))
        elif kind == "id-left":
            out.append((kind, P.ZERO, lam(), a, lam()))
        elif kind == "id-right":
            out.append((kind, a, lam(), P.ZERO, lam()))
        elif kind == "id-both":
            out.append((kind, P.ZERO, lam(), P.ZERO, lam()))
        elif special:
            s = special[(i // len(kinds)) % len(special)]
            other = [a, s, s.negate(), special[(i // len(kinds) + 1) % len(special)]][(i // len(kinds)) % 4]
            out.append((kind, s, lam(), other, lam()))
        else:
            out.append((kind, a, lam(), a.double(), lam()))
    return out
