"""CPU-side verification of the CUDA path's arithmetic and bookkeeping (no GPU needed).

tests/hostemu compiles the *device* headers for the host with an emulated PTX carry flag and runs the
per-thread kernel bodies in loops.  These tests compare that against the oracle bit-for-bit, mirroring
the reference's MSM tests (test/point.test.ts:264-305,685-722,825-862; test/slow-curves.test.ts:185-252)
and field tests (test/modular.test.ts).  The real parity tests (through libnmsm.so on an H100) are in
test_gpu_parity.py.
"""
import random

import pytest

import arith_cases as A
import helpers as H
from oracle import noble_ref as R

ALL = ["secp256k1", "ed25519", "bn254_G1", "bn254_G2", "bls12_381_G1", "bls12_381_G2"]
FIELDS = {fid: p for fid, (_, p, _) in A.FIELDS.items()}


def _fop(field, op, a, b=0):
    return _fop_n(field, op, [a], [b])[0]


def _fop_n(field, op, avals, bvals=None):
    """emu_field_n over a batch: Montgomery / plain words in, ints out"""
    import ctypes

    import numpy as np

    n = A.FIELDS[field][2]
    la = np.array(A.words(avals, n), np.uint32)
    lb = np.array(A.words(bvals if bvals is not None else [0] * len(avals), n), np.uint32)
    out = np.zeros(len(avals) * n, np.uint32)
    cp = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    assert H.hostemu().emu_field_n(field, op, len(avals), cp(la), cp(lb), cp(out)) == 0
    return A.ints(out, n)


def _label(field, op):
    return "%s op %d" % (A.FIELDS[field][0], op)


@pytest.mark.parametrize("field", sorted(A.FIELDS))
def test_field_ops_match_bigint(field):
    """mont_mul/add/sub/neg/sqr/inv/from/to-Montgomery/canonical_in_range vs Python ints (modular.ts:888-1038 semantics),
    for the four base fields and the four scalar fields, on arith_cases' carry-edge values and Montgomery-target pairs."""
    _, p, n = A.FIELDS[field]
    Rm = 1 << (32 * n)
    Ri = pow(Rm, -1, p)
    pairs = A.binary_pairs(field)
    a = [x for x, _ in pairs]
    b = [y for _, y in pairs]
    A.assert_same(_label(field, A.MUL), _fop_n(field, A.MUL, a, b), [x * y * Ri % p for x, y in pairs], pairs)
    A.assert_same(_label(field, A.ADD), _fop_n(field, A.ADD, a, b), [(x + y) % p for x, y in pairs], pairs)
    A.assert_same(_label(field, A.SUB), _fop_n(field, A.SUB, a, b), [(x - y) % p for x, y in pairs], pairs)
    vals = A.field_values(field)
    A.assert_same(_label(field, A.SQR), _fop_n(field, A.SQR, vals), [x * x * Ri % p for x in vals], vals)
    A.assert_same(_label(field, A.NEG), _fop_n(field, A.NEG, vals), [(-x) % p for x in vals], vals)
    A.assert_same(_label(field, A.FROM_MONT_IN), _fop_n(field, A.FROM_MONT_IN, vals), [x * Rm % p for x in vals], vals)
    mont = [x * Rm % p for x in vals]
    A.assert_same(_label(field, A.TO_CANON), _fop_n(field, A.TO_CANON, mont), vals, mont)
    near = vals + [p, p + 1, 2 * p - 1 if 2 * p < Rm else p + 2, Rm - 1, p | 0xFFFFFFFF, p + (1 << 32)]
    near = [x for x in near if x < Rm]
    A.assert_same(_label(field, A.IN_RANGE), [w & 1 for w in _fop_n(field, A.IN_RANGE, near)],
                  [1 if x < p else 0 for x in near], near)
    inv_in = mont[:16]
    A.assert_same(_label(field, A.INV_XGCD), _fop_n(field, A.INV_XGCD, inv_in),
                  [(pow(x, -1, p) * Rm) % p if x else 0 for x in vals[:16]], inv_in)


@pytest.mark.parametrize("field", sorted(A.FIELDS))
def test_divsteps_inverse(field):
    """csrc/inv_divsteps.cuh: batched division-step inversion equals pow(x, -1, p) on plain integers and equals
    field.cuh's inv in Montgomery form, for all eight moduli, on arith_cases' edge values and random ones."""
    _, p, n = A.FIELDS[field]
    Rm = pow(2, 32 * n, p)
    vals = A.inverse_values(field)
    A.assert_same(_label(field, A.INV_WORDS), _fop_n(field, A.INV_WORDS, vals), [pow(x, -1, p) for x in vals], vals)
    xm = [x * Rm % p for x in vals[:60]]
    want = [pow(x, -1, p) * Rm % p for x in vals[:60]]
    for op in (A.DIVSTEPS, A.INV_XGCD, A.INV):
        A.assert_same(_label(field, op), _fop_n(field, op, xm), want, xm)
    assert _fop(field, A.DIVSTEPS, 0) == 0


@pytest.mark.parametrize("field", [2, 3])
def test_fp2_lazy_reduction_multiplication(field):
    """fp2.cuh mul_lazy (Karatsuba on plain double-width products, two Montgomery reductions) against Python integers and
    against the three-multiplication form, on the extreme residues (0, 1, p - 1 in every slot: the operand sums reach
    2p - 2 and the double-width differences their bounds) and random ones."""
    import ctypes
    import random as _r

    import numpy as np

    p = FIELDS[field]
    n = 12 if field == 3 else 8
    Rm = 1 << (32 * n)
    rinv = pow(Rm, -1, p)
    lib = H.hostemu()
    rnd = _r.Random(field)
    ext = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (1 << (32 * n - 34)) - 1 if field == 3 else p // 3]
    cases = [(a0, a1, b0, b1) for a0 in ext[:5] for a1 in ext[:5] for b0 in (0, p - 1, 1) for b1 in (0, p - 1, 2)]
    cases += [tuple(rnd.choice(ext) for _ in range(4)) for _ in range(200)]
    cases += [tuple(rnd.randrange(p) for _ in range(4)) for _ in range(1500)]
    cp = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    for a0, a1, b0, b1 in cases:
        a = H.u32(a0.to_bytes(4 * n, "little") + a1.to_bytes(4 * n, "little"))
        b = H.u32(b0.to_bytes(4 * n, "little") + b1.to_bytes(4 * n, "little"))
        want = ((a0 * b0 - a1 * b1) * rinv % p, (a0 * b1 + a1 * b0) * rinv % p)
        for form in (1, 0):
            out = np.zeros(2 * n, np.uint32)
            assert lib.emu_fp2_mul(field, form, cp(a), cp(b), cp(out)) == 0
            raw = out.tobytes()
            got = (int.from_bytes(raw[: 4 * n], "little"), int.from_bytes(raw[4 * n:], "little"))
            assert got == want, (form, hex(a0), hex(a1), hex(b0), hex(b1))


@pytest.mark.parametrize("name", ALL)
def test_msm_soak(name):
    """test/slow-curves.test.ts:185-252 construction (every 17th scalar zero), several window sizes."""
    nmax = 129 if "G2" not in name else 33
    P, pts, scalars, _ = H.soak_inputs(name, nmax)
    pb, sb = H.pack_points(name, pts), H.pack_scalars(scalars)
    step = len(pb) // nmax
    for size in ([31, 32, 33, 127, 129] if "G2" not in name else [31, 33]):
        exp = H.expected_tuple(name, R.pippenger(P, pts[:size], scalars[:size]))
        for c, L in ((0, 0), (5, 3), (13, 32)):
            got, err, _ = H.emu_msm(name, pb[: size * step], sb[: size * 32], size, c, L)
            assert err == (0xFFFFFFFF, 0xFFFFFFFF)
            assert got == exp, (name, size, c, L)


@pytest.mark.parametrize("name", ALL)
def test_msm_fixed_base_table_route(name):
    """nmsm_points_precompute route: levels 2^(c*j)*P_i, every digit into ONE bucket window (MsmPlan.stride).
    Same soak construction; table window sizes below, at and above the 16-bit limit of the ordinary plan, and
    identity points / cancelling pairs / n-1 scalars so that table levels of O and -P are exercised."""
    nmax = 67 if "G2" not in name else 19
    P, pts, scalars, _ = H.soak_inputs(name, nmax, seed_offset=5)
    pts[3] = P.ZERO
    pts[8] = pts[7].negate()
    scalars[8] = scalars[7]
    scalars[9] = P.Fn.ORDER - 1
    pts = R.normalizeZ(P, pts)
    pb, sb = H.pack_points(name, pts), H.pack_scalars(scalars)
    step = len(pb) // nmax
    for size, c, L in ((nmax, 7, 0), (nmax, 13, 5), (33 if "G2" not in name else 9, 17, 0), (5, 4, 1)):
        exp = H.expected_tuple(name, R.pippenger(P, pts[:size], scalars[:size]))
        got, err, plan = H.emu_msm(name, pb[: size * step], sb[: size * 32], size, 0, L, table_c=c)
        assert err == (0xFFFFFFFF, 0xFFFFFFFF)
        assert plan[0] <= c and plan[1] == 1 and plan[2] == 1 << (plan[0] - 1)  # digit widths are balanced: max width <= c
        assert got == exp, (name, size, c, L)


@pytest.mark.parametrize("name", ["secp256k1", "ed25519", "bls12_381_G1"])
def test_msm_basic_cases(name):
    """test/point.test.ts:264-305: [G]*[0]=O, empty, [O]*[123]=O, [G]*[123], {G,2G,4G,8G}*{3,5,7,11}=129G."""
    P = R.CURVES[name]
    G = P.BASE
    cases = [
        ([G], [0]),
        ([P.ZERO], [123]),
        ([G], [123]),
        ([G, G.double(), G.double().double(), G.double().double().double()], [3, 5, 7, 11]),
        ([G, G.negate()], [5, 5]),  # P + (-P) inside one bucket
        ([G, G], [P.Fn.ORDER - 1, 1]),  # n-1 and 1: cancels to O
        ([G], [P.Fn.ORDER - 1]),
    ]
    for pts, sc in cases:
        pts = R.normalizeZ(P, pts)
        exp = H.expected_tuple(name, R.pippenger(P, pts, sc))
        for c, L in ((0, 0), (2, 1), (16, 4)):
            got, err, _ = H.emu_msm(name, H.pack_points(name, pts), H.pack_scalars(sc), len(pts), c, L)
            assert got == exp, (name, sc, c, L)


@pytest.mark.parametrize("name", ["secp256k1", "bls12_381_G1", "ed25519"])
def test_msm_same_point_same_scalar(name):
    """test/point.test.ts:842-853: L copies of G with scalar 2^10-1 -> equal-operand additions everywhere."""
    P = R.CURVES[name]
    n = 300
    s = 2**10 - 1
    exp = H.expected_tuple(name, P.BASE.multiply((n * s) % P.Fn.ORDER))
    pb = H.point_bytes(name, P.BASE) * n
    for c, L in ((0, 0), (4, 7), (11, 32)):
        got, err, _ = H.emu_msm(name, pb, H.pack_scalars([s] * n), n, c, L)
        assert got == exp, (name, c, L)


def test_msm_validation_indices():
    """curve.ts:390-404: first invalid point / scalar index is reported (points before scalars)."""
    name = "bls12_381_G1"
    P, pts, scalars, _ = H.soak_inputs(name, 20)
    sc = list(scalars)
    sc[7] = P.Fn.ORDER
    sc[11] = P.Fn.ORDER + 5
    _, err, _ = H.emu_msm(name, H.pack_points(name, pts), H.pack_scalars(sc), 20)
    assert err == (0xFFFFFFFF, 7)
    pb = bytearray(H.pack_points(name, pts))
    pb[96 * 5: 96 * 5 + 48] = (P.Fp.ORDER).to_bytes(48, "little")  # x == p: out of range
    _, err, _ = H.emu_msm(name, bytes(pb), H.pack_scalars(sc), 20)
    assert err == (5, 7)


@pytest.mark.parametrize("name", ALL)
def test_mul_batch(name):
    """Point.multiply / multiplyUnsafe (weierstrass.ts:900-928, edwards.ts:555-577) incl. edge scalars."""
    P = R.CURVES[name]
    n_order = P.Fn.ORDER
    rng = R.Xorshift64(0xDEADBEEF)
    base = P.BASE.multiplyUnsafe(rng.rndBelow(n_order - 1) + 1)
    scalars = [1, 2, 3, n_order - 1, n_order - 2, 2**128 - 1, 2**128, 2**64 + 1, 0x5555555555555555 << 60]
    scalars += [rng.rndBelow(n_order - 1) + 1 for _ in range(3 if "G2" in name else 8)]
    scalars = [s % n_order or 1 for s in scalars]
    pts = R.normalizeZ(P, [base] * (len(scalars) - 2) + [P.BASE, P.ZERO])
    res, err = H.emu_mul_batch(name, H.pack_points(name, pts), H.pack_scalars(scalars), len(scalars), False)
    assert err == (0xFFFFFFFF, 0xFFFFFFFF)
    for p, s, got in zip(pts, scalars, res):
        assert got == H.expected_tuple(name, p.multiplyUnsafe(s))
        if not p.is0():
            assert got == H.expected_tuple(name, p.multiply(s))
    # scalar 0: rejected by multiply, identity for multiplyUnsafe; scalar == n rejected by both
    res, err = H.emu_mul_batch(name, H.pack_points(name, pts[:2]), H.pack_scalars([5, 0]), 2, False)
    assert err == (0xFFFFFFFF, 1)
    res, err = H.emu_mul_batch(name, H.pack_points(name, pts[:2]), H.pack_scalars([5, 0]), 2, True)
    assert err == (0xFFFFFFFF, 0xFFFFFFFF) and res[1] == H.expected_tuple(name, P.ZERO)
    res, err = H.emu_mul_batch(name, H.pack_points(name, pts[:2]), H.pack_scalars([n_order, 1]), 2, True)
    assert err == (0xFFFFFFFF, 0)


@pytest.mark.parametrize("name", ALL)
def test_point_table_multiply(name):
    """nmsm_point_table_* bodies (Point.precompute + cached multiply, curve.ts:532-606) with small tables: signed
    digits with carries through every level (n-1, 2^k-1, alternating bits), both scalar ranges."""
    P = R.CURVES[name]
    n_order = P.Fn.ORDER
    rng = R.Xorshift64(0xFACADE)
    base = R.normalizeZ(P, [P.BASE.multiplyUnsafe(rng.rndBelow(n_order - 1) + 1)])[0]
    scalars = [1, 2, 15, 16, 17, 128, 129, 255, 256, n_order - 1, n_order - 2, 2**128 - 1, 2**128,
               0x5555555555555555 << 60, (1 << (n_order.bit_length() - 1)) - 1]
    scalars += [rng.rndBelow(n_order - 1) + 1 for _ in range(2 if "G2" in name else 6)]
    scalars = [s % n_order or 1 for s in scalars]
    pb = H.point_bytes(name, base)
    for tb in ((5, 8) if "G2" not in name else (8,)):
        res, err = H.emu_point_table(name, pb, H.pack_scalars(scalars), len(scalars), False, table_bits=tb)
        assert err == (0xFFFFFFFF, 0xFFFFFFFF)
        for s, got in zip(scalars, res):
            assert got == H.expected_tuple(name, base.multiply(s)), (name, tb, s)
    res, err = H.emu_point_table(name, pb, H.pack_scalars([5, 0, 7]), 3, False)
    assert err == (0xFFFFFFFF, 1) and res[1] is None
    res, err = H.emu_point_table(name, pb, H.pack_scalars([5, 0, 7]), 3, True)
    assert err == (0xFFFFFFFF, 0xFFFFFFFF) and res[1] == H.expected_tuple(name, P.ZERO)
    assert res[2] == H.expected_tuple(name, base.multiplyUnsafe(7))
    res, err = H.emu_point_table(name, pb, H.pack_scalars([n_order, 1]), 2, True)
    assert err == (0xFFFFFFFF, 0) and res[0] is None
    # the identity as the table point: every multiple is the identity
    res, err = H.emu_point_table(name, H.point_bytes(name, P.ZERO), H.pack_scalars([3, n_order - 1]), 2, True)
    assert res == [H.expected_tuple(name, P.ZERO)] * 2


def test_bls12_381_g1_points_outside_the_subgroup():
    """The reference's pippenger / multiply are the plain group law on E(Fp).  Points outside the prime-order subgroup:
    NMSM_BLS12_381_G1_ANY (no GLV) and the multiply batch of either id must match the oracle; the GLV id is only
    specified for torsion-free points (include/nmsm.h), where both ids agree."""
    P = R.CURVES["bls12_381_G1"]
    rng = R.Xorshift64(0xC0FAC7)
    bad = H.bls_g1_non_subgroup_points(5)
    good = [P.BASE.multiplyUnsafe(rng.rndBelow(P.Fn.ORDER - 1) + 1) for _ in range(4)]
    pts = R.normalizeZ(P, bad + good)
    scalars = [rng.rndBelow(P.Fn.ORDER) for _ in pts]
    scalars[1] = P.Fn.ORDER - 1
    exp = H.expected_tuple("bls12_381_G1", R.pippenger(P, pts, scalars))
    pb, sb = H.pack_points("bls12_381_G1", pts), H.pack_scalars(scalars)
    for c, L in ((0, 0), (5, 3)):
        got, err, _ = H.emu_msm("bls12_381_G1_any", pb, sb, len(pts), c, L)
        assert got == exp
    got, _, _ = H.emu_msm("bls12_381_G1_any", pb, sb, len(pts), table_c=9)  # fixed-base table route, no GLV
    assert got == exp
    # subgroup points only: the GLV id and the plain id agree with the oracle
    gp, gs = H.pack_points("bls12_381_G1", pts[5:]), H.pack_scalars(scalars[5:])
    exp_g = H.expected_tuple("bls12_381_G1", R.pippenger(P, pts[5:], scalars[5:]))
    assert H.emu_msm("bls12_381_G1", gp, gs, 4)[0] == exp_g == H.emu_msm("bls12_381_G1_any", gp, gs, 4)[0]
    # Point.multiply on the non-subgroup points (what isTorsionFree / clearCofactor evaluate), both ids
    ks = [P.Fn.ORDER - 1, 0x396C8C005555E1568C00AAAB0000AAAB, 5, rng.rndBelow(P.Fn.ORDER), 1]
    for name in ("bls12_381_G1", "bls12_381_G1_any"):
        res, err = H.emu_mul_batch(name, H.pack_points("bls12_381_G1", pts[:5]), H.pack_scalars(ks), 5, False)
        assert err == (0xFFFFFFFF, 0xFFFFFFFF)
        for pt, k, got in zip(pts[:5], ks, res):
            assert got == H.expected_tuple("bls12_381_G1", pt.multiplyUnsafe(k)), (name, k)


def test_bls12_381_g2_psi_split():
    """BLS12-381 G2 (id 5) splits k four ways along psi (msm_body.cuh gls_split): the device digits against a Python
    statement of the same rule, k = sum (+-mag_i) z^i (mod r) with mag_i < 2^63; single-term MSMs whose scalars select
    each of P, -psi(P), psi^2(P), -psi^3(P) on their own (the constants of curve_consts.cuh Bls381G2Gls) against the
    oracle; and twist points OUTSIDE the prime-order subgroup, where psi is not [x]: NMSM_BLS12_381_G2_ANY (plain
    windows) matches the oracle's pippenger, and nmsm_mul_batch of either id does (multiply never uses psi)."""
    import ctypes
    import random as _r

    import numpy as np

    name = "bls12_381_G2"
    P = R.CURVES[name]
    r = P.Fn.ORDER
    z = 0xD201000000010000
    assert r == z**4 - z**2 + 1
    half = z // 2
    lib = H.hostemu()
    rnd = _r.Random(11)
    cases = [0, 1, 2, r - 1, r - 2, z - 1, z, z + 1, z * z, z**3, z**3 - 1, half, half + 1, half * z, (half + 1) * z**3,
             (half + 1) * (1 + z + z * z + z**3) % r, r // 2, z**3 * (z - 1)]
    cases += [rnd.randrange(r) for _ in range(3000)]
    for k in cases:
        kw = np.frombuffer(k.to_bytes(32, "little"), dtype=np.uint32).copy()
        out = np.zeros(12, np.uint32)
        assert lib.emu_gls_split(kw.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p)) == 0
        mags = [int(out[2 * j]) | (int(out[2 * j + 1]) << 32) for j in range(4)]
        negs = [int(out[8 + j]) for j in range(4)]
        assert all(m < (1 << 63) for m in mags), hex(k)
        assert sum((-m if s else m) * z**j for j, (m, s) in enumerate(zip(mags, negs))) % r == k, hex(k)
    # one term, scalars that isolate the sub-terms (and mixtures with carries)
    base = P.BASE.multiplyUnsafe(0xA5A5F00D1234567)
    for k in [1, z, z * z, z**3, r - 1, r - z, half + 1, (half + 1) * z**3 % r, z**3 + z * z + z + 1] + cases[-6:]:
        for c, L in ((0, 0), (7, 2)):
            got, err, plan = H.emu_msm(name, H.pack_points(name, R.normalizeZ(P, [base])), H.pack_scalars([k]), 1, c, L)
            assert err == (0xFFFFFFFF, 0xFFFFFFFF)
            assert got == H.expected_tuple(name, base.multiplyUnsafe(k) if k else P.ZERO), (hex(k), c)
    assert plan[1] == (64 + 6) // 7  # 63-bit digits + sign: ceil(64 / c) windows
    # fixed-base table over the four-way split set
    pts = R.normalizeZ(P, [P.BASE.multiplyUnsafe(rnd.randrange(1, r)) for _ in range(9)] + [P.ZERO])
    scalars = [rnd.randrange(r) for _ in pts]
    exp = H.expected_tuple(name, R.pippenger(P, pts, scalars))
    pb, sb = H.pack_points(name, pts), H.pack_scalars(scalars)
    assert H.emu_msm(name, pb, sb, len(pts), table_c=9)[0] == exp
    assert H.emu_msm(name, pb, sb, len(pts), 11, 3)[0] == exp == H.emu_msm(name + "_any", pb, sb, len(pts), 11, 3)[0]
    # points outside the subgroup
    bad = R.normalizeZ(P, H.bls_g2_non_subgroup_points(3) + [pts[0]])
    bs = [rnd.randrange(r) for _ in bad]
    exp_bad = H.expected_tuple(name, R.pippenger(P, bad, bs))
    bpb, bsb = H.pack_points(name, bad), H.pack_scalars(bs)
    for c, L in ((0, 0), (6, 3)):
        assert H.emu_msm(name + "_any", bpb, bsb, len(bad), c, L)[0] == exp_bad
    assert H.emu_msm(name + "_any", bpb, bsb, len(bad), table_c=8)[0] == exp_bad
    assert H.emu_msm(name, bpb, bsb, len(bad))[0] != exp_bad  # psi is not [x] off the subgroup: id 5 is not specified there
    ks = [r - 1, 5, rnd.randrange(r)]
    for nm in (name, name + "_any"):
        res, err = H.emu_mul_batch(nm, H.pack_points(name, bad[:3]), H.pack_scalars(ks), 3, False)
        assert err == (0xFFFFFFFF, 0xFFFFFFFF)
        for pt, k, got in zip(bad[:3], ks, res):
            assert got == H.expected_tuple(name, pt.multiplyUnsafe(k)), (nm, k)
    got, _ = H.emu_torsion(name, H.pack_points(name, bad), len(bad))
    assert got == [0, 0, 0, 1]


def test_torsion_free_batch():
    """nmsm_points_torsion_free body (isTorsionFree, weierstrass.ts:971-975 / edwards.ts:584-586) against the oracle's
    n*P == O on subgroup points, points outside the subgroup, small-order points and the identity."""
    G1 = R.CURVES["bls12_381_G1"]
    rng = R.Xorshift64(0x7045)
    pts = H.bls_g1_non_subgroup_points(3) + [G1.BASE.multiplyUnsafe(rng.rndBelow(G1.Fn.ORDER - 1) + 1) for _ in range(3)] + [G1.ZERO]
    pts = R.normalizeZ(G1, pts)
    exp = [1 if p.multiplyUnsafe(G1.Fn.ORDER - 1).add(p).is0() else 0 for p in pts]
    assert exp == [0, 0, 0, 1, 1, 1, 1]
    for name in ("bls12_381_G1", "bls12_381_G1_any"):
        got, err = H.emu_torsion(name, H.pack_points("bls12_381_G1", pts), len(pts))
        assert got == exp and err[0] == 0xFFFFFFFF
    ED = R.CURVES["ed25519"]
    p = ED.Fp.ORDER
    t2 = ED.fromAffine({"x": 0, "y": p - 1})  # order 2
    base = ED.BASE.multiplyUnsafe(12345)
    epts = R.normalizeZ(ED, [base, t2, base.add(t2), ED.ZERO, ED.BASE])
    got, _ = H.emu_torsion("ed25519", H.pack_points("ed25519", epts), len(epts))
    assert got == [1, 0, 0, 1, 1]
    S = R.CURVES["secp256k1"]
    spts = R.normalizeZ(S, [S.BASE, S.BASE.multiplyUnsafe(77), S.ZERO])
    got, _ = H.emu_torsion("secp256k1", H.pack_points("secp256k1", spts), 3)
    assert got == [1, 1, 1]
    bad = bytearray(H.pack_points("secp256k1", spts))
    bad[64:96] = b"\xff" * 32
    _, err = H.emu_torsion("secp256k1", bytes(bad), 3)
    assert err[0] == 1


def test_glv_split_and_constants():
    """BLS12-381 G1 GLV: k = v1 + v2*lambda (mod r), |v| < 2^127, and phi(P) = (beta*x, y) = lambda*P."""
    import ctypes
    import random as _r

    import numpy as np

    P = R.CURVES["bls12_381_G1"]
    r, p = P.Fn.ORDER, P.Fp.ORDER
    lam = 0xD201000000010000**2 - 1
    beta = 0x1A0111EA397FE699EC02408663D4DE85AA0D857D89759AD4897D29650FB85F9B409427EB4F49FFFD8BFD00000000AAAC
    assert lam * lam + lam + 1 == r and pow(beta, 3, p) == 1
    g = P.BASE.toAffine()
    assert R.affine_tuple(P, P.BASE.multiplyUnsafe(lam)) == (beta * g["x"] % p, g["y"])
    rnd = _r.Random(5)
    ks = [0, 1, 2, lam - 1, lam, lam + 1, lam // 2, lam // 2 + 1, lam // 2 + 2, r - 1, r - 2, r - lam, r - lam - 1,
          lam * (lam // 2), lam * (lam // 2 + 1), lam * (lam // 2 + 1) + lam // 2 + 1]
    ks += [rnd.randrange(r) for _ in range(3000)]
    lib = H.hostemu()
    for k in ks:
        a = H.u32(k.to_bytes(32, "little"))
        out = np.zeros(10, np.uint32)
        lib.emu_glv_split(a.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p))
        m1 = int.from_bytes(out[:4].tobytes(), "little")
        m2 = int.from_bytes(out[4:8].tobytes(), "little")
        v1 = -m1 if out[8] else m1
        v2 = -m2 if out[9] else m2
        assert (v1 + v2 * lam - k) % r == 0 and m1 < 2**127 and m2 < 2**127, hex(k)


@pytest.mark.parametrize("name", ["bls12_381_G1", "secp256k1"])
def test_msm_giant_bucket_tile_stitching(name):
    """One bucket spanning thousands of accumulate segments (all scalars equal) exercises both tile levels."""
    P = R.CURVES[name]
    n = 2600
    s = 0x0F0F
    exp = H.expected_tuple(name, P.BASE.multiply((n * s) % P.Fn.ORDER))
    pb = H.point_bytes(name, P.BASE) * n
    got, err, plan = H.emu_msm(name, pb, H.pack_scalars([s] * n), n, 4, 1)  # L = 1: 2600 segments per bucket
    assert got == exp, plan
    got, err, plan = H.emu_msm(name, pb, H.pack_scalars([s] * n), n, 4, 2)
    assert got == exp, plan


# ---- ed25519 batch verification pieces (next-row f1) --------------------------------------------
def _emu_ed_verify(sigs, msgs, pks, z):
    import ctypes
    import struct

    lib = H.hostemu()
    n = len(sigs)
    offs = [0]
    for m in msgs:
        offs.append(offs[-1] + len(m))
    ok, bad = ctypes.c_int(0), ctypes.c_longlong(-1)
    rc = lib.emu_ed25519_verify_batch(b"".join(sigs), b"".join(pks), b"".join(msgs) or b"\0",
                                      struct.pack("<%dQ" % (n + 1), *offs), n, z, ctypes.byref(ok), ctypes.byref(bad))
    assert rc == 0
    return bool(ok.value), int(bad.value)


def test_ed25519_decompress_and_sha512_match_oracle():
    import ctypes
    import hashlib

    import numpy as np

    from conftest import load_golden

    lib = H.hostemu()
    g = load_golden("ed25519.json")
    encs = [bytes.fromhex(v["pk"]) for v in g["vectors"][:24]] + [bytes.fromhex(v["vk_bytes"]) for v in g["zip215"][:40]]
    encs += [bytes.fromhex(v["sig_bytes"])[:32] for v in g["zip215"][40:80]]
    encs += [bytes([2] + [0] * 31), bytes([0xFF] * 32), bytes([0xEC] + [0xFF] * 30 + [0x7F])]
    for e in encs:
        out = np.zeros(16, np.uint32)
        ok = lib.emu_ed25519_decompress(e, out.ctypes.data_as(ctypes.c_void_p))
        try:
            P = R.ed25519_point_from_bytes(e, True)
            assert ok == 1
            a = P.toAffine()
            assert int.from_bytes(out[:8].tobytes(), "little") == a["x"] % R.ED25519_CURVE["p"]
            assert int.from_bytes(out[8:].tobytes(), "little") == a["y"] % R.ED25519_CURVE["p"]
        except ValueError:
            assert ok == 0, e.hex()
    for mlen in (0, 1, 47, 48, 63, 64, 111, 112, 127, 128, 200, 1000):
        r, a, m = bytes(range(32)), bytes(range(32, 64)), bytes((7 * i) & 255 for i in range(mlen))
        d = ctypes.create_string_buffer(64)
        lib.emu_sha512_rAM(r, a, m or b"\0", ctypes.c_uint64(mlen), d)
        assert d.raw == hashlib.sha512(r + a + m).digest(), mlen


def test_ed25519_batch_verify_matches_individual_reference_verify():
    """batch accepts <=> every individual verify (edwards.ts:942-989) accepts; incl. ZIP-215 cases."""
    from conftest import load_golden

    g = load_golden("ed25519.json")
    vec = g["vectors"][:12]
    sigs = [bytes.fromhex(v["sig"]) for v in vec]
    msgs = [bytes.fromhex(v["msg"]) for v in vec]
    pks = [bytes.fromhex(v["pk"]) for v in vec]
    z = bytes((i * 37 + 11) & 255 for i in range(16 * len(vec)))
    assert all(R.ed25519_verify(s, m, p) for s, m, p in zip(sigs, msgs, pks))
    assert _emu_ed_verify(sigs, msgs, pks, z) == (True, -1)
    bad = list(sigs)
    b = bytearray(bad[5])
    b[40] ^= 1  # corrupt s of one signature: individual verify fails, batch must fail
    bad[5] = bytes(b)
    assert R.ed25519_verify(bad[5], msgs[5], pks[5]) is False
    assert _emu_ed_verify(bad, msgs, pks, z)[0] is False
    m2 = list(msgs)
    m2[0] = m2[0] + b"!"
    assert _emu_ed_verify(sigs, m2, pks, z)[0] is False
    # s >= l is rejected up front with its index
    b = bytearray(sigs[3])
    b[63] |= 0xF0
    bad = list(sigs)
    bad[3] = bytes(b)
    assert _emu_ed_verify(bad, msgs, pks, z) == (False, 3)
    # ZIP-215 vectors (message "Zcash"): each alone, and all valid ones in one batch
    zs = g["zip215"]
    valid = [v for v in zs if v["valid_zip215"]][:20]
    invalid = [v for v in zs if not v["valid_zip215"]][:6]
    for v in valid[:8] + invalid:
        got = _emu_ed_verify([bytes.fromhex(v["sig_bytes"])], [b"Zcash"], [bytes.fromhex(v["vk_bytes"])], bytes(range(16)))
        assert got[0] == v["valid_zip215"], v
    allz = bytes((i * 5 + 3) & 255 for i in range(16 * len(valid)))
    assert _emu_ed_verify([bytes.fromhex(v["sig_bytes"]) for v in valid], [b"Zcash"] * len(valid),
                          [bytes.fromhex(v["vk_bytes"]) for v in valid], allz)[0] is True


def test_point_decoders_match_oracle():
    """codec.cuh (SEC1-33 secp256k1, Zcash-48 BLS12-381 G1) vs the oracle decode restatements on the reference's vectors
    plus flag / range edge cases."""
    import ctypes

    import numpy as np

    from conftest import load_golden

    lib = H.hostemu()

    def emu(curve, enc, words):
        out = np.zeros(words, np.uint32)
        st = lib.emu_decode(curve, enc, out.ctypes.data_as(ctypes.c_void_p))
        half = words // 2
        return st, int.from_bytes(out[:half].tobytes(), "little"), int.from_bytes(out[half:].tobytes(), "little")

    g = load_golden("bls12_381.json")["G1_Compressed"]
    cases = [bytes.fromhex(c) for c in g[:60]] + [bytes.fromhex(g[777])]
    p = R.BLS12_381_G1_CURVE["p"]
    cases += [bytes([0xC0] + [0] * 47), bytes([0xE0] + [0] * 47), bytes([0xC0] + [0] * 46 + [1]), bytes([0x40] + [0] * 47),
              bytes([0x80]) + bytes(47), (p | (1 << 383)).to_bytes(48, "big"), bytes([0x9F] + [0xFF] * 47),
              bytes([0x80]) + (5).to_bytes(47, "big"), bytes([0xA0]) + (5).to_bytes(47, "big")]
    for enc in cases:
        st, x, y = emu(4, enc, 24)
        try:
            ex, ey = R.bls12_381_g1_decode(enc)
            if not (enc[0] & 0x80):
                raise ValueError("uncompressed form not taken by this entry point")
            assert (st, x, y) == ((2 if (ex, ey) == (0, 0) else 1), ex, ey), enc.hex()
        except ValueError:
            assert st == 0, enc.hex()
    # G2, 96-byte compressed: reference vectors + flag / range / non-residue cases + c1 == 0 roots
    g2 = load_golden("bls12_381.json")["G2_Compressed"]

    def emu_g2(enc):
        out = np.zeros(48, np.uint32)
        st = lib.emu_decode(5, enc, out.ctypes.data_as(ctypes.c_void_p))
        w = [int.from_bytes(out[12 * k:12 * (k + 1)].tobytes(), "little") for k in range(4)]
        return st, (w[0], w[1]), (w[2], w[3])

    cases2 = [bytes.fromhex(c) for c in g2[:24]] + [bytes.fromhex(g2[200])]
    cases2 += [bytes([0xC0] + [0] * 95), bytes([0xE0] + [0] * 95), bytes([0xC0] + [0] * 94 + [1]), bytes([0x40] + [0] * 95),
               bytes([0x80]) + bytes(95), bytes([0x9F] + [0xFF] * 95),
               bytes([0x80]) + bytes(47) + p.to_bytes(48, "big"),   # c0 == p: out of range
               (p | (1 << 383)).to_bytes(48, "big") + bytes(48)]    # c1 == p
    for xv in range(1, 14):  # small x = (xv, 0) and (0, xv): squares and non-squares, both sort bits
        for enc_x in (bytes(48) + xv.to_bytes(48, "big"), xv.to_bytes(48, "big") + bytes(48)):
            for flag in (0x80, 0xA0):
                cases2.append(bytes([enc_x[0] | flag]) + enc_x[1:])
    n_ok = 0
    for enc in cases2:
        st, x, y = emu_g2(enc)
        try:
            ex, ey = R.bls12_381_g2_decode(enc)
            if not (enc[0] & 0x80):
                raise ValueError("uncompressed form not taken by this entry point")
            assert (st, x, y) == ((2 if (ex, ey) == ((0, 0), (0, 0)) else 1), ex, ey), enc.hex()
            n_ok += 1
        except ValueError:
            assert st == 0, enc.hex()
    assert n_ok > 40
    # fp2_sqrt directly, incl. the c1 == 0 branches the decoder rarely reaches (tower.ts:481-485)
    F2 = R.Field2(R.Field(p))
    rnd_ = __import__("random").Random(4)
    vals = [(4, 0), (5, 0), (p - 4, 0), (0, 9), (0, 0), (3, 7)] + [(rnd_.randrange(p), rnd_.randrange(p)) for _ in range(6)]
    for v in vals + [F2.sqr(v) for v in vals]:
        inp = np.frombuffer(v[0].to_bytes(48, "little") + v[1].to_bytes(48, "little"), dtype=np.uint32).copy()
        out = np.zeros(24, np.uint32)
        ok = lib.emu_fp2_sqrt(inp.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p))
        try:
            exp = F2.sqrt(v)
        except ValueError:
            exp = None
        assert bool(ok) == (exp is not None), v
        if ok:
            r = (int.from_bytes(out[:12].tobytes(), "little"), int.from_bytes(out[12:].tobytes(), "little"))
            assert r in (exp, F2.neg(exp)), v
    s = load_golden("secp256k1.json")["isPoint33"]
    sample = s[:80] + [c for c in s if not c[1]]
    pk = R.SECP256K1_CURVE["p"]
    sample += [["02" + pk.to_bytes(32, "big").hex(), False], ["05" + "11" * 32, False], ["02" + "00" * 32, None]]
    for enc_hex, exp in sample:
        enc = bytes.fromhex(enc_hex)
        st, x, y = emu(0, enc, 16)
        try:
            ex, ey = R.secp256k1_decode_sec1(enc)
            assert (st, x, y) == (1, ex, ey), enc_hex
            assert exp in (True, None)
        except ValueError:
            assert st == 0, enc_hex


@pytest.mark.parametrize("cid,name,lam,bits", [
    (0, "secp256k1", 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72, 129),
    (2, "bn254_G1", 0x30644E72E131A029048B6E193FD84104CC37A73FEC2BC5E9B8CA0B2D36636F23, 127),
])
def test_glv_lattice_split(cid, name, lam, bits):
    """glv_split_lattice: k = v1 + v2*lambda (mod n) with short halves; phi(P) = (beta*x, y) = lambda*P; for secp256k1
    the halves equal the reference's _splitEndoScalar (weierstrass.ts:121-148) via the oracle."""
    import ctypes
    import random as _r

    import numpy as np

    P = R.CURVES[name]
    n, p = P.Fn.ORDER, P.Fp.ORDER
    assert (lam * lam + lam + 1) % n == 0
    lg = P.BASE.multiplyUnsafe(lam).toAffine()
    g = P.BASE.toAffine()
    assert lg["y"] == g["y"] and (lg["x"] * pow(g["x"], -1, p)) % p in (
        0x7AE96A2B657C07106E64479EAC3434E99CF0497512F58995C1396C28719501EE,
        0x30644E72E131A0295E6DD9E7E0ACCCB0C28F069FBB966E3DE4BD44E5607CFD48)
    rnd = _r.Random(8)
    ks = [0, 1, 2, n - 1, n - 2, lam, lam + 1, lam - 1, n >> 1, (n >> 1) + 1] + [rnd.randrange(n) for _ in range(3000)]
    lib = H.hostemu()
    for k in ks:
        a = H.u32(k.to_bytes(32, "little"))
        out = np.zeros(12, np.uint32)
        lib.emu_glv_split_lattice(cid, a.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p))
        m1 = int.from_bytes(out[:5].tobytes(), "little")
        m2 = int.from_bytes(out[5:10].tobytes(), "little")
        v1 = -m1 if out[10] else m1
        v2 = -m2 if out[11] else m2
        assert (v1 + v2 * lam - k) % n == 0 and m1 >> bits == 0 and m2 >> bits == 0, hex(k)
        if name == "secp256k1":
            k1neg, k1, k2neg, k2 = R.split_endo_scalar(k, R.SECP256K1_ENDO["basises"], n)
            assert (m1, m2) == (k1, k2) and (not m1 or bool(out[10]) == k1neg) and (not m2 or bool(out[11]) == k2neg)


@pytest.mark.parametrize("name", ["secp256k1", "ed25519", "bn254_G2", "bls12_381_G1", "bls12_381_G1_any"])
def test_window_groups_hostemu(name):
    """Window-group pipelining (engine.cuh submit_msm) on the device bodies: per-window accumulate segments, per-group
    stitch / reduce, Horner steps across groups — every group count gives the oracle's pippenger, also for inputs
    whose buckets span many segments (small L) and for degenerate scalars."""
    cname = "bls12_381_G1" if name.endswith("_any") else name
    n = 160
    P, pts, scalars, _ = H.soak_inputs(cname, n, seed_offset=11)
    scalars[5] = P.Fn.ORDER - 1
    exp = H.expected_tuple(cname, R.pippenger(P, pts, scalars))
    pb, sb = H.pack_points(cname, pts), H.pack_scalars(scalars)
    for groups, c, L in ((2, 0, 0), (3, 5, 1), (8, 4, 2), (64, 3, 3)):
        got, err, plan = H.emu_msm(name, pb, sb, n, forced_c=c, forced_L=L, groups=groups)
        assert err == (0xFFFFFFFF, 0xFFFFFFFF)
        assert got == exp, (name, groups, c, L, plan)
    same = [(P.Fn.ORDER - 1) // 5] * n
    exp2 = H.expected_tuple(cname, R.pippenger(P, pts, same))
    got, _, _ = H.emu_msm(name, pb, H.pack_scalars(same), n, forced_c=6, forced_L=1, groups=4)
    assert got == exp2


def test_strict_ed25519_decode_and_on_curve_hostemu():
    """ed_decompress(zip215 = false) = the reference's fromBytes default (edwards.ts:405-436); point_on_curve =
    isValidXY (weierstrass.ts:617-624)."""
    import ctypes

    import numpy as np

    from conftest import load_golden

    lib = H.hostemu()
    g = load_golden("ed25519.json")
    p = R.ED25519_CURVE["p"]
    encs = [bytes.fromhex(v["pk"]) for v in g["vectors"][:8]] + [bytes.fromhex(v["vk_bytes"]) for v in g["zip215"][:60]]
    encs += [p.to_bytes(32, "little"), (p + 1).to_bytes(32, "little"), ((1 << 255) | 1).to_bytes(32, "little"),
             ((1 << 255) | (p - 1)).to_bytes(32, "little"), (1).to_bytes(32, "little")]
    rejected = 0
    for e in encs:
        out = np.zeros(16, np.uint32)
        ok = lib.emu_ed25519_decompress_strict(e, out.ctypes.data_as(ctypes.c_void_p))
        try:
            a = R.ed25519_point_from_bytes(e, False).toAffine()
            assert ok == 1, e.hex()
            assert int.from_bytes(out[:8].tobytes(), "little") == a["x"] and int.from_bytes(out[8:].tobytes(), "little") == a["y"]
        except ValueError:
            rejected += 1
            assert ok == 0, e.hex()
    assert rejected >= 4
    for name in ("secp256k1", "ed25519", "bn254_G1", "bn254_G2", "bls12_381_G1", "bls12_381_G2"):
        P, pts, _, _ = H.soak_inputs(name, 6)
        for i, q in enumerate(pts):
            b = bytearray(H.point_bytes(name, q))
            arr = np.frombuffer(bytes(b), dtype=np.uint32).copy()
            assert lib.emu_on_curve(H.CURVE_IDS[name], arr.ctypes.data_as(ctypes.c_void_p)) == 1, name
            b[len(b) // 2] ^= 2
            arr = np.frombuffer(bytes(b), dtype=np.uint32).copy()
            assert lib.emu_on_curve(H.CURVE_IDS[name], arr.ctypes.data_as(ctypes.c_void_p)) == 0, name


@pytest.mark.parametrize("name", ["secp256k1", "bn254_G2", "bls12_381_G1", "bls12_381_G1_any"])
def test_paired_accumulation_hostemu(name):
    """The NMSM_PAIRED=1 build option of k_accumulate (same-bucket neighbours added in affine first, one shared inversion:
    msm_body.cuh accumulate_pairs_pass1/2) against the oracle, incl. the inputs where a pair is P + P or P + (-P) and must
    fall back to the complete mixed addition."""
    cname = "bls12_381_G1" if name.endswith("_any") else name
    lib = H.hostemu()
    prev = lib.emu_set_paired(1)
    try:
        n = 200
        P, pts, scalars, _ = H.soak_inputs(cname, n, seed_offset=21)
        exp = H.expected_tuple(cname, R.pippenger(P, pts, scalars))
        pb, sb = H.pack_points(cname, pts), H.pack_scalars(scalars)
        for c, L in ((0, 0), (4, 7), (3, 64), (6, 2)):
            got, err, plan = H.emu_msm(name, pb, sb, n, forced_c=c, forced_L=L)
            assert got == exp, (name, c, L, plan)
        # degenerate: the same point many times with equal scalars (every pair is P + P), P and -P next to each other,
        # ZERO points inside pairs
        G = pts[3]
        deg = [G] * 40 + [pts[5], pts[5].negate()] * 6 + [P.ZERO, pts[7], P.ZERO, P.ZERO]
        dsc = [9] * 40 + [5] * 12 + [3, 4, 5, 6]
        exp2 = H.expected_tuple(cname, R.pippenger(P, deg, dsc))
        for c, L in ((4, 8), (2, 64), (5, 3)):
            got, _, _ = H.emu_msm(name, H.pack_points(cname, deg), H.pack_scalars(dsc), len(deg), forced_c=c, forced_L=L)
            assert got == exp2, (name, c, L)
    finally:
        lib.emu_set_paired(prev)
