"""Subgroup checks and the point kernels on points of small and mixed order, through tests/hostemu (the device bodies
compiled for the CPU), against mul_any (torsion_cases.py).  The GPU counterparts are in test_gpu_torsion.py."""
import random

import pytest

import helpers as H
import torsion_cases as TC
from oracle import noble_ref as R

ALL_IDS = list(range(8))
MUL_IDS = [1, 3, 4, 5, 6, 7]
MSM_IDS = [1, 3, 6, 7]


def _pack(name, pts):
    return H.pack_points(name, pts)


@pytest.mark.parametrize("cid", ALL_IDS)
def test_torsion_free_every_order(cid):
    """nmsm_points_torsion_free's body on subgroup, small-order, mixed and random points and the identity: the flag is
    r P == O by mul_any.  On BLS12-381 G1 (r - 1) T = O for every small-order T, so the final addition starts from the
    identity; secp256k1 and bn254 G1 have cofactor 1 and every on-curve point passes."""
    name = TC.NAME_OF_ID[cid]
    r = TC.r_of(name)
    pl = TC.points(name)
    want = [1 if TC.mul_any(p, r).is0() else 0 for _, p, _ in pl]
    assert want == [1 if kind in ("subgroup", "identity") else 0 for kind, _, _ in pl]
    got, err = H.emu_torsion(TC.ID_NAME[cid], _pack(name, [p for _, p, _ in pl]), len(pl))
    assert err[0] == 0xFFFFFFFF
    assert got == want, [(kind, q) for (kind, _, q), g, w in zip(pl, got, want) if g != w]


@pytest.mark.parametrize("cid", MUL_IDS)
def test_mul_batch_small_and_mixed_order(cid):
    """nmsm_mul_batch's body (Point.multiply, independent of the subgroup for every id) on every point of the lists
    with 1, 2, q - 1, q, q + 1, 2q, m q, r - 1, r - 2, (r - 1) / 2, h and random scalars."""
    name = TC.NAME_OF_ID[cid]
    cases = TC.mul_cases(name)
    pts = [p for p, _ in cases]
    ks = [k for _, k in cases]
    got, err = H.emu_mul_batch(TC.ID_NAME[cid], _pack(name, pts), H.pack_scalars(ks), len(ks), False)
    assert err == (0xFFFFFFFF, 0xFFFFFFFF)
    bad = [(i, hex(k)) for i, (p, k) in enumerate(cases) if got[i] != TC.expected(name, p, k)]
    assert not bad, bad[:8]


@pytest.mark.parametrize("cid", MUL_IDS)
@pytest.mark.parametrize("bits", [5, 8])
def test_point_table_small_order_base(cid, bits):
    """nmsm_point_table_* bodies with a small table whose base is a small-order point (identity entries at digits
    d = 0 mod q, and for ed25519 at every level j >= 1 once 2^bits T = O), a mixed point and a random point outside the
    subgroup.  The table bodies never use an endomorphism, so ids 4 and 5 are held to the same results."""
    name = TC.NAME_OF_ID[cid]
    rnd = random.Random("table-%d-%d" % (cid, bits))
    pl = TC.points(name)
    small = [(p, q) for p, q in TC.small_points(name) if q <= 1 << (bits - 1)] or TC.small_points(name)[:1]
    bases = small[:2] + [(p, q) for kind, p, q in pl if kind == "mixed"][:1] + [(p, 0) for kind, p, _ in pl
                                                                              if kind == "random"][:1]
    for base, q in bases:
        ks = TC.table_scalars(name, q if q > 1 else 3, bits, rnd)
        got, err = H.emu_point_table(TC.ID_NAME[cid], H.point_bytes(name, base), H.pack_scalars(ks), len(ks), False,
                                     table_bits=bits)
        assert err == (0xFFFFFFFF, 0xFFFFFFFF)
        for k, g in zip(ks, got):
            assert g == TC.expected(name, base, k), (q, hex(k))
        got, err = H.emu_point_table(TC.ID_NAME[cid], H.point_bytes(name, base), H.pack_scalars([0, q or 1]), 2, True,
                                     table_bits=bits)
        assert got == [TC.expected(name, base, 0), TC.expected(name, base, q or 1)]


@pytest.mark.parametrize("cid", MSM_IDS)
def test_msm_small_and_mixed_order(cid):
    """MSM bodies (plain windows: ids 1, 3, 6, 7) on sets of mixed, random and small-order points, on sets whose torsion
    parts cancel and on all-small-order sets whose sum is O, for forced window sizes and segment lengths and through
    the fixed-base table route.  Ids 4 and 5 are left out: their contract excludes points outside the subgroup."""
    name = TC.NAME_OF_ID[cid]
    for label, pts, sc in TC.msm_sets(name):
        want = TC.expected_sum(name, pts, sc)
        pb, sb = _pack(name, pts), H.pack_scalars(sc)
        for c, L in ((0, 0), (2, 1), (3, 2), (5, 3), (13, 32)):
            got, err, _ = H.emu_msm(TC.ID_NAME[cid], pb, sb, len(pts), c, L)
            assert err == (0xFFFFFFFF, 0xFFFFFFFF)
            assert got == want, (label, c, L)
        for tc in (4, 9):
            assert H.emu_msm(TC.ID_NAME[cid], pb, sb, len(pts), table_c=tc)[0] == want, (label, tc)


def test_case_lists_are_what_they_claim():
    """The generators themselves: every small-order point has the order it is listed with, mixed points are outside
    the subgroup, and the group orders kill random points."""
    for name in TC.WITH_COFACTOR:
        for kind, p, q in TC.points(name):
            if kind == "small":
                assert TC.mul_any(p, q).is0() and not p.is0()
                assert all(not TC.mul_any(p, q // f).is0() for f in (2, 3, 5, 7) if q % f == 0)
            if kind in ("mixed", "random"):
                assert not TC.mul_any(p, TC.r_of(name)).is0()
        rq = TC.random_point(name, random.Random(1))
        assert TC.mul_any(rq, TC.GROUP_ORDER[name]).is0()
    P = R.CURVES["bls12_381_G1"]
    assert R.affine_tuple(P, TC.mul_any(P.BASE, 12345)) == R.affine_tuple(P, P.BASE.multiply(12345))
