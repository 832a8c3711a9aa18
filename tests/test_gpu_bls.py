"""BLS12-381 pairing checks and BLS signature verification on the GPU (nmsm_bls12_381_pairing_check_batch,
nmsm_bls12_381_verify_batch): every verdict is compared with the oracle (oracle.bls_pairing_ref) or with the verdict
known from how the input was constructed (bilinearity, swapped signatures)."""
import random

import pytest

import bls_cases as C
from oracle import bls_pairing_ref as B

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _check(nmsm, checks):
    g1, g2, off = C.pack_checks(checks)
    return [b == 1 for b in nmsm.pairing_check_batch_packed(g1, g2, off, len(checks))]


@pytest.fixture(scope="module")
def pool():
    """true and false checks of 1, 2, 3, 4 and 8 pairs"""
    rnd = random.Random(5)
    out = {}
    for k in (2, 3, 4, 8):
        out[k] = (C.true_check(rnd, k), C.false_check(rnd, k))
    g = (C.g1_mul(3), C.g2_mul(5))
    out[1] = ([(g[0], C.ID2)], [g])  # one pair: only an identity pair gives 1
    return out


def test_checks_of_1_2_3_4_8_pairs(nmsm, pool):
    checks, want = [], []
    for k, (t, f) in sorted(pool.items()):
        checks += [t, f]
        want += [True, False]
    assert _check(nmsm, checks) == want


def test_identity_pairs_and_empty_checks(nmsm, pool):
    t, f = pool[3]
    checks = [[], t + [(C.ID1, C.g2_mul(7))], f + [(C.g1_mul(9), C.ID2)], [(C.ID1, C.ID2)], [], t]
    assert _check(nmsm, checks) == [True, True, False, True, True, True]


def test_generators_and_off_subgroup_points_match_oracle(nmsm):
    rnd = random.Random(8)
    g1, g2 = C.g1_mul(1), C.g2_mul(1)
    p1, q1 = C.g1_off_subgroup(rnd), C.g2_off_subgroup(rnd)
    checks = [[(g1, g2)], [(p1, g2)], [(g1, q1)], [(p1, q1), (p1, q1)], [(p1, q1), (B.affine(B.G1.fromAffine(
        {"x": p1[0], "y": p1[1]}).negate()), q1)]]
    want = [B.pairing_check(c) for c in checks]
    assert _check(nmsm, checks) == want
    assert want[0] is False


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 127, 4097])
def test_batches_with_scattered_false_checks(nmsm, pool, n):
    rnd = random.Random(n)
    checks, want = [], []
    for _ in range(n):
        k = rnd.choice([1, 2, 3, 4, 8])
        ok = rnd.random() < 0.8
        checks.append(pool[k][0 if ok else 1])
        want.append(ok)
    assert _check(nmsm, checks) == want


def test_check_spanning_miller_chunks(nmsm):
    """one check of 2^16 + 6 pairs (the Miller workspace holds 2^16) between two small ones: the partial product is
    carried across the chunk boundary"""
    g1, g2 = C.g1_mul(11), C.g2_mul(13)
    ng1 = B.affine(B.G1.fromAffine({"x": g1[0], "y": g1[1]}).negate())
    big = [(g1, g2), (ng1, g2)] * ((1 << 15) + 3)
    t = C.true_check(random.Random(3), 2)
    f = C.false_check(random.Random(4), 2)
    assert _check(nmsm, [f, big, t, f]) == [False, True, True, False]
    assert _check(nmsm, [big[:-1]]) == [False]


def test_off_curve_points_are_point_errors_with_their_index(nmsm, pool):
    from nmsm import NmsmError

    t = pool[4][0]
    bad1 = (t[0][0][0], (t[0][0][1] + 1) % B.P)
    bad2 = (t[0][1][0], (t[0][1][1][0], (t[0][1][1][1] + 1) % B.P))
    checks = [t, t[:2] + [(bad1, t[2][1])] + t[3:], [(t[0][0], bad2)]]
    with pytest.raises(NmsmError) as e:
        _check(nmsm, checks)
    assert e.value.code == -3 and e.value.index == 6
    checks = [t, [(t[0][0], bad2)], t[:1] + [(bad1, t[1][1])]]
    with pytest.raises(NmsmError) as e:  # G1 is reported before G2
        _check(nmsm, checks)
    assert e.value.code == -3 and e.value.index == 6
    with pytest.raises(NmsmError) as e:  # x >= p
        _check(nmsm, [[((B.P, 0), t[0][1])]])
    assert e.value.code == -3 and e.value.index == 0
    with pytest.raises(ValueError):
        nmsm.pairing_check_batch([[(nmsm.bls12_381.G1.Point(bad1[0], bad1[1]), nmsm.bls12_381.G2.Point.BASE)]])


def test_bad_offsets_are_argument_errors(nmsm, pool):
    import ctypes
    import struct

    from nmsm import NmsmError

    t = pool[2][0]
    g1, g2, _ = C.pack_checks([t, t])
    lib = nmsm._lib.load()
    out = ctypes.create_string_buffer(2)
    for offs in ([1, 2, 4], [0, 3, 2], [0, 4, 2], [0, 2, 1 << 31]):
        rc = lib.nmsm_bls12_381_pairing_check_batch(g1, g2, struct.pack("<3Q", *offs), 2, out)
        assert rc == -1, offs
    assert lib.nmsm_bls12_381_pairing_check_batch(None, g2, struct.pack("<3Q", 0, 2, 4), 2, out) == -1
    with pytest.raises(NmsmError) as e:
        nmsm.pairing_check_batch_packed(g1, g2, struct.pack("<3Q", 1, 2, 4), 2)
    assert e.value.code == -1
    assert nmsm.pairing_check_batch_packed(b"", b"", struct.pack("<Q", 0), 0) == b""


def test_mirror_pairing_check_batch_on_points(nmsm, pool):
    G1, G2 = nmsm.bls12_381.G1.Point, nmsm.bls12_381.G2.Point
    conv = lambda p, c: c.ZERO if p in (C.ID1, C.ID2) else c(p[0], p[1])  # noqa: E731
    checks = [[(conv(p, G1), conv(q, G2)) for p, q in pool[4][k]] for k in (0, 1)]
    assert nmsm.pairing_check_batch(checks + [[]]) == [True, False, True]


# ---- verification ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def edge():
    cases = C.edge_cases()
    return cases, [B.bls_verify(c[1], c[2], c[3]) for c in cases]


def _verify(nmsm, items):
    G2 = nmsm.bls12_381.G2.Point
    hs = [G2.ZERO if i[1] == C.ID2 else G2(i[1][0], i[1][1]) for i in items]
    return nmsm.bls_verify_batch([i[0] for i in items], hs, [i[2] for i in items])


def test_verify_edge_set_matches_oracle(nmsm, edge):
    cases, want = edge
    got = _verify(nmsm, [c[1:] for c in cases])
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    names = dict(zip((c[0] for c in cases), got))
    assert names["valid"] and names["valid-2"] and sum(got) == 2


@pytest.fixture(scope="module")
def signed():
    rnd = random.Random(21)
    return [C.keypair_item(rnd) for _ in range(6)]


@pytest.mark.parametrize("n", [1, 2, 33, 4097])
def test_verify_batches_with_scattered_invalid_items(nmsm, signed, n):
    rnd = random.Random(100 + n)
    items, want = [], []
    for _ in range(n):
        a = rnd.randrange(len(signed))
        if rnd.random() < 0.85:
            items.append(signed[a])
            want.append(True)
        else:
            b = (a + 1 + rnd.randrange(len(signed) - 1)) % len(signed)
            items.append((signed[b][0], signed[a][1], signed[a][2]))  # another key's signature
            want.append(False)
    assert _verify(nmsm, items) == want


def test_verify_single_form_points_and_errors(nmsm, signed):
    sig, H, pk = signed[0]
    G1, G2 = nmsm.bls12_381.G1.Point, nmsm.bls12_381.G2.Point
    Hp = G2(H[0], H[1])
    assert nmsm.bls12_381.verify(sig, Hp, pk) is True
    x, y = B.R.bls12_381_g1_decode(pk)
    assert nmsm.bls12_381.verify(sig, Hp, G1(x, y)) is True
    sx, sy = B.R.bls12_381_g2_decode(sig)
    assert nmsm.bls12_381.verify(G2(sx, sy), Hp, pk) is True
    with pytest.raises(NotImplementedError, match="hash-to-curve"):
        nmsm.bls12_381.verify(sig, b"message", pk)
    assert nmsm.bls_verify_batch([], [], []) == []
    from nmsm import NmsmError

    bad = G2(H[0], (H[1][0], (H[1][1] + 1) % B.P))
    with pytest.raises(ValueError):
        nmsm.bls_verify_batch([sig, sig], [Hp, bad], [pk, pk])
    with pytest.raises(NmsmError) as e:
        nmsm.bls_verify_batch_packed(sig * 2, pk * 2, C.g2_bytes(H) + bad.to_packed(), 2)
    assert e.value.code == -3 and e.value.index == 1


def test_interleaved_with_ecdsa_msm_and_reinit(nmsm, signed, pool):
    import ecdsa_cases as E
    from oracle import ecdsa_ref as ER

    cases = E.edge_cases()
    items = [c[1:] for c in cases]
    want_e = [ER.secp256k1_ecdsa_verify(*i) for i in items]
    sig, H, pk = signed[1]
    G2 = nmsm.bls12_381.G2.Point
    Hp = G2(H[0], H[1])
    G1p = nmsm.bls12_381.G1.Point
    for _ in range(2):
        assert nmsm.bls12_381.verify(sig, Hp, pk) is True
        assert nmsm.ecdsa_verify_batch([i[0] for i in items], [i[1] for i in items], [i[2] for i in items]) == want_e
        assert _check(nmsm, [pool[2][0], pool[2][1]]) == [True, False]
        r = nmsm.pippenger(G1p, [G1p.BASE, G1p.BASE.multiply(7)], [2, 3])
        assert r.equals(G1p.BASE.multiply(23))
    lib = nmsm._lib.load()
    lib.nmsm_shutdown()
    nmsm._lib.check(lib.nmsm_init(0))
    assert _check(nmsm, [pool[3][0], pool[3][1]]) == [True, False]
    assert nmsm.bls12_381.verify(sig, Hp, pk) is True


def test_profiling_slots(nmsm, signed, pool):
    nmsm.set_profiling(True)
    try:
        _check(nmsm, [pool[4][0]] * 64)
        ms = list(nmsm.last_timing()[0].values())
        assert ms[0] > 0 and ms[1] > 0 and abs(ms[-1] - (ms[0] + ms[1])) < 1e-3 * max(1.0, ms[-1])
        _verify(nmsm, signed * 8)
        ms = list(nmsm.last_timing()[0].values())
        assert ms[0] > 0 and ms[1] > 0 and ms[2] > 0 and abs(ms[-1] - (ms[0] + ms[1] + ms[2])) < 1e-3 * max(1.0, ms[-1])
    finally:
        nmsm.set_profiling(False)
