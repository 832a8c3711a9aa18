"""bn254 pairing checks on the GPU (nmsm_bn254_pairing_check_batch) and the EIP-197 helper: every verdict is compared
with the oracle (oracle.bn254_pairing_ref) or with the verdict known from how the input was constructed
(bilinearity)."""
import ctypes
import random
import struct

import pytest

import bn254_pairing_cases as C
from oracle import bn254_pairing_ref as B

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _check(nmsm, checks):
    g1, g2, off = C.pack_checks(checks)
    return [b == 1 for b in nmsm.bn254_pairing_check_batch_packed(g1, g2, off, len(checks))]


@pytest.fixture(scope="module")
def pool():
    return C.random_pool()


def test_checks_of_1_2_3_4_8_pairs(nmsm, pool):
    checks, want = [], []
    for k, (t, f) in sorted(pool.items()):
        checks += [t, f]
        want += [True, False]
    assert _check(nmsm, checks) == want


def test_groth16_shaped_checks(nmsm):
    rnd = random.Random(12)
    checks = [C.groth16_check(rnd), C.groth16_check(rnd, perturb=True), C.groth16_check(rnd)]
    assert _check(nmsm, checks) == [True, False, True]


def test_identity_pairs_and_empty_checks(nmsm, pool):
    t, f = pool[3]
    checks = [[], t + [(C.ID1, C.g2_mul(7))], f + [(C.g1_mul(9), C.ID2)], [(C.ID1, C.ID2)], [], t]
    assert _check(nmsm, checks) == [True, True, False, True, True, True]


def test_generators_and_off_subgroup_points_match_oracle(nmsm):
    rnd = random.Random(8)
    g1, g2 = C.g1_mul(1), C.g2_mul(1)
    q1 = C.g2_off_subgroup(rnd)
    checks = [[(g1, g2)], [(g1, q1)], [(g1, q1), (C.g1_neg(g1), q1)], [(g1, q1), (g1, q1)]]
    want = [B.pairing_check(c) for c in checks]
    assert _check(nmsm, checks) == want
    assert want[0] is False and want[2] is True


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
    big = [(g1, g2), (C.g1_neg(g1), g2)] * ((1 << 15) + 3)
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
    assert e.value.code == -3 and e.value.index == 6 and "G1 point of pair 6" in str(e.value)
    checks = [t, [(t[0][0], bad2)], t[:1] + [(bad1, t[1][1])]]
    with pytest.raises(NmsmError) as e:  # G1 is reported before G2
        _check(nmsm, checks)
    assert e.value.code == -3 and e.value.index == 6
    with pytest.raises(NmsmError) as e:
        _check(nmsm, [t, [(t[0][0], bad2)]])
    assert e.value.code == -3 and e.value.index == 4 and "G2 point of pair 4" in str(e.value)
    with pytest.raises(NmsmError) as e:  # x >= p
        _check(nmsm, [[((B.P, 0), t[0][1])]])
    assert e.value.code == -3 and e.value.index == 0
    with pytest.raises(ValueError):
        nmsm.bn254_pairing_check_batch([[(nmsm.bn254.G1.Point(bad1[0], bad1[1]), nmsm.bn254.G2.Point.BASE)]])


def test_bad_offsets_are_argument_errors(nmsm, pool):
    from nmsm import NmsmError

    t = pool[2][0]
    g1, g2, _ = C.pack_checks([t, t])
    lib = nmsm._lib.load()
    out = ctypes.create_string_buffer(2)
    for offs in ([1, 2, 4], [0, 3, 2], [0, 4, 2], [0, 2, 1 << 31]):
        rc = lib.nmsm_bn254_pairing_check_batch(g1, g2, struct.pack("<3Q", *offs), 2, out)
        assert rc == -1, offs
    assert lib.nmsm_bn254_pairing_check_batch(None, g2, struct.pack("<3Q", 0, 2, 4), 2, out) == -1
    assert lib.nmsm_bn254_pairing_check_batch(g1, g2, None, 2, out) == -1
    with pytest.raises(NmsmError) as e:
        nmsm.bn254_pairing_check_batch_packed(g1, g2, struct.pack("<3Q", 1, 2, 4), 2)
    assert e.value.code == -1
    assert nmsm.bn254_pairing_check_batch_packed(b"", b"", struct.pack("<Q", 0), 0) == b""


def test_mirror_pairing_check_batch_on_points(nmsm, pool):
    G1, G2 = nmsm.bn254.G1.Point, nmsm.bn254.G2.Point
    conv = lambda p, c: c.ZERO if p in (C.ID1, C.ID2) else c(p[0], p[1])  # noqa: E731
    checks = [[(conv(p, G1), conv(q, G2)) for p, q in pool[4][k]] for k in (0, 1)]
    assert nmsm.bn254_pairing_check_batch(checks + [[]]) == [True, False, True]


def test_eip197_helper(nmsm, pool):
    rnd = random.Random(40)
    t, f = pool[2]
    g16 = C.groth16_check(rnd)
    inputs = [C.eip197_bytes(t), C.eip197_bytes(f), b"", C.eip197_bytes(g16), C.eip197_bytes([(C.ID1, C.ID2)]),
              C.eip197_bytes(t + [(C.ID1, C.g2_mul(3)), (C.g1_mul(3), C.ID2)]), C.eip197_bytes([(C.g1_mul(1), C.g2_mul(1))])]
    assert nmsm.bn254_eip197_pairing_batch(inputs) == [True, False, True, True, True, True, False]
    q_off = C.g2_off_subgroup(rnd)
    with pytest.raises(ValueError, match="input 1: G2 point of pair 1 is not in the subgroup"):
        nmsm.bn254_eip197_pairing_batch([inputs[0], C.eip197_bytes([(C.ID1, C.ID2), (C.g1_mul(1), q_off)])])
    bad = bytearray(inputs[0])
    bad[32 + 31] ^= 1  # G1 y of pair 0
    with pytest.raises(ValueError, match="input 0: G1 point of pair 0 is not on the curve"):
        nmsm.bn254_eip197_pairing_batch([bytes(bad)])
    bad = bytearray(inputs[0])
    bad[192 + 160 + 31] ^= 1  # G2 y_real of pair 1
    with pytest.raises(ValueError, match="input 1: G2 point of pair 1 is not on the curve"):
        nmsm.bn254_eip197_pairing_batch([inputs[2], bytes(bad)])


def test_interleaved_with_bls_checks_msm_and_reinit(nmsm, pool):
    import bls_cases as BC

    rnd = random.Random(9)
    bls_t, bls_f = BC.true_check(rnd, 2), BC.false_check(rnd, 2)
    bls_args = BC.pack_checks([bls_t, bls_f])
    G1p = nmsm.bn254.G1.Point
    for _ in range(2):
        assert _check(nmsm, [pool[2][0], pool[2][1]]) == [True, False]
        assert nmsm.pairing_check_batch_packed(*bls_args, 2) == b"\x01\x00"
        r = nmsm.pippenger(G1p, [G1p.BASE, G1p.BASE.multiply(7)], [2, 3])
        assert r.equals(G1p.BASE.multiply(23))
        assert _check(nmsm, [pool[3][1], pool[3][0]]) == [False, True]
    lib = nmsm._lib.load()
    lib.nmsm_shutdown()
    nmsm._lib.check(lib.nmsm_init(0))
    assert _check(nmsm, [pool[4][0], pool[4][1]]) == [True, False]
    assert nmsm.pairing_check_batch_packed(*bls_args, 2) == b"\x01\x00"


def test_profiling_slots(nmsm, pool):
    nmsm.set_profiling(True)
    try:
        _check(nmsm, [pool[4][0]] * 64)
        ms = list(nmsm.last_timing()[0].values())
        assert ms[0] > 0 and ms[1] > 0 and abs(ms[-1] - (ms[0] + ms[1])) < 1e-3 * max(1.0, ms[-1])
        assert all(m == 0 for m in ms[2:-1])
    finally:
        nmsm.set_profiling(False)
