"""The EIP-4844 prover on the GPU (nmsm.KzgSetup over nmsm_bls12_381_kzg_setup_create and the three batch calls):
commitments and proofs are byte-equal to the oracle's scalar prover under the seeded tau (at several sizes, across the
1024-blob chunk, z on and off the domain), every case where the spec raises is None without touching its neighbours,
the results pass the existing verifiers, and bad setup points are reported with their index."""
import random

import pytest

import kzg_cases as C
import kzg_prove_cases as P
from oracle import kzg_ref as K
import kzg_prove_ref as KP

pytestmark = pytest.mark.gpu
R = C.R


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


@pytest.fixture(scope="module")
def lagrange():
    return KP.setup_g1_lagrange(C.TAU)  # ~17 s in the oracle


@pytest.fixture(scope="module")
def setup(nmsm, lagrange):
    s = nmsm.KzgSetup(lagrange)
    yield s
    s.close()


def _tiled(count, distinct=3):
    base = [C.blob_item(s) for s in range(1, 1 + min(count, distinct))]
    return [base[k % len(base)] for k in range(count)]


@pytest.mark.parametrize("n", [1, 3, 1025])
def test_commitments_match_oracle(setup, n):
    items = _tiled(n)
    assert setup.blob_to_kzg_commitment_batch([i[0] for i in items]) == [i[1] for i in items]


def test_unit_blobs_pick_the_bit_reversed_setup_point(setup, lagrange):
    """f_p = 1 and every other element 0 commits to KZG_SETUP_G1_LAGRANGE[brp(p)]: every lane position of the comb"""
    ps = (0, 1, 3, 31, 32, 1000, 4095)
    blobs = [C.blob_with(C.ZERO_BLOB, p, 1) for p in ps]
    assert setup.blob_to_kzg_commitment_batch(blobs) == [KP.bit_reversal_permutation(lagrange)[p] for p in ps]


def test_zero_blob_gives_identities(setup):
    blob = C.random_blob(30)
    assert setup.blob_to_kzg_commitment_batch([C.ZERO_BLOB, blob, C.ZERO_BLOB])[::2] == [C.IDENTITY] * 2
    got = setup.compute_kzg_proof_batch([C.ZERO_BLOB] * 3, [5, 0, P.BRP[1]])
    assert got == [(C.IDENTITY, bytes(32))] * 3
    assert setup.compute_blob_kzg_proof_batch([C.ZERO_BLOB], [C.IDENTITY]) == [C.IDENTITY]


@pytest.mark.parametrize("index", [0, 1, 4095])
def test_element_out_of_range_is_none_for_that_blob_only(setup, index):
    (b1, c1, p1, _, _), (b2, c2, p2, _, _) = C.blob_item(1), C.blob_item(2)
    bad = C.blob_with(b1, index, R)
    blobs = [b1, bad, b2]
    out, ok = setup.blob_to_kzg_commitment_batch_packed(b"".join(blobs), 3)
    assert ok == b"\1\0\1" and out == c1 + bytes(48) + c2
    proofs, ys, ok = setup.compute_kzg_proof_batch_packed(b"".join(blobs), C.be(7) * 3, 3)
    assert ok == b"\1\0\1" and proofs[48:96] == bytes(48) and ys[32:64] == bytes(32)
    assert setup.compute_blob_kzg_proof_batch(blobs, [c1, c1, c2]) == [p1, None, p2]


def test_compute_kzg_proof_matches_oracle(setup):
    blob = C.random_blob(31)
    cases = P.z_cases(seed=2)
    zs = [z for _, z in cases] + [R, (1 << 256) - 1]
    got = setup.compute_kzg_proof_batch([blob] * len(zs), zs)
    for (name, z), g in zip(cases, got):
        proof, y = P.expected_proof(blob, z)
        assert g == (proof, C.be(y)), name
    assert got[-2:] == [None, None]


def test_compute_kzg_proof_on_the_domain_across_blobs(setup):
    blobs = [C.random_blob(s) for s in (32, 33, 34, 35)]
    zs = [P.BRP[k] for k in P.DOMAIN_INDICES]
    got = setup.compute_kzg_proof_batch(blobs, zs)
    for blob, z, g in zip(blobs, zs, got):
        proof, y = P.expected_proof(blob, z)
        assert g == (proof, C.be(y))
        assert y == K.blob_to_polynomial(blob)[P.BRP.index(z)]


def test_compute_blob_kzg_proof_matches_oracle_and_verifies(nmsm, setup):
    items = _tiled(5)
    blobs, cs = [i[0] for i in items], [i[1] for i in items]
    proofs = setup.compute_blob_kzg_proof_batch(blobs, cs)
    assert proofs == [i[2] for i in items]
    assert nmsm.kzg_verify_blob_proof_batch(blobs, cs, proofs, C.SETUP) == [True] * 5


def test_invalid_commitments_are_none(setup):
    (b1, c1, p1, _, _), (b2, c2, p2, _, _) = C.blob_item(1), C.blob_item(2)
    bad = [C.off_curve_g1(), C.small_order_g1(), C.NON_CANONICAL_IDENTITY, C.uncompressed_flag(c1)]
    blobs = [b1] + [b1] * len(bad) + [b2]
    got = setup.compute_blob_kzg_proof_batch(blobs, [c1] + bad + [c2])
    assert got == [p1] + [None] * len(bad) + [p2]


def test_round_trip_through_the_verifiers(nmsm, setup):
    blobs = [C.random_blob(s) for s in (41, 42, 43, 44)]
    cs = setup.blob_to_kzg_commitment_batch(blobs)
    proofs = setup.compute_blob_kzg_proof_batch(blobs, cs)
    assert nmsm.kzg_verify_blob_proof_batch(blobs, cs, proofs, C.SETUP) == [True] * 4
    assert nmsm.kzg_verify_blob_proof_batch(blobs, cs, proofs, C.OTHER_SETUP) == [False] * 4
    rnd = random.Random(45)
    zs = [rnd.randrange(R) for _ in blobs[:2]] + [P.BRP[3], 0]
    opened = setup.compute_kzg_proof_batch(blobs, zs)
    pis, ys = [o[0] for o in opened], [o[1] for o in opened]
    assert nmsm.kzg_verify_proof_batch(cs, zs, ys, pis, C.SETUP) == [True] * 4
    assert nmsm.kzg_verify_proof_batch(cs, zs, ys, pis, C.OTHER_SETUP) == [False] * 4


@pytest.mark.parametrize("index,enc", [(7, "off_curve"), (4095, "small_order"), (0, "identity"), (100, "two")])
def test_setup_point_errors(nmsm, lagrange, index, enc):
    from nmsm import _lib

    bad = {"off_curve": C.off_curve_g1(), "small_order": C.small_order_g1(), "identity": C.IDENTITY}
    pts = list(lagrange)
    if enc == "two":  # the smallest bad index is reported
        pts[3000], pts[index] = C.off_curve_g1(), C.small_order_g1()
    else:
        pts[index] = bad[enc]
    with pytest.raises(ValueError) as e:
        nmsm.KzgSetup(pts)
    assert e.value.__cause__.code == _lib.ERR_POINT and e.value.__cause__.index == index


def test_two_setups_are_independent(nmsm, setup):
    tau2 = C.TAU + 1
    other = nmsm.KzgSetup(KP.setup_g1_lagrange(tau2))
    try:
        blob = C.random_blob(50)
        z = 12345
        want1, want2 = K.commit_value(P.f_tau(blob)), K.commit_value(P.f_tau(blob, tau2))
        assert other.blob_to_kzg_commitment_batch([blob]) == [want2]
        assert setup.blob_to_kzg_commitment_batch([blob]) == [want1]
        proof2, y = P.expected_proof(blob, z, tau2)
        assert other.compute_kzg_proof_batch([blob], [z]) == [(proof2, C.be(y))]
        assert setup.compute_kzg_proof_batch([blob], [z]) == [(P.expected_proof(blob, z)[0], C.be(y))]
    finally:
        other.close()


def test_closed_setup_is_an_argument_error(nmsm, lagrange):
    from nmsm import _lib

    s = nmsm.KzgSetup(lagrange)
    s.close()
    with pytest.raises(_lib.NmsmError) as e:
        s.blob_to_kzg_commitment_batch([C.ZERO_BLOB])
    assert e.value.code == _lib.ERR_ARG
    assert s.blob_to_kzg_commitment_batch([]) == []
