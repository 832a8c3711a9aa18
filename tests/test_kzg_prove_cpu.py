"""The EIP-4844 prover without a GPU: the oracle's Lagrange setup and quotient against the scalar identities that pin
the order conventions (a natural-order setup under the spec's bit reversal commits to f(tau), and the quotient opens
f at z), and the prover bodies of kzg.cuh run on the host through tests/hostemu against the oracle: the quotient, the
G1 compression and the comb lincomb over a small table."""
import random

import pytest

import kzg_cases as C
import kzg_prove_cases as P
from oracle import hash_to_g1_ref as H
from oracle import kzg_ref as K
import kzg_prove_ref as KP

R = K.BLS_MODULUS
Z_CASES = P.z_cases()


@pytest.fixture(scope="module")
def setup_scalars():
    return KP.setup_g1_lagrange_scalars(C.TAU)


@pytest.fixture(scope="module")
def poly():
    return K.blob_to_polynomial(C.random_blob(21))


# ---- the oracle ----------------------------------------------------------------------------------------------------
def test_lagrange_setup_commits_to_f_tau(setup_scalars, poly):
    assert P.lincomb_scalar(poly, setup_scalars) == K.evaluate_polynomial_in_evaluation_form(poly, C.TAU)


def test_lagrange_setup_is_the_natural_order_basis(setup_scalars):
    assert sum(setup_scalars) % R == 1  # sum_i L_i = 1
    # the basis polynomial of omega^1, evaluated at tau through the barycentric formula of the bit-reversed domain
    e1 = [0] * 4096
    e1[K.BRP_ROOTS_OF_UNITY.index(K.ROOTS_OF_UNITY[1])] = 1
    assert K.evaluate_polynomial_in_evaluation_form(e1, C.TAU) == setup_scalars[1]


@pytest.mark.parametrize("name,z", Z_CASES, ids=[n for n, _ in Z_CASES])
def test_quotient_opens_f_at_z(setup_scalars, poly, name, z):
    y = K.evaluate_polynomial_in_evaluation_form(poly, z)
    q = KP.compute_quotient(poly, z, y)
    f_tau = K.evaluate_polynomial_in_evaluation_form(poly, C.TAU)
    assert P.lincomb_scalar(q, setup_scalars) == (f_tau - y) * pow(C.TAU - z, -1, R) % R


def test_within_domain_quotient_is_the_spec_sum(poly):
    m = 2048
    z, y = K.BRP_ROOTS_OF_UNITY[m], poly[m]
    q = KP.compute_quotient(poly, z, y)
    want = sum((poly[i] - y) * K.BRP_ROOTS_OF_UNITY[i] * pow(z * (z - K.BRP_ROOTS_OF_UNITY[i]), -1, R)
               for i in range(4096) if i != m) % R
    assert q[m] == want == KP.compute_quotient_eval_within_domain(z, poly, y)


def test_mirror_setup_argument_checks():
    import nmsm

    with pytest.raises(ValueError):
        nmsm.KzgSetup(b"\0" * 100)
    with pytest.raises(ValueError):
        nmsm.KzgSetup([b"\0" * 48] * 4095)
    with pytest.raises(TypeError):
        nmsm.KzgSetup([1] * 4096)


# ---- host emulation of the prover bodies ---------------------------------------------------------------------------
@pytest.mark.parametrize("name,z", Z_CASES, ids=[n for n, _ in Z_CASES])
def test_emu_quotient_matches_oracle(poly, name, z):
    blob = b"".join(C.be(v) for v in poly)
    y = K.evaluate_polynomial_in_evaluation_form(poly, z)
    assert P.emu_quotient(blob, z, y) == (KP.compute_quotient(poly, z, y), True)


def test_emu_quotient_rejects_z_out_of_range(poly):
    blob = b"".join(C.be(v) for v in poly)
    q, ok = P.emu_quotient(blob, R, 0)
    assert not ok and q == poly  # the blob is left alone


def test_emu_compress_matches_oracle():
    rnd = random.Random(22)
    pts = [K.g1_mul(rnd.randrange(1, R), K.G1_GEN) for _ in range(6)]
    pts += [H.point_neg(p) for p in pts[:3]] + [K.G1_GEN, None]
    want = [H.g1_encode(p) for p in pts]
    assert {w[0] & 0x20 for w in want[:-1]} == {0, 0x20}  # both sort bits occur
    assert P.emu_compress(pts) == want


def test_emu_lincomb_matches_oracle():
    rnd = random.Random(23)
    points = [H.g1_encode(K.g1_mul(rnd.randrange(1, R), K.G1_GEN)) for _ in range(5)]
    rows = [[rnd.randrange(R) for _ in range(5)], [0, R - 1, 1, (R - 1) // 2, (R + 1) // 2], [0] * 5,
            [rnd.randrange(R) for _ in range(4)] + [R], [1 << 255] + [0] * 4]
    for lanes in (1, 2, 8):
        got = P.emu_lincomb(points, rows, lanes)
        for row, (c, ok) in zip(rows[:3], got[:3]):
            assert ok and c == KP.g1_lincomb(points, row)
        assert got[2][0] == C.IDENTITY
        assert [ok for _, ok in got[3:]] == [False, False]
