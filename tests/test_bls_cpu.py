"""BLS12-381 pairing without a GPU: the oracle's self-consistency (bilinearity, order r, non-degeneracy, sign/verify),
the generated Frobenius constants and the final-exponent identity, and the device bodies (fp12.cuh, pairing.cuh) run
on the host through tests/hostemu/pairing_emu.cpp, compared with the oracle bit for bit."""
import os
import random
import re
import subprocess
import sys

import pytest

import bls_cases as C
import nmsm
from oracle import bls_pairing_ref as B

P, N = B.P, B.N
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- oracle self-tests ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def e_gen():
    return B.pairing(C.g1_mul(1), C.g2_mul(1))


def test_oracle_generator_pairing_is_not_one_and_has_order_r(e_gen):
    assert e_gen != B.O12
    assert B.f12_pow(e_gen, N) == B.O12


def test_oracle_bilinearity(e_gen):
    rnd = random.Random(1)
    a, b = rnd.randrange(1, N), rnd.randrange(1, N)
    assert B.pairing(C.g1_mul(a), C.g2_mul(b)) == B.f12_pow(e_gen, a * b % N)


def test_oracle_inverse_pair_cancels():
    rnd = random.Random(2)
    p, q = C.g1_mul(rnd.randrange(1, N)), C.g2_mul(rnd.randrange(1, N))
    neg = B.affine(B.G1.fromAffine({"x": p[0], "y": p[1]}).negate())
    assert B.pairing_check([(neg, q), (p, q)])
    assert not B.pairing_check([(p, q), (p, q)])


def test_oracle_untwist_rejects_points_off_the_twist():
    q = C.g2_mul(1)
    with pytest.raises(AssertionError):
        B.untwist((q[0], (q[1][0], (q[1][1] + 1) % P)))


def test_oracle_sign_verify_round_trip():
    rnd = random.Random(3)
    sig, H, pk = C.keypair_item(rnd)
    assert B.bls_verify(sig, H, pk)
    sig2, H2, pk2 = C.keypair_item(rnd)
    assert not B.bls_verify(sig, H, pk2) and not B.bls_verify(sig, H2, pk) and not B.bls_verify(sig2, H, pk)


# ---- constants -----------------------------------------------------------------------------------------------------
def test_final_exponent_identity():
    """the hard-part chain of pairing.cuh computes 3 (p^4 - p^2 + 1) / r as l0 + l1 p + l2 p^2 + l3 p^3"""
    x = -B.X_ABS
    assert (P ** 4 - P ** 2 + 1) % N == 0
    l3 = (x - 1) ** 2
    l2 = l3 * x
    l1 = l2 * x - l3
    l0 = l1 * x + 3
    assert B.M * (P ** 4 - P ** 2 + 1) // N == l0 + l1 * P + l2 * P ** 2 + l3 * P ** 3
    assert B.FINAL_EXP == B.M * (P ** 6 - 1) * (P ** 2 + 1) * ((P ** 4 - P ** 2 + 1) // N)
    assert N % 3 != 0


def _generated():
    return subprocess.check_output([sys.executable, os.path.join(ROOT, "noble-curves_b200", "tools", "gen_consts.py")],
                                   text=True)


def test_generator_reproduces_committed_header():
    with open(os.path.join(ROOT, "noble-curves_b200", "csrc", "curve_consts.cuh")) as f:
        assert f.read() == _generated()


def test_frobenius_constants_are_their_defining_powers_of_xi():
    text = _generated()
    R = 1 << 384
    rinv = pow(R, -1, P)

    def const(name):
        m = re.search(r"%s\(int i\) \{\n    constexpr uint32_t t\[12\] = \{([^}]*)\}" % name, text)
        words = [int(w.strip().rstrip("u"), 16) for w in m.group(1).split(",")]
        return sum(w << (32 * i) for i, w in enumerate(words)) * rinv % P

    xi = (1, 1)
    for k in (1, 2, 3):
        e = P ** k - 1
        for nm, want in (("FROB6_C1_%d" % k, B.F2.pow(xi, e // 3)), ("FROB6_C2_%d" % k, B.F2.pow(xi, 2 * e // 3)),
                         ("FROB12_C1_%d" % k, B.F2.pow(xi, e // 6))):
            assert (const(nm + "_C0_MONT"), const(nm + "_C1_MONT")) == want, nm


# ---- host build of the device bodies -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def elems():
    rnd = random.Random(4)
    r12 = lambda: B.unflat([rnd.randrange(P) for _ in range(12)])  # noqa: E731
    return [r12() for _ in range(3)]


def test_fp12_mul_sqr_inverse_conj_match_oracle(elems):
    for a, b in zip(elems, elems[1:] + elems[:1]):
        assert C.emu_fp12(0, a, b) == B.f12_mul(a, b)
        assert C.emu_fp12(1, a) == B.f12_sqr(a)
        assert C.emu_fp12(3, a) == B.f12_inv(a)
        assert C.emu_fp12(7, a) == B.f12_conj(a)


def test_fp12_frobenius_matches_oracle(elems):
    a = elems[0]
    for k in (1, 2, 3):
        assert C.emu_fp12(3 + k, a) == B.f12_frobenius(a, k), k


def test_sparse_line_product_matches_full_product(elems):
    a = elems[1]
    l = ((elems[2][0][0], elems[2][0][1], elems[2][0][2]), B.Z6)
    line = ((l[0][0], l[0][1], (0, 0)), ((0, 0), l[0][2], (0, 0)))  # l0 + l1 v + l4 v w
    assert C.emu_fp12(10, a, l) == B.f12_mul(a, line)


def test_cyclotomic_square_and_exp_match_oracle(elems):
    c = B.f12_pow(elems[0], (P ** 6 - 1) * (P ** 2 + 1))
    assert C.emu_fp12(2, c) == B.f12_sqr(c)
    assert C.emu_fp12(8, c) == B.f12_pow(c, B.X_ABS)


def test_final_exponentiation_matches_oracle(elems):
    assert C.emu_fp12(9, elems[0]) == B.final_exp(elems[0])


def test_pairing_values_match_oracle():
    rnd = random.Random(6)
    g = (C.g1_mul(1), C.g2_mul(1))
    sub = (C.g1_mul(rnd.randrange(1, N)), C.g2_mul(rnd.randrange(1, N)))
    off = (C.g1_off_subgroup(rnd), C.g2_off_subgroup(rnd))
    for pairs in ([g], [sub], [(off[0], g[1])], [(g[0], off[1])], [off], [g, sub, (C.ID1, g[1])]):
        assert C.emu_pairing(pairs) == B.pairing_product(pairs)


def test_check_bodies_with_small_chunks_carry_products_across_chunks():
    rnd = random.Random(7)
    t2, f2, t3 = C.true_check(rnd, 2), C.false_check(rnd, 2), C.true_check(rnd, 3)
    checks = [t2, [], f2, t3 + t2, [(C.ID1, C.ID2)], f2 + t3, t3]
    want = [True, True, False, True, True, False, True]
    for chunk in (1, 2, 3, 5, 64):
        assert C.emu_pairing_check(checks, chunk) == (want, (None, None)), chunk
    bad = (t2[0][0][0], (t2[0][0][1] + 1) % P)
    _, err = C.emu_pairing_check([t2, [(bad, t2[0][1])], [(t2[0][0], (t2[0][1][0], ((0, 0))))]], 2)
    assert err == (2, 3)


def test_verify_bodies_match_oracle_on_edge_set():
    cases = C.edge_cases()
    got, err = C.emu_verify([c[1:] for c in cases], chunk=6)
    want = [B.bls_verify(*c[1:]) for c in cases]
    assert err is None
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    names = dict(zip((c[0] for c in cases), got))
    assert names["valid"] and names["valid-2"] and sum(got) == 2


def test_verify_bodies_report_bad_message_points():
    rnd = random.Random(9)
    sig, H, pk = C.keypair_item(rnd)
    bad = (H[0], (H[1][0], (H[1][1] + 1) % P))
    got, err = C.emu_verify([(sig, H, pk), (sig, bad, pk), (sig, ((P, 0), H[1]), pk)])
    assert err == 1 and got[0]


def test_mirror_argument_validation_without_device():
    G1, G2 = nmsm.bls12_381.G1.Point, nmsm.bls12_381.G2.Point
    sig, pk = bytes(96), bytes(48)
    with pytest.raises(NotImplementedError, match="hash-to-curve"):
        nmsm.bls12_381.verify(sig, b"msg", pk)
    with pytest.raises(ValueError, match="equal length"):
        nmsm.bls_verify_batch([sig], [G2.BASE, G2.BASE], [pk])
    with pytest.raises(ValueError, match="length 96"):
        nmsm.bls_verify_batch([bytes(95)], [G2.BASE], [pk])
    with pytest.raises(ValueError, match="length 48"):
        nmsm.bls_verify_batch([sig], [G2.BASE], [bytes(49)])
    with pytest.raises(TypeError, match="message"):
        nmsm.bls_verify_batch([sig], [G1.BASE], [pk])
    with pytest.raises(TypeError, match="pairs expected"):
        nmsm.pairing_check_batch([[(G2.BASE, G1.BASE)]])
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.bls_verify_batch_packed(sig, pk, bytes(191), 1)
    with pytest.raises(ValueError, match="pair count"):
        nmsm.pairing_check_batch_packed(bytes(96), bytes(192), C.offsets([2]), 1)
    assert nmsm._bls_g2_compress(G2.ZERO) == bytes([0xC0]) + bytes(95)
