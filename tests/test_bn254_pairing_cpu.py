"""bn254 pairing without a GPU: the oracle's self-consistency (bilinearity, order r, non-degeneracy), the generated
Frobenius and twist constants and the final-exponent identity, the device bodies (fp12.cuh, pairing_bn254.cuh,
pairing_check.cuh) run on the host through tests/hostemu/bn254_pairing_emu.cpp and compared with the oracle bit for bit,
and the Python mirror's argument and EIP-197 parsing errors."""
import math
import os
import random
import re
import subprocess
import sys

import pytest

import bn254_pairing_cases as C
import nmsm
from oracle import bn254_pairing_ref as B

P, N, U = B.P, B.N, B.U
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
    assert B.pairing_check([(C.g1_neg(p), q), (p, q)])
    assert not B.pairing_check([(p, q), (p, q)])


def test_oracle_untwist_rejects_points_off_the_twist():
    q = C.g2_mul(1)
    with pytest.raises(AssertionError):
        B.untwist((q[0], (q[1][0], (q[1][1] + 1) % P)))


# ---- constants -----------------------------------------------------------------------------------------------------
def test_final_exponent_identity():
    """the hard-part chain of pairing_bn254.cuh computes M (p^4 - p^2 + 1) / r as l0 + l1 p + l2 p^2 + l3 p^3"""
    assert (P ** 4 - P ** 2 + 1) % N == 0
    l0 = 1 + 6 * U + 12 * U ** 2 + 12 * U ** 3
    l1 = 4 * U + 6 * U ** 2 + 12 * U ** 3
    l2 = 6 * U + 6 * U ** 2 + 12 * U ** 3
    l3 = -1 + 4 * U + 6 * U ** 2 + 12 * U ** 3
    assert B.M == 2 * U * (6 * U * U + 3 * U + 1)
    assert B.M * (P ** 4 - P ** 2 + 1) // N == l0 + l1 * P + l2 * P ** 2 + l3 * P ** 3
    assert B.FINAL_EXP == B.M * (P ** 6 - 1) * (P ** 2 + 1) * ((P ** 4 - P ** 2 + 1) // N)
    assert math.gcd(B.M, N) == 1


def _generated():
    return subprocess.check_output([sys.executable, os.path.join(ROOT, "noble-curves_b200", "tools", "gen_consts.py")],
                                   text=True)


def _block(text, struct):
    return text[text.index("struct %s {" % struct):].split("\n};", 1)[0]


def _const(block, name):
    m = re.search(r"%s\(int i\) \{\n    constexpr uint32_t t\[(\d+)\] = \{([^}]*)\}" % name, block)
    words = [int(w.strip().rstrip("u"), 16) for w in m.group(2).split(",")]
    return sum(w << (32 * i) for i, w in enumerate(words))


def test_frobenius_and_twist_constants_are_their_defining_powers_of_xi():
    frob = _block(_generated(), "Bn254Frob")
    rinv = pow(1 << 256, -1, P)
    f2 = lambda nm: (_const(frob, nm + "_C0_MONT") * rinv % P, _const(frob, nm + "_C1_MONT") * rinv % P)  # noqa: E731
    xi = B.XI
    for k in (1, 2, 3):
        e = P ** k - 1
        for nm, want in (("FROB6_C1_%d" % k, B.F2.pow(xi, e // 3)), ("FROB6_C2_%d" % k, B.F2.pow(xi, 2 * e // 3)),
                         ("FROB12_C1_%d" % k, B.F2.pow(xi, e // 6))):
            assert f2(nm) == want, nm
    assert f2("TWIST_X1") == B.F2.pow(xi, (P - 1) // 3)
    assert f2("TWIST_Y1") == B.F2.pow(xi, (P - 1) // 2)
    assert (_const(frob, "TWIST_X2_MONT") * rinv % P, 0) == B.F2.pow(xi, (P * P - 1) // 3)
    assert B.F2.pow(xi, (P * P - 1) // 2) == (P - 1, 0)  # so -pi^2(x', y') = (x' TWIST_X2, y')


def test_twist_frobenius_constants_agree_with_the_untwisted_frobenius():
    """pi(Q) from the constants equals the oracle's p-th power of the untwisted point, and -pi^2(Q) likewise"""
    frob = _block(_generated(), "Bn254Frob")
    rinv = pow(1 << 256, -1, P)
    f2 = lambda nm: (_const(frob, nm + "_C0_MONT") * rinv % P, _const(frob, nm + "_C1_MONT") * rinv % P)  # noqa: E731
    q = C.g2_mul(7)
    conj = lambda a: (a[0], (-a[1]) % P)  # noqa: E731
    x, y = B.untwist(q)
    q1 = (B.F2.mul(conj(q[0]), f2("TWIST_X1")), B.F2.mul(conj(q[1]), f2("TWIST_Y1")))
    assert B.untwist(q1) == (B.f12_frobenius(x, 1), B.f12_frobenius(y, 1))
    q2 = (B.F2.mul(q[0], _const(frob, "TWIST_X2_MONT") * rinv % P), q[1])
    assert B.untwist(q2) == (B.f12_frobenius(x, 2), B.f12_sub(B.from_fp(0), B.f12_frobenius(y, 2)))


def test_ate_loop_constants():
    ate = _block(_generated(), "Bn254Ate")
    assert _const(ate, "U") == U and U.bit_length() == 63 and bin(U).count("1") == 28
    pos, neg = _const(ate, "NAF_POS"), _const(ate, "NAF_NEG")
    assert pos - neg == 6 * U + 2 == 0x19D797039BE763BA8
    assert pos & neg == 0 and (pos | neg) & ((pos | neg) >> 1) == 0  # non-adjacent
    assert (pos | neg).bit_length() == 66 and bin(pos | neg).count("1") == 22
    rinv = pow(1 << 256, -1, P)
    b3 = (_const(ate, "B3_C0_MONT") * rinv % P, _const(ate, "B3_C1_MONT") * rinv % P)
    assert b3 == B.F2.mul(C.B2, 3) and B.F2.mul(C.B2, B.XI) == (3, 0)  # b' = 3 / xi: the D-type twist


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
    line = ((l[0][0], (0, 0), (0, 0)), (l[0][1], l[0][2], (0, 0)))  # l0 + l3 w + l4 v w
    assert C.emu_fp12(10, a, l) == B.f12_mul(a, line)


def test_cyclotomic_square_and_exp_match_oracle(elems):
    c = B.f12_pow(elems[0], (P ** 6 - 1) * (P ** 2 + 1))
    assert C.emu_fp12(2, c) == B.f12_sqr(c)
    assert C.emu_fp12(8, c) == B.f12_pow(c, U)


def test_final_exponentiation_matches_oracle(elems):
    assert C.emu_fp12(9, elems[0]) == B.final_exp(elems[0])


def test_pairing_values_match_oracle():
    rnd = random.Random(6)
    g = (C.g1_mul(1), C.g2_mul(1))
    sub = (C.g1_mul(rnd.randrange(1, N)), C.g2_mul(rnd.randrange(1, N)))
    q_off = C.g2_off_subgroup(rnd)
    for pairs in ([g], [sub], [(g[0], q_off)], [(sub[0], q_off), sub], [g, sub, (C.ID1, g[1]), (g[0], C.ID2)], []):
        assert C.emu_pairing(pairs) == B.pairing_product(pairs)


def test_check_bodies_with_small_chunks_carry_products_across_chunks():
    rnd = random.Random(7)
    t2, f2, t3 = C.true_check(rnd, 2), C.false_check(rnd, 2), C.true_check(rnd, 3)
    g16 = C.groth16_check(rnd)
    checks = [t2, [], f2, t3 + t2, [(C.ID1, C.ID2)], f2 + t3, t3, g16, C.groth16_check(rnd, perturb=True)]
    want = [True, True, False, True, True, False, True, True, False]
    for chunk in (1, 2, 3, 5, 64):
        assert C.emu_pairing_check(checks, chunk) == (want, (None, None)), chunk
    bad = (t2[0][0][0], (t2[0][0][1] + 1) % P)
    _, err = C.emu_pairing_check([t2, [(bad, t2[0][1])], [(t2[0][0], (t2[0][1][0], (0, 0)))]], 2)
    assert err == (2, 3)
    _, err = C.emu_pairing_check([t2, [((P, 0), t2[0][1]), (t2[0][0], ((P, 0), (0, 0)))]], 3)
    assert err == (2, 3)


# ---- Python mirror without a device ------------------------------------------------------------------------------
def test_mirror_argument_validation_without_device():
    G1, G2 = nmsm.bn254.G1.Point, nmsm.bn254.G2.Point
    with pytest.raises(TypeError, match="pairs expected"):
        nmsm.bn254_pairing_check_batch([[(G2.BASE, G1.BASE)]])
    with pytest.raises(TypeError, match="pairs expected"):
        nmsm.bn254_pairing_check_batch([[(nmsm.bls12_381.G1.Point.BASE, G2.BASE)]])
    with pytest.raises(ValueError, match="pair count"):
        nmsm.bn254_pairing_check_batch_packed(bytes(64), bytes(128), C.offsets([2]), 1)
    with pytest.raises(ValueError, match="n_checks"):
        nmsm.bn254_pairing_check_batch_packed(bytes(64), bytes(128), C.offsets([1]), 2)


def test_eip197_parsing_errors_without_device():
    g = (C.g1_mul(1), C.g2_mul(1))
    good = C.eip197_bytes([g])
    with pytest.raises(TypeError, match="input 0"):
        nmsm.bn254_eip197_pairing_batch(["00"])
    with pytest.raises(ValueError, match="input 1: length 191"):
        nmsm.bn254_eip197_pairing_batch([good, good[:-1]])
    for k in range(6):  # every coordinate, including both halves of both Fp2 values
        bad = bytearray(good)
        bad[32 * k:32 * k + 32] = P.to_bytes(32, "big")
        with pytest.raises(ValueError, match="input 2: .*>= p"):
            nmsm.bn254_eip197_pairing_batch([good, b"", bytes(bad)])
    assert nmsm.bn254_eip197_pairing_batch([]) == []
