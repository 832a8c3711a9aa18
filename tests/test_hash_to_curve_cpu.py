"""Hash to BLS12-381 G2 without a GPU: the oracle (oracle.hash_to_curve_ref) against the RFC 9380 known answers and the
group structure, the device bodies (hash_to_curve.cuh) run on the host through tests/hostemu against the oracle, step by
step on chosen inputs and end to end on 200 messages, and the host mirror's argument checks."""
import random

import pytest

import h2c_cases as C
import nmsm
from oracle import hash_to_curve_ref as H


def test_oracle_known_answers():
    dst, msg, ln, want = C.XMD_KAT
    assert H.expand_message_xmd(msg, dst, ln) == want
    for msg, want in C.KATS.items():
        assert H.g2_packed(H.hash_to_g2(msg, H.DST_QUUX)) == C.kat_packed(want), msg


def test_oracle_h_eff_and_outputs_in_g2():
    assert H.H_EFF == 3 * (H.X * H.X - 1) * H.H2
    for msg in C.random_messages(6, seed=1, max_len=80):
        pt = H.hash_to_g2(msg, H.DST_G2_POP)
        assert pt is not None and H.on_e2(pt) and H.in_g2(pt)


def test_oracle_oversize_dst_rule():
    long_dst = bytes(range(256))
    tag = H.dst_prime_tag(long_dst)
    assert len(tag) == 32 and H.expand_message_xmd(b"m", long_dst, 256) == H.expand_message_xmd(b"m", tag, 256)
    assert H.dst_prime_tag(long_dst[:255]) == long_dst[:255]


def test_host_reduce512_is_canonical_at_the_bounds():
    p = H.P
    rnd = random.Random(2)
    edges = [0, 1, p - 1, p, p + 1, 2 ** 384 - 1, 2 ** 384, 2 ** 512 - 1, p * 2 ** 128, (p - 1) * 2 ** 128 + 2 ** 384 - 1,
             int.from_bytes(b"\xff" * 64, "big"), int.from_bytes(b"\xff" * 16 + bytes(48), "big")]
    edges += [rnd.randrange(2 ** 512) for _ in range(50)]
    for e in edges:
        assert C.emu_reduce512(e) == e % p, hex(e)


def test_host_hash_to_field_matches_oracle():
    for dst in (b"D", H.DST_G2_POP, H.DST_QUUX, bytes(range(1, 256))):
        for msg in C.random_messages(len(C.EDGE_LENGTHS), seed=len(dst)):
            assert C.emu_hash_to_field(msg, dst) == H.hash_to_field(msg, dst), (len(msg), len(dst))


def test_host_map_special_branches():
    """u = 0 takes the tv1 = 0 branch; gx1 non-square takes x2 = Z u^2 x1; every point lands on E2' and then E2"""
    cases = C.special_us()
    assert H.sqrt(H.g_iso(H.map_to_curve_sswu(dict(cases)["gx1-nonsquare"])[0])) is not None
    for name, u in cases:
        want = H.map_to_curve_sswu(u)
        assert C.emu_sswu(u) == want, name
        assert C.emu_iso_map(want) == H.iso_map(want), name
        assert H.on_e2(H.iso_map(want)), name
    # u = 0: x1 = B'/(Z A'), whose g is a square, so the first branch is taken
    x0, _ = H.map_to_curve_sswu((0, 0))
    assert x0 == H.mul(H.B_ISO, H.inv(H.mul(H.Z_SSWU, H.A_ISO)))


def test_host_clear_cofactor_is_h_eff_on_all_of_e2():
    pts = C.e2_non_subgroup_points(6) + [None]
    for pt in pts:
        assert C.emu_clear_cofactor(pt) == H.clear_cofactor(pt)
    # points whose sum is the identity or a doubling reach the complete branches of the addition
    q = C.e2_non_subgroup_points(1, seed=4)[0]
    assert C.emu_clear_cofactor(H.point_add(q, q)) == H.clear_cofactor(H.point_add(q, q))


def test_host_hash_matches_oracle_on_200_messages():
    msgs = C.random_messages(200, seed=3)
    got = C.emu_hash(msgs, H.DST_G2_NUL)
    want = C.oracle_packed(msgs, H.DST_G2_NUL)
    bad = [k for k in range(len(msgs)) if got[k] != want[k]]
    assert not bad, [len(msgs[k]) for k in bad]


def test_host_hash_known_answers():
    got = C.emu_hash(list(C.KATS), H.DST_QUUX)
    assert got == [C.kat_packed(v) for v in C.KATS.values()]


def test_mirror_argument_validation_without_device():
    with pytest.raises(ValueError, match="non-empty"):
        nmsm.bls_hash_to_g2_batch([b"m"], b"")
    with pytest.raises(TypeError, match="message"):
        nmsm.bls_hash_to_g2_batch(["m"])
    with pytest.raises(TypeError, match="DST"):
        nmsm.bls_hash_to_g2_batch([b"m"], 5)
    with pytest.raises(TypeError, match="options"):
        nmsm.bls12_381.G2.hashToCurve(b"m", "DST")
    with pytest.raises(ValueError, match="equal length"):
        nmsm.bls_verify_messages_batch([bytes(96)], [b"m", b"n"], [bytes(48)])
    with pytest.raises(ValueError, match="length 96"):
        nmsm.bls_verify_messages_batch([bytes(95)], [b"m"], [bytes(48)])
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.bls_hash_to_g2_batch_packed(b"m", bytes(8), 1, b"D")
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.bls_verify_messages_batch_packed(bytes(96), bytes(48), b"m", bytes(8), 1, b"D")
    assert nmsm.bls_hash_to_g2_batch([]) == []
    assert nmsm.bls_verify_messages_batch([], [], []) == []
    # byte messages still raise in the hashed-point entry points
    with pytest.raises(NotImplementedError, match="hash-to-curve"):
        nmsm.bls_verify_batch([bytes(96)], [b"m"], [bytes(48)])
