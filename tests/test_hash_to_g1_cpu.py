"""Hash to BLS12-381 G1 and short-signature verification without a GPU: the oracle (oracle.hash_to_g1_ref) against the
RFC 9380 J.9.1 known answers and the isogeny's curve identity, the device bodies (hash_to_curve.cuh, pairing.cuh) run on
the host through tests/hostemu against the oracle step by step and end to end, the prepare body's verdicts on the edge
set, and the host mirror's argument checks."""
import random

import pytest

import h2g1_cases as C
import nmsm
from oracle import hash_to_g1_ref as H

P = H.P


def test_oracle_known_answers():
    for msg, want in C.KATS.items():
        pt = H.hash_to_g1(msg, H.DST_QUUX)
        assert pt == want, msg
        assert H.in_g1(pt)


def test_isogeny_maps_e1_prime_onto_e1():
    """for random points of E1', (x_num/x_den, y' y_num/y_den) satisfies y^2 = x^3 + 4: one wrong coefficient of the
    11-isogeny breaks this"""
    rnd = random.Random(1)
    hits = 0
    while hits < 24:
        x = rnd.randrange(P)
        y = H.sqrt(H.g_iso(x))
        if y is None:
            continue
        hits += 1
        img = H.iso_map((x, y))
        assert img is not None and H.on_e1(img), hex(x)


def test_oracle_sswu_lands_on_e1_prime_and_outputs_in_g1():
    for name, u in C.special_us():
        x, y = H.map_to_curve_sswu(u)
        assert y * y % P == H.g_iso(x) and H.sgn0(y) == H.sgn0(u), name
    for msg in C.random_messages(6, seed=1, max_len=80):
        pt = H.hash_to_g1(msg, H.DST_G1_POP)
        assert pt is not None and H.in_g1(pt)
    assert H.H_EFF == 1 - H.X


def test_oracle_oversize_dst_rule():
    long_dst = bytes(range(256)) + b"x" * 44
    tag = H.dst_prime_tag(long_dst)
    assert len(tag) == 32 and H.hash_to_field(b"m", long_dst) == H.hash_to_field(b"m", tag)


def test_host_hash_to_field_matches_oracle():
    for dlen in list(range(1, 256, 17)) + [255]:
        dst = bytes((5 * k + 3) & 0xFF for k in range(dlen))
        for msg in C.random_messages(len(C.EDGE_LENGTHS), seed=dlen):
            assert C.emu_hash_to_field(msg, dst) == H.hash_to_field(msg, dst), (len(msg), dlen)
    # an oversize tag reaches the device as its 32-byte hash
    long_dst = bytes(range(256)) * 2
    assert C.emu_hash_to_field(b"abc", H.dst_prime_tag(long_dst)) == H.hash_to_field(b"abc", long_dst)


def test_host_map_special_branches():
    """u = 0 and u = +-sqrt(-1/11) take the tv1 = 0 branch; g(x1) non-square takes x2 = Z u^2 x1 with the
    sqrt(-Z) root; every point lands on E1' and then E1"""
    cases = dict(C.special_us())
    assert H.sqrt(H.g_iso(C._x1(cases["gx1-nonsquare"]))) is None
    for name, u in cases.items():
        want = H.map_to_curve_sswu(u)
        assert C.emu_sswu(u) == want, name
        assert C.emu_iso_map(want) == H.iso_map(want), name
        assert H.on_e1(H.iso_map(want)), name
    for name in ("u=0", "u=sqrt(-1/Z)", "u=-sqrt(-1/Z)"):
        u = cases[name]
        zu2 = H.Z_SSWU * u * u % P
        assert (zu2 * zu2 + zu2) % P == 0, name


def test_host_iso_map_on_random_points():
    rnd = random.Random(3)
    n = 0
    while n < 8:
        x = rnd.randrange(P)
        y = H.sqrt(H.g_iso(x))
        if y is None:
            continue
        n += 1
        assert C.emu_iso_map((x, y)) == H.iso_map((x, y))


def test_host_clear_cofactor_is_h_eff_off_g1():
    pts = C.e1_non_subgroup_points(6) + [None]
    for pt in pts:
        want = H.clear_cofactor(pt)
        assert C.emu_clear_cofactor(pt) == want
        assert want is None or H.in_g1(want)
    q = pts[0]
    assert C.emu_clear_cofactor(H.point_add(q, q)) == H.clear_cofactor(H.point_add(q, q))
    # a point of order 3 (x = 0, y = 2): cleared to the identity, or to a point of G1
    assert C.emu_clear_cofactor((0, 2)) == H.clear_cofactor((0, 2))


def test_host_hash_matches_oracle_on_200_messages():
    msgs = C.random_messages(200, seed=3)
    got = C.emu_hash(msgs, H.DST_G1_NUL)
    want = C.oracle_packed(msgs, H.DST_G1_NUL)
    bad = [k for k in range(len(msgs)) if got[k] != want[k]]
    assert not bad, [len(msgs[k]) for k in bad]


def test_host_hash_known_answers():
    assert C.emu_hash(list(C.KATS), H.DST_QUUX) == [C.kat_packed(v) for v in C.KATS.values()]


def test_host_short_verify_edge_set():
    cases = C.edge_cases()
    items = [(sig, H.hash_to_g1(msg, H.DST_G1_NUL), pk) for _, sig, msg, pk in cases]
    got, err = C.emu_short_verify(items)
    want = [H.short_verify(*it) for it in items]
    assert err is None
    assert got == want, [(c[0], g, w) for c, g, w in zip(cases, got, want) if g != w]
    names = {c[0]: v for c, v in zip(cases, want)}
    assert names["valid"] and names["valid-2"] and names["valid-empty-message"]
    assert sum(want) == 3


def test_host_short_verify_message_point_errors():
    (sig, msg, pk), = C.signed_triples(1, seed=8)
    h = H.hash_to_g1(msg, H.DST_G1_NUL)
    items = [(sig, h, pk), (sig, None, pk), (sig, (h[0], (h[1] + 1) % P), pk), (sig, (P, 2), pk)]
    got, err = C.emu_short_verify(items)
    assert got[:2] == [True, False] and err == 2


def test_mirror_argument_validation_without_device():
    with pytest.raises(ValueError, match="non-empty"):
        nmsm.bls_hash_to_g1_batch([b"m"], b"")
    with pytest.raises(TypeError, match="message"):
        nmsm.bls_hash_to_g1_batch(["m"])
    with pytest.raises(TypeError, match="DST"):
        nmsm.bls_hash_to_g1_batch([b"m"], 5)
    with pytest.raises(TypeError, match="options"):
        nmsm.bls12_381.G1.hashToCurve(b"m", "DST")
    with pytest.raises(ValueError, match="equal length"):
        nmsm.bls_short_verify_messages_batch([bytes(48)], [b"m", b"n"], [bytes(96)])
    with pytest.raises(ValueError, match="equal length"):
        nmsm.bls_short_verify_batch([bytes(48)], [], [bytes(96)])
    with pytest.raises(ValueError, match="length 48"):
        nmsm.bls_short_verify_messages_batch([bytes(96)], [b"m"], [bytes(48)])  # a long-signature pair
    with pytest.raises(ValueError, match="length 96"):
        nmsm.bls_short_verify_messages_batch([bytes(48)], [b"m"], [bytes(48)])
    with pytest.raises(TypeError, match="signature"):
        nmsm.bls_short_verify_messages_batch([nmsm.bls12_381.G2.Point.BASE], [b"m"], [bytes(96)])
    with pytest.raises(TypeError, match="publicKey"):
        nmsm.bls_short_verify_messages_batch([bytes(48)], [b"m"], [nmsm.bls12_381.G1.Point.BASE])
    with pytest.raises(TypeError, match="G1.Point"):
        nmsm.bls_short_verify_batch([bytes(48)], [b"m"], [bytes(96)])
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.bls_hash_to_g1_batch_packed(b"m", bytes(8), 1, b"D")
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.bls_short_verify_batch_packed(bytes(48), bytes(96), bytes(95), 1)
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.bls_short_verify_messages_batch_packed(bytes(48), bytes(96), b"m", bytes(8), 1, b"D")
    assert nmsm.bls_hash_to_g1_batch([]) == []
    assert nmsm.bls_short_verify_batch([], [], []) == []
    assert nmsm.bls_short_verify_messages_batch([], [], []) == []
    assert nmsm.DST_G1_NUL == H.DST_G1_NUL and nmsm.DST_G1_POP == H.DST_G1_POP
    # the long-signature entry points keep refusing byte messages
    with pytest.raises(NotImplementedError, match="hash-to-curve"):
        nmsm.bls_verify_batch([bytes(96)], [b"m"], [bytes(48)])
