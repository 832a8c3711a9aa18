"""BLS12-381 aggregate verification without a GPU: the oracle (oracle.bls_aggregate_ref) on aggregates built by
construction and against single verification, the device bodies (bls_aggregate.cuh) run on the host through
tests/hostemu/bls_agg_emu.cpp against the oracle at small tile sizes and Miller chunks, and the host mirror's argument
checks and packing."""
import random

import pytest

import bls_agg_cases as C
import bls_cases as BC
import nmsm
from oracle import bls_aggregate_ref as A
from oracle import bls_pairing_ref as B


@pytest.fixture(scope="module")
def edge():
    cases = C.edge_checks()
    return cases, C.oracle([c for _, c in cases])


def test_oracle_real_aggregate_verifies():
    rnd = random.Random(1)
    sks = [rnd.randrange(1, B.N) for _ in range(4)]
    pks = [BC.g1_mul(k) for k in sks]
    sig = C.sign_agg(sks, b"block-root")
    assert A.aggregate_verify(sig, [(b"block-root", pks)], C.DST)
    assert not A.aggregate_verify(sig, [(b"block-root", pks[:3])], C.DST)
    assert not A.aggregate_verify(sig, [(b"block-root", pks)], b"OTHER-TAG")
    # the same keys split over two groups of the same message sum to the same pairing product
    assert A.aggregate_verify(sig, [(b"block-root", pks[:2]), (b"block-root", pks[2:])], C.DST)


def test_oracle_one_key_one_group_equals_bls_verify():
    rnd = random.Random(2)
    sk, other = rnd.randrange(1, B.N), rnd.randrange(1, B.N)
    msg = b"one signer"
    h = A.hashed(msg, C.DST)
    for sig, pk in ((C.sign_agg([sk], msg), sk), (C.sign_agg([sk], msg), other), (C.sign_agg([other], msg), sk)):
        want = B.bls_verify(sig, h, B.public_key(pk))
        assert A.aggregate_verify(sig, [(msg, [BC.g1_mul(pk)])], C.DST) == want


def test_oracle_edge_verdicts(edge):
    cases, want = edge
    got = dict(zip([n for n, _ in cases], want))
    for name in ("valid-3", "valid-1", "valid-two-groups", "p-and-minus-p", "duplicate-key"):
        assert got[name], name
    for name in ("empty-check", "empty-group", "identity-key", "sum-identity", "wrong-message", "swapped-key",
                 "sig-identity", "sig-off-subgroup", "sig-nonsquare", "key-off-subgroup"):
        assert not got[name], name


@pytest.mark.parametrize("tile,chunk,cap", [(1, 1, 1 << 20), (2, 2, 1 << 20), (3, 5, 1 << 20), (32, 1, 1 << 20),
                                            (32, 5, 1 << 20), (1, 2, 2), (2, 5, 1)])
def test_serial_statement_matches_oracle(edge, tile, chunk, cap):
    cases, want = edge
    got, bad_key, pair_err = C.emu_aggregate([c for _, c in cases], tile, chunk, cap)
    assert bad_key is None and pair_err == (None, None)
    assert got == want, [n for (n, _), g, w in zip(cases, got, want) if g != w]


def test_serial_statement_reports_the_smallest_bad_key():
    rnd = random.Random(3)
    sks = [rnd.randrange(1, B.N) for _ in range(3)]
    pks = [BC.g1_mul(k) for k in sks]
    sig = C.sign_agg(sks, b"m")
    x = 5
    while pow((x ** 3 + 4) % B.P, (B.P - 1) // 2, B.P) == 1:
        x += 1
    off_curve = (x, 1)
    big_x = (B.P, pks[0][1])
    checks = [(sig, [(b"m", pks)]), (sig, [(b"m", pks[:2] + [off_curve]), (b"n", [big_x])])]
    for tile in (1, 32):
        _, bad_key, _ = C.emu_aggregate(checks, tile, 5)
        assert bad_key == 5
    checks = [(sig, [(b"m", pks)]), (sig, [(b"m", [big_x] + pks[:2])])]
    assert C.emu_aggregate(checks, 2, 5)[1] == 3


def test_mirror_layout_and_grouping_without_device():
    k1, k2 = bytes(48), b"\x01" * 48
    sigs, goff, msgs, koff, keys = nmsm._bls_agg_layout([(b"s" * 96, [(b"a", [k1, k2]), (b"", [k1])]),
                                                         (b"t" * 96, [])])
    assert sigs == [b"s" * 96, b"t" * 96] and goff == [0, 2, 2] and msgs == [b"a", b""]
    assert koff == [0, 2, 3] and keys == [k1, k2, k1]
    # verifyBatch: pairs with equal message bytes form one group, in first-seen order
    groups = nmsm._bls_verify_batch_groups([b"x", b"y", bytearray(b"x"), b"z"], ["k0", "k1", "k2", "k3"])
    assert groups == [(b"x", ["k0", "k2"]), (b"y", ["k1"]), (b"z", ["k3"])]


def test_mirror_argument_validation_without_device():
    G2 = nmsm.bls12_381.G2.Point
    with pytest.raises(TypeError, match="bytes"):
        nmsm.bls12_381.verifyBatch(bytes(96), [G2.BASE], [bytes(48)])
    with pytest.raises(TypeError, match="bytes"):
        nmsm.bls_aggregate_verify_batch([(bytes(96), [(G2.BASE, [bytes(48)])])])
    with pytest.raises(ValueError, match="equal length"):
        nmsm.bls12_381.verifyBatch(bytes(96), [b"m", b"n"], [bytes(48)])
    with pytest.raises(ValueError, match="equal length"):
        nmsm.bls_fast_aggregate_verify_batch([bytes(96)], [b"m", b"n"], [[bytes(48)]])
    with pytest.raises(TypeError, match="check 0"):
        nmsm.bls_aggregate_verify_batch([bytes(96)])
    with pytest.raises(ValueError, match="length 96"):
        nmsm.bls_aggregate_verify_batch([(bytes(95), [(b"m", [bytes(48)])])])
    with pytest.raises(TypeError, match="message"):
        nmsm.bls_aggregate_verify_batch([(bytes(96), [("m", [bytes(48)])])])
    with pytest.raises(ValueError, match="non-empty"):
        nmsm.bls_aggregate_verify_batch([(bytes(96), [(b"m", [bytes(48)])])], b"")
    with pytest.raises(TypeError, match="publicKey"):
        nmsm._bls_agg_keys([5])
    with pytest.raises(ValueError, match="length 48"):
        nmsm._bls_agg_keys([bytes(47)])
    with pytest.raises(ValueError, match="n_checks"):
        nmsm.bls_aggregate_verify_batch_packed(bytes(96), bytes(8), b"", bytes(8), b"", bytes(8), 1, b"D")
    with pytest.raises(ValueError, match="group count"):
        nmsm.bls_aggregate_verify_batch_packed(bytes(96), bytes(8) + (1).to_bytes(8, "little"), b"", bytes(8), b"",
                                               bytes(16), 1, b"D")
    assert nmsm.bls_aggregate_verify_batch([]) == []
    assert nmsm.bls_fast_aggregate_verify_batch([], [], []) == []
