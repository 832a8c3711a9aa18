"""Hash to BLS12-381 G2 and BLS verification from message bytes on the GPU (nmsm_bls12_381_hash_to_g2_batch,
nmsm_bls12_381_verify_msg_batch): points compared byte for byte with the oracle (oracle.hash_to_curve_ref), verdicts
with the oracle's verification and with nmsm_bls12_381_verify_batch on the same messages hashed first."""
import ctypes
import random

import pytest

import bls_cases as BC
import h2c_cases as C
from oracle import bls_pairing_ref as B
from oracle import hash_to_curve_ref as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _hash(nmsm, msgs, dst):
    data, off = C.pack_messages(msgs)
    xy = nmsm.bls_hash_to_g2_batch_packed(data, off, len(msgs), dst)
    return [xy[192 * k:192 * k + 192] for k in range(len(msgs))]


def test_known_answers_through_the_c_abi(nmsm):
    assert _hash(nmsm, list(C.KATS), H.DST_QUUX) == [C.kat_packed(v) for v in C.KATS.values()]
    pt = nmsm.bls12_381.G2.hashToCurve(b"abc", {"DST": H.DST_QUUX})
    assert pt.to_packed() == C.kat_packed(C.KATS[b"abc"]) and pt._valid


def test_4096_messages_match_oracle_and_are_torsion_free(nmsm):
    msgs = C.random_messages(4096, seed=7)
    got = _hash(nmsm, msgs, H.DST_G2_NUL)
    want = C.oracle_packed(msgs, H.DST_G2_NUL)
    bad = [k for k in range(len(msgs)) if got[k] != want[k]]
    assert not bad, [(k, len(msgs[k])) for k in bad[:10]]
    ok = nmsm.torsion_free_packed(7, b"".join(got), len(got))
    assert ok == b"\1" * len(got)


@pytest.mark.parametrize("dlen", [1, 43, 255, 256, 300])
def test_dst_lengths(nmsm, dlen):
    dst = H.DST_G2_POP if dlen == 43 else bytes((7 * k + 1) & 0xFF for k in range(dlen))
    msgs = C.random_messages(len(C.EDGE_LENGTHS), seed=dlen)
    assert _hash(nmsm, msgs, dst) == C.oracle_packed(msgs, dst, workers=1)


def test_mirror_returns_g2_points(nmsm):
    pts = nmsm.bls_hash_to_g2_batch([b"", b"x" * 100], H.DST_G2_POP)
    assert [p.to_packed() for p in pts] == C.oracle_packed([b"", b"x" * 100], H.DST_G2_POP, workers=1)
    assert nmsm.bls12_381.G2.hashToCurve(b"m").to_packed() == H.g2_packed(H.hash_to_g2(b"m", H.DST_G2_NUL))


def test_n_zero_and_more_than_one_block(nmsm):
    assert nmsm.bls_hash_to_g2_batch([]) == []
    msgs = [bytes([k & 0xFF, k >> 8]) for k in range(300)]  # 3 blocks of 128 threads, the last partial
    got = _hash(nmsm, msgs, b"T")
    sample = list(range(0, 300, 37)) + [255, 256, 299]
    assert [got[k] for k in sample] == C.oracle_packed([msgs[k] for k in sample], b"T", workers=1)


def test_error_codes(nmsm):
    lib = nmsm._lib.load()
    out = ctypes.create_string_buffer(192)
    off = (ctypes.c_uint64 * 2)(0, 1)
    m = ctypes.c_char_p(b"m")
    d = ctypes.c_char_p(b"D")
    ERR_ARG = nmsm._lib.ERR_ARG
    assert lib.nmsm_bls12_381_hash_to_g2_batch(m, off, 1, d, 0, out) == ERR_ARG  # empty DST
    assert lib.nmsm_bls12_381_hash_to_g2_batch(m, off, 1, None, 1, out) == ERR_ARG
    assert lib.nmsm_bls12_381_hash_to_g2_batch(m, None, 1, d, 1, out) == ERR_ARG
    assert lib.nmsm_bls12_381_hash_to_g2_batch(None, off, 1, d, 1, out) == ERR_ARG
    assert lib.nmsm_bls12_381_hash_to_g2_batch(m, off, 1 << 30, d, 1, out) == ERR_ARG
    bad0 = (ctypes.c_uint64 * 2)(1, 1)
    assert lib.nmsm_bls12_381_hash_to_g2_batch(m, bad0, 1, d, 1, out) == ERR_ARG
    dec = (ctypes.c_uint64 * 3)(0, 1, 0)
    assert lib.nmsm_bls12_381_hash_to_g2_batch(m, dec, 2, d, 1, out) == ERR_ARG
    assert b"non-decreasing" in lib.nmsm_last_error()
    assert lib.nmsm_bls12_381_hash_to_g2_batch(None, None, 0, d, 1, None) == 0  # n = 0 writes nothing
    sig, pk, ok = ctypes.c_char_p(bytes(96)), ctypes.c_char_p(bytes(48)), ctypes.create_string_buffer(1)
    assert lib.nmsm_bls12_381_verify_msg_batch(sig, pk, m, off, 1, d, 0, ok) == ERR_ARG
    assert lib.nmsm_bls12_381_verify_msg_batch(None, pk, m, off, 1, d, 1, ok) == ERR_ARG
    assert lib.nmsm_bls12_381_verify_msg_batch(sig, pk, m, bad0, 1, d, 1, ok) == ERR_ARG
    assert lib.nmsm_bls12_381_verify_msg_batch(sig, pk, m, off, 1 << 30, d, 1, ok) == ERR_ARG
    with pytest.raises(nmsm.NmsmError):
        nmsm.bls_hash_to_g2_batch_packed(b"m", bytes(16), 1, b"")


def _signed(rnd, msg, dst):
    sk = rnd.randrange(1, B.N)
    h = H.hash_to_g2(msg, dst)
    hp = B.G2.fromAffine({"x": h[0], "y": h[1]})
    return B.sign(sk, hp), B.public_key(sk)


def test_verify_msg_against_oracle(nmsm):
    """valid, corrupted-signature, wrong-message, wrong-DST and undecodable-key items in one batch"""
    rnd = random.Random(9)
    dst, other = H.DST_G2_POP, H.DST_G2_NUL
    sigs, msgs, pks, want = [], [], [], []
    for k in range(48):
        msg = bytes(rnd.randrange(256) for _ in range(rnd.randrange(120)))
        kind = k % 6
        sig, pk = _signed(rnd, msg, other if kind == 3 else dst)
        if kind == 1:  # corrupted signature: another valid encoding
            sig, _ = _signed(rnd, msg + b"!", dst)
        elif kind == 2:  # wrong message
            msg = msg + b"?"
        elif kind == 4:  # undecodable key: x >= p
            pk = bytes([0x9A]) + b"\xff" * 47
        elif kind == 5:  # identity key
            pk = bytes([0xC0]) + bytes(47)
        sigs.append(sig)
        msgs.append(msg)
        pks.append(pk)
        want.append(kind == 0)
    got = nmsm.bls_verify_messages_batch(sigs, msgs, pks, dst)
    assert got == want
    hashed = nmsm.bls_hash_to_g2_batch(msgs, dst)
    assert nmsm.bls_verify_batch(sigs, hashed, pks) == got
    for k in range(0, 48, 7):
        h = H.hash_to_g2(msgs[k], dst)
        assert B.bls_verify(sigs[k], h, pks[k]) == want[k]


def test_verify_msg_equals_verify_on_hashed_points_beyond_one_block(nmsm):
    rnd = random.Random(10)
    n = 300
    items = [BC.keypair_item(rnd) for _ in range(4)]
    msgs = [bytes([k & 0xFF]) * (k % 70) for k in range(n)]
    sigs = [items[k % 4][0] for k in range(n)]
    pks = [items[(k // 4) % 4][2] for k in range(n)]
    sig_m, pk_m = _signed(rnd, msgs[5], b"T")
    sigs[5], pks[5] = sig_m, pk_m
    got = nmsm.bls_verify_messages_batch(sigs, msgs, pks, b"T")
    assert got == nmsm.bls_verify_batch(sigs, nmsm.bls_hash_to_g2_batch(msgs, b"T"), pks)
    assert got[5] and sum(got) >= 1


def test_profiling_slots(nmsm):
    msgs = C.random_messages(64, seed=5)
    nmsm.set_profiling(True)
    try:
        _hash(nmsm, msgs, b"D")
        ms, _ = nmsm.last_timing()
        assert ms["prepare"] > 0 and ms["total"] == pytest.approx(ms["prepare"])
        rnd = random.Random(1)
        sig, pk = _signed(rnd, msgs[0], b"D")
        assert nmsm.bls_verify_messages_batch([sig], [msgs[0]], [pk], b"D") == [True]
        ms, _ = nmsm.last_timing()
        slots = [ms[k] for k in ("prepare", "count", "scan", "scatter")]
        assert all(v > 0 for v in slots) and ms["total"] == pytest.approx(sum(slots), rel=1e-4)
    finally:
        nmsm.set_profiling(False)
