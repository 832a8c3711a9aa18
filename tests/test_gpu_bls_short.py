"""Hash to BLS12-381 G1 and short-signature verification on the GPU (nmsm_bls12_381_hash_to_g1_batch,
nmsm_bls12_381_short_verify_batch, nmsm_bls12_381_short_verify_msg_batch): points compared byte for byte with the
oracle (oracle.hash_to_g1_ref), verdicts with the oracle's verification, and the two verify entry points with each
other."""
import ctypes
import random

import pytest

import bls_cases as BC
import h2g1_cases as C
from oracle import hash_to_g1_ref as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _hash(nmsm, msgs, dst):
    data, off = C.pack_messages(msgs)
    xy = nmsm.bls_hash_to_g1_batch_packed(data, off, len(msgs), dst)
    return [xy[96 * k:96 * k + 96] for k in range(len(msgs))]


def _short_packed(nmsm, triples, dst=H.DST_G1_NUL):
    sigs, msgs, pks = zip(*triples)
    data, off = C.pack_messages(msgs)
    return nmsm.bls_short_verify_messages_batch_packed(b"".join(sigs), b"".join(pks), data, off, len(triples), dst)


def test_known_answers_through_the_c_abi(nmsm):
    assert _hash(nmsm, list(C.KATS), H.DST_QUUX) == [C.kat_packed(v) for v in C.KATS.values()]
    pt = nmsm.bls12_381.G1.hashToCurve(b"abc", {"DST": H.DST_QUUX})
    assert pt.to_packed() == C.kat_packed(C.KATS[b"abc"]) and pt._valid


def test_4096_messages_match_oracle_and_are_torsion_free(nmsm):
    msgs = C.random_messages(4096, seed=7)
    got = _hash(nmsm, msgs, H.DST_G1_NUL)
    want = C.oracle_packed(msgs, H.DST_G1_NUL)
    bad = [k for k in range(len(msgs)) if got[k] != want[k]]
    assert not bad, [(k, len(msgs[k])) for k in bad[:10]]
    ok = nmsm.torsion_free_packed(6, b"".join(got), len(got))  # NMSM_BLS12_381_G1_ANY
    assert ok == b"\1" * len(got)


@pytest.mark.parametrize("dlen", [1, 43, 255, 256, 300])
def test_dst_lengths(nmsm, dlen):
    dst = H.DST_G1_POP if dlen == 43 else bytes((7 * k + 1) & 0xFF for k in range(dlen))
    msgs = C.random_messages(len(C.EDGE_LENGTHS), seed=dlen)
    assert _hash(nmsm, msgs, dst) == C.oracle_packed(msgs, dst, workers=1)


def test_mirror_returns_g1_points(nmsm):
    pts = nmsm.bls_hash_to_g1_batch([b"", b"x" * 100], H.DST_G1_POP)
    assert [p.to_packed() for p in pts] == C.oracle_packed([b"", b"x" * 100], H.DST_G1_POP, workers=1)
    assert nmsm.bls12_381.G1.hashToCurve(b"m").to_packed() == H.g1_packed(H.hash_to_g1(b"m", H.DST_G1_NUL))


def test_n_zero_and_not_a_multiple_of_32(nmsm):
    assert nmsm.bls_hash_to_g1_batch([]) == []
    for n in (1, 33, 300):  # partial warps and a partial last block of 128 threads
        msgs = [bytes([k & 0xFF, k >> 8, n & 0xFF]) for k in range(n)]
        got = _hash(nmsm, msgs, b"T")
        sample = sorted(set(list(range(0, n, 37)) + [n - 1, n // 2]))
        assert [got[k] for k in sample] == C.oracle_packed([msgs[k] for k in sample], b"T", workers=1), n


def test_edge_set_against_oracle(nmsm):
    cases = C.edge_cases()
    names = [c[0] for c in cases]
    sigs, msgs, pks = [c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases]
    hs = [H.hash_to_g1(m, H.DST_G1_NUL) for m in msgs]
    want = [H.short_verify(s, h, k) for s, h, k in zip(sigs, hs, pks)]
    assert sum(want) == 3
    got = nmsm.bls_short_verify_messages_batch(sigs, msgs, pks)
    assert got == want, [(nm, g, w) for nm, g, w in zip(names, got, want) if g != w]
    pts = nmsm.bls_hash_to_g1_batch(msgs)
    assert nmsm.bls_short_verify_batch(sigs, pts, pks) == want
    assert [nmsm.bls12_381.verifyShortSignature(s, m, k) for s, m, k in zip(sigs[:4], msgs[:4], pks[:4])] == want[:4]


def test_mirror_accepts_points(nmsm):
    rnd = random.Random(4)
    sk = rnd.randrange(1, H.N)
    msg = b"point arguments"
    h = H.hash_to_g1(msg, H.DST_G1_NUL)
    sig_pt = nmsm.bls12_381.G1.Point.fromAffine({"x": H.scalar_mul(sk, h)[0], "y": H.scalar_mul(sk, h)[1]})
    pk_pt = nmsm.bls12_381.G2.Point.BASE.multiply(sk)
    assert nmsm.bls12_381.verifyShortSignature(sig_pt, msg, pk_pt)
    assert nmsm.bls12_381.verifyShortSignature(sig_pt, nmsm.bls12_381.G1.hashToCurve(msg), pk_pt)
    assert not nmsm.bls12_381.verifyShortSignature(sig_pt.negate(), msg, pk_pt)


def test_large_batch_with_scattered_corruptions(nmsm):
    """2^16 + 3 signatures tiled from 256 oracle-signed triples, with corruptions at scattered indices"""
    base = C.signed_triples(256, seed=12)
    n = (1 << 16) + 3
    triples = [base[k % len(base)] for k in range(n)]
    rnd = random.Random(13)
    want = [True] * n
    for k in sorted(set(rnd.sample(range(n), 400)) | {0, n - 1}):
        sig, msg, pk = triples[k]
        kind = k % 4
        if kind == 0:
            triples[k] = (sig, msg + b"!", pk)  # wrong message
        elif kind == 1:
            triples[k] = (bytes([sig[0] ^ 0x20]) + sig[1:], msg, pk)  # negated signature
        elif kind == 2:
            triples[k] = (sig, msg, base[(k + 1) % len(base)][2] if base[(k + 1) % len(base)][2] != pk
                          else base[(k + 2) % len(base)][2])  # another key
        else:
            triples[k] = (bytes([0xC0]) + bytes(47), msg, pk)  # identity signature
        want[k] = False
    got = _short_packed(nmsm, triples)
    assert got == bytes(want), [k for k in range(n) if got[k] != want[k]][:10]


def test_short_verify_msg_equals_short_verify_on_hashed_points(nmsm):
    triples = C.signed_triples(64, seed=14)
    triples[5] = (triples[5][0], triples[5][1] + b"?", triples[5][2])
    sigs, msgs, pks = zip(*triples)
    data, off = C.pack_messages(msgs)
    pts = nmsm.bls_hash_to_g1_batch_packed(data, off, len(msgs), H.DST_G1_NUL)
    by_pts = nmsm.bls_short_verify_batch_packed(b"".join(sigs), b"".join(pks), pts, len(msgs))
    assert _short_packed(nmsm, triples) == by_pts
    assert by_pts == bytes(k != 5 for k in range(64))


def test_interleaved_with_long_signatures(nmsm):
    rnd = random.Random(15)
    long_items = [BC.keypair_item(rnd) for _ in range(3)]
    short = C.signed_triples(40, seed=16)
    for _ in range(2):
        assert nmsm.bls_verify_batch([i[0] for i in long_items],
                                     [nmsm.bls12_381.G2.Point.fromAffine({"x": i[1][0], "y": i[1][1]})
                                      for i in long_items],
                                     [i[2] for i in long_items]) == [True] * 3
        assert _short_packed(nmsm, short) == b"\1" * 40
        msgs = [b"a", b"bc"]
        assert [p.to_packed() for p in nmsm.bls_hash_to_g2_batch(msgs)] != []
        assert _hash(nmsm, msgs, H.DST_G1_NUL) == C.oracle_packed(msgs, H.DST_G1_NUL, workers=1)


def test_error_codes(nmsm):
    lib = nmsm._lib.load()
    out = ctypes.create_string_buffer(96)
    off = (ctypes.c_uint64 * 2)(0, 1)
    m = ctypes.c_char_p(b"m")
    d = ctypes.c_char_p(b"D")
    ERR_ARG, ERR_POINT = nmsm._lib.ERR_ARG, nmsm._lib.ERR_POINT
    h2g1 = lib.nmsm_bls12_381_hash_to_g1_batch
    assert h2g1(m, off, 1, d, 0, out) == ERR_ARG  # empty DST
    assert h2g1(m, off, 1, None, 1, out) == ERR_ARG
    assert h2g1(m, None, 1, d, 1, out) == ERR_ARG
    assert h2g1(None, off, 1, d, 1, out) == ERR_ARG
    assert h2g1(m, off, 1, d, 1, None) == ERR_ARG
    assert h2g1(m, off, 1 << 30, d, 1, out) == ERR_ARG
    bad0 = (ctypes.c_uint64 * 2)(1, 1)
    assert h2g1(m, bad0, 1, d, 1, out) == ERR_ARG
    dec = (ctypes.c_uint64 * 3)(0, 1, 0)
    assert h2g1(m, dec, 2, d, 1, out) == ERR_ARG
    assert b"non-decreasing" in lib.nmsm_last_error()
    assert h2g1(None, None, 0, d, 1, None) == 0  # n = 0 writes nothing
    sig, pk, ok = ctypes.c_char_p(bytes(48)), ctypes.c_char_p(bytes(96)), ctypes.create_string_buffer(2)
    sv = lib.nmsm_bls12_381_short_verify_batch
    pts = ctypes.c_char_p(bytes(96))
    assert sv(None, pk, pts, 1, ok) == ERR_ARG
    assert sv(sig, None, pts, 1, ok) == ERR_ARG
    assert sv(sig, pk, None, 1, ok) == ERR_ARG
    assert sv(sig, pk, pts, 1, None) == ERR_ARG
    assert sv(sig, pk, pts, 1 << 30, ok) == ERR_ARG
    assert sv(None, None, None, 0, None) == 0
    svm = lib.nmsm_bls12_381_short_verify_msg_batch
    assert svm(sig, pk, m, off, 1, d, 0, ok) == ERR_ARG
    assert svm(sig, pk, m, off, 1, None, 1, ok) == ERR_ARG
    assert svm(None, pk, m, off, 1, d, 1, ok) == ERR_ARG
    assert svm(sig, None, m, off, 1, d, 1, ok) == ERR_ARG
    assert svm(sig, pk, None, off, 1, d, 1, ok) == ERR_ARG
    assert svm(sig, pk, m, None, 1, d, 1, ok) == ERR_ARG
    assert svm(sig, pk, m, off, 1, d, 1, None) == ERR_ARG
    assert svm(sig, pk, m, bad0, 1, d, 1, ok) == ERR_ARG
    assert svm(sig, pk, m, off, 1 << 30, d, 1, ok) == ERR_ARG
    assert svm(None, None, None, None, 0, d, 1, None) == 0
    # NMSM_ERR_POINT names the smallest message point that is out of range or off the curve
    (s0, m0, k0), = C.signed_triples(1, seed=17)
    h = H.hash_to_g1(m0, H.DST_G1_NUL)
    hs = [h, None, (h[0], (h[1] + 1) % H.P), (H.P, 2), (h[0], (h[1] + 1) % H.P)]
    with pytest.raises(nmsm.NmsmError) as e:
        nmsm.bls_short_verify_batch_packed(s0 * 5, k0 * 5, b"".join(H.g1_packed(x) for x in hs), 5)
    assert e.value.code == ERR_POINT and e.value.index == 2
    assert nmsm.bls_short_verify_batch_packed(s0 * 2, k0 * 2, H.g1_packed(h) + bytes(96), 2) == b"\1\0"
    with pytest.raises(nmsm.NmsmError):
        nmsm.bls_hash_to_g1_batch_packed(b"m", bytes(16), 1, b"")


def test_profiling_slots(nmsm):
    triples = C.signed_triples(64, seed=18)
    msgs = [t[1] for t in triples]
    nmsm.set_profiling(True)
    try:
        _hash(nmsm, msgs, H.DST_G1_NUL)
        ms, _ = nmsm.last_timing()
        assert ms["prepare"] > 0 and ms["total"] == pytest.approx(ms["prepare"])
        assert _short_packed(nmsm, triples) == b"\1" * 64
        ms, _ = nmsm.last_timing()
        slots = [ms[k] for k in ("prepare", "count", "scan", "scatter")]
        assert all(v > 0 for v in slots) and ms["total"] == pytest.approx(sum(slots), rel=1e-4)
        sigs, _, pks = zip(*triples)
        data, off = C.pack_messages(msgs)
        pts = nmsm.bls_hash_to_g1_batch_packed(data, off, len(msgs), H.DST_G1_NUL)
        assert nmsm.bls_short_verify_batch_packed(b"".join(sigs), b"".join(pks), pts, 64) == b"\1" * 64
        ms, _ = nmsm.last_timing()
        slots = [ms[k] for k in ("prepare", "count", "scan")]
        assert all(v > 0 for v in slots) and ms["scatter"] == 0
        assert ms["total"] == pytest.approx(sum(slots), rel=1e-4)
    finally:
        nmsm.set_profiling(False)
