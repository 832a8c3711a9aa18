"""secp256k1 ECDSA public-key recovery and Ethereum ecrecover on the GPU (nmsm_secp256k1_recover_batch,
nmsm_secp256k1_ecrecover_batch): every key and address is compared per item with the oracle (oracle.recover_ref, the
reference's Signature.recoverPublicKey and the ECREC precompile) or with what is known from how the batch was built."""
import ctypes
import random
import struct

import pytest

import ecdsa_cases as E
import recover_cases as RC
import schnorr_cases as S
from oracle import ecdsa_ref as ER
from oracle import noble_ref as R
from oracle import recover_ref as RR
from oracle import schnorr_ref as SR

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _recover_packed(nmsm, sigs, msgs, prehash):
    s, m, off = RC.pack(sigs, msgs)
    return nmsm.ecdsa_recover_batch_packed(s, m, off, len(sigs), nmsm.ECDSA_PREHASH if prehash else 0)


def _compare_with_oracle(nmsm, cases):
    """cases: [(name, sig65, msg, prehash, ...)]; one batch per prehash mode, mismatches reported by name"""
    for prehash in (True, False):
        sub = [c for c in cases if c[3] == prehash]
        xy, ok = _recover_packed(nmsm, [c[1] for c in sub], [c[2] for c in sub], prehash)
        bad = []
        for k, c in enumerate(sub):
            want = RR.secp256k1_recover_public_key(c[1], c[2], prehash=prehash)
            if ok[k] != (want is not None) or xy[64 * k:64 * k + 64] != RC.xy_bytes(want):
                bad.append(c[0])
        assert not bad, (prehash, bad)


def test_edge_set_matches_oracle(nmsm):
    cases = RC.edge_cases()
    _compare_with_oracle(nmsm, cases)
    names = {c[0]: c for c in cases}
    for name in ("rec2-x=n+t", "rec3-x=n+t", "u1G=u2R", "high-s", "raw-8192", "h=0"):
        c = names[name]
        assert nmsm.ecdsa_recover_batch([c[1]], [c[2]], prehash=c[3])[0] is not None, name
    for name in ("Q=O", "raw-8193", "rec2-r+n>=p", "rec=27", "r-no-sqrt"):
        c = names[name]
        assert nmsm.ecdsa_recover_batch([c[1]], [c[2]], prehash=c[3]) == [None], name


def test_ecrecover_edge_set_matches_oracle(nmsm):
    cases = RC.ecrecover_cases()
    words, ok = nmsm.eth_ecrecover_batch_packed(b"".join(c[1] for c in cases), len(cases))
    got = [words[32 * k:32 * k + 32] if ok[k] else b"" for k in range(len(cases))]
    want = [RR.eth_ecrecover(c[1]) for c in cases]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    assert got == [c[2] for c in cases]
    assert all(words[32 * k:32 * k + 32] == bytes(32) for k in range(len(cases)) if not ok[k])


def test_ecrecover_helper_pads_and_truncates(nmsm):
    cases = {c[0]: c[1] for c in RC.ecrecover_cases()}
    good = cases["v=27"]
    inputs = [b"", good[:127], good, good + bytes(range(72)), cases["key-1"], cases["v=1d"]]
    got = nmsm.eth_ecrecover_batch(inputs)
    assert got == [RR.eth_ecrecover(i) for i in inputs]
    assert got[0] == b"" and got[2] == got[3] != b"" and got[4] == bytes(12) + RC.KEY1_ADDRESS


def test_key1_address_through_the_c_abi(nmsm):
    lib = nmsm._lib.load()
    data = dict((c[0], c[1]) for c in RC.ecrecover_cases())["key-1"]
    out, ok = ctypes.create_string_buffer(32), ctypes.create_string_buffer(1)
    nmsm._lib.check(lib.nmsm_secp256k1_ecrecover_batch(ctypes.cast(ctypes.c_char_p(data), ctypes.c_void_p), 1, out, ok))
    assert ok.raw == b"\x01" and out.raw == bytes(12) + RC.KEY1_ADDRESS


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097])
def test_batches_with_scattered_failures(nmsm, n):
    items, want_ok, keys = RC.corrupt(RC.signed_batch(n, seed=500 + n), seed=600 + n)
    xy, ok = _recover_packed(nmsm, [i[0] for i in items], [i[1] for i in items], True)
    assert [b == 1 for b in ok] == want_ok, [k for k in range(n) if (ok[k] == 1) != want_ok[k]][:10]
    for k in range(n):
        if keys[k] is not None:
            assert xy[64 * k:64 * k + 64] == RC.xy_bytes(keys[k]), k
        if not want_ok[k]:
            assert xy[64 * k:64 * k + 64] == bytes(64), k
    for k in random.Random(n).sample(range(n), min(n, 12)):  # oracle sample
        assert xy[64 * k:64 * k + 64] == RC.xy_bytes(RR.secp256k1_recover_public_key(*items[k])), k
    if n >= 32:  # recovered and failed items side by side within one warp
        assert any(0 < sum(ok[w:w + 32]) < len(ok[w:w + 32]) for w in range(0, n, 32))


def test_warp_with_q_at_infinity_and_bad_r_lanes(nmsm):
    """One warp of raw-message items: Q = O (fed 1 to the second inversion), an r whose x has no square root (fed 1 to
    the first), the doubling path, and valid neighbours."""
    rnd = random.Random(21)
    d = rnd.randrange(1, E.N)
    items = []
    for _ in range(64):
        h = rnd.randrange(E.N)
        items.append(("valid", RC.sign_rec(d, h, rnd), E.be32(h), False, RC.key_of(d)))
    special = {c[0]: c for c in RC.edge_cases() + RC.constructed_cases(seed=99)}
    items[3] = special["Q=O"]
    items[7] = special["r-no-sqrt"][:3] + (False, None)
    items[8] = special["u1G=u2R"]
    items[40] = special["rec3-x=n+t"]
    _compare_with_oracle(nmsm, items)
    xy, ok = _recover_packed(nmsm, [c[1] for c in items], [c[2] for c in items], False)
    assert ok[3] == 0 and ok[7] == 0 and ok[8] == 1 and sum(ok[:32]) == 30 and sum(ok) == 62


def test_recovered_keys_verify_their_signatures(nmsm):
    cases = [c for c in RC.edge_cases() if c[4] is not None]
    cases += [(str(k), s, m, True, key) for k, (s, m, key) in enumerate(RC.signed_batch(64, seed=41))]
    for prehash in (True, False):
        sub = [c for c in cases if c[3] == prehash]
        keys = nmsm.ecdsa_recover_batch([c[1] for c in sub], [c[2] for c in sub], prehash=prehash)
        assert all(k is not None for k in keys)
        got = nmsm.ecdsa_verify_batch([c[1][1:] for c in sub], [c[2] for c in sub], keys, prehash=prehash, lowS=False)
        assert all(got), [c[0] for c, g in zip(sub, got) if not g]


def test_openssl_batches(nmsm):
    pytest.importorskip("cryptography")
    for prehash, seed in ((True, 51), (False, 52)):
        items = E.openssl_sign(257, seed=seed, prehash=prehash)
        per_rec = []
        for rec in (0, 1):
            per_rec.append(nmsm.ecdsa_recover_batch([bytes([rec]) + s for s, _, _ in items], [m for _, m, _ in items],
                                                    prehash=prehash))
        for k, (_, _, pk) in enumerate(items):
            want = E.compressed(E.PT.fromAffine(dict(zip("xy", R.secp256k1_decode_sec1(pk)))))
            assert [per_rec[0][k], per_rec[1][k]].count(want) == 1, (prehash, k)


def test_single_form(nmsm):
    c = RC.edge_cases()[0]
    key = nmsm.secp256k1.recoverPublicKey(c[1], c[2], prehash=c[3])
    assert key == E.compressed(E.PT.fromAffine({"x": c[4][0], "y": c[4][1]}))
    with pytest.raises(ValueError, match="recovery failed"):
        nmsm.secp256k1.recoverPublicKey(bytes([4]) + c[1][1:], c[2], prehash=c[3])


def test_argument_errors_and_empty_batch(nmsm):
    c = RC.edge_cases()[0]
    sig, msg = c[1], c[2]
    off = lambda *v: struct.pack("<%dQ" % len(v), *v)  # noqa: E731
    with pytest.raises(ValueError, match=r"msg_off\[0\] must be 0"):
        nmsm.ecdsa_recover_batch_packed(sig, msg, off(1, len(msg)), 1, 0)
    with pytest.raises(ValueError, match=r"msg_off must be non-decreasing \(index 2\)"):
        nmsm.ecdsa_recover_batch_packed(sig * 2, msg, off(0, len(msg), 0), 2, 0)
    with pytest.raises(ValueError, match="unknown flag"):
        nmsm.ecdsa_recover_batch_packed(sig, msg, off(0, len(msg)), 1, 2)
    assert nmsm.ecdsa_recover_batch([], []) == []
    lib = nmsm._lib.load()
    xy, ok = ctypes.create_string_buffer(b"\xaa" * 64, 64), ctypes.create_string_buffer(b"\xaa", 1)
    z = ctypes.create_string_buffer(16)
    assert lib.nmsm_secp256k1_recover_batch(z, z, z, 0, 0, xy, ok) == 0
    assert lib.nmsm_secp256k1_ecrecover_batch(z, 0, xy, ok) == 0
    assert xy.raw == b"\xaa" * 64 and ok.raw == b"\xaa"


def test_n_bound_is_checked_before_the_offsets_are_read(nmsm):
    """n >= 2^31 with one-element buffers: every secp256k1 batch entry point returns the argument error instead of
    reading offs[n]."""
    lib = nmsm._lib.load()
    buf = ctypes.create_string_buffer(256)
    off = ctypes.create_string_buffer(16)
    big = 1 << 31
    calls = {
        "verify": lambda: lib.nmsm_secp256k1_verify_batch(buf, buf, off, buf, off, big, 1, buf),
        "schnorr": lambda: lib.nmsm_secp256k1_schnorr_verify_batch(buf, buf, buf, off, big, buf),
        "recover": lambda: lib.nmsm_secp256k1_recover_batch(buf, buf, off, big, 1, buf, buf),
        "ecrecover": lambda: lib.nmsm_secp256k1_ecrecover_batch(buf, big, buf, buf),
    }
    for name, call in calls.items():
        assert call() == nmsm._lib.ERR_ARG, name
        assert lib.nmsm_last_error().decode() == "n must be < 2^31", name


def test_profiling_slots(nmsm):
    c = RC.edge_cases()[0]
    nmsm.set_profiling(True)
    try:
        nmsm.ecdsa_recover_batch([c[1]] * 300, [c[2]] * 300, prehash=c[3])
        ms = list(nmsm.last_timing()[0].values())
    finally:
        nmsm.set_profiling(False)
    assert ms[0] > 0 and ms[1] > 0 and ms[-1] >= max(ms[0], ms[1])
    assert ms[-1] == pytest.approx(ms[0] + ms[1], abs=0.01)  # three events, each with ~0.5 us resolution


def _recover_round(nmsm):
    _compare_with_oracle(nmsm, RC.edge_cases())


def _ecdsa_round(nmsm):
    cases = E.edge_cases()
    got = nmsm.ecdsa_verify_batch([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
    assert got == [ER.secp256k1_ecdsa_verify(c[1], c[2], c[3]) for c in cases] and any(got)


def _schnorr_round(nmsm):
    cases = S.edge_cases()
    got = nmsm.schnorr_verify_batch([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
    assert got == [SR.secp256k1_schnorr_verify(*c[1:]) for c in cases] and any(got)


def test_recover_ecdsa_and_schnorr_share_one_context(nmsm):
    _recover_round(nmsm)
    _ecdsa_round(nmsm)
    _recover_round(nmsm)
    _schnorr_round(nmsm)
    _recover_round(nmsm)


def test_recover_builds_the_shared_table_after_reinit(nmsm):
    """Last in this module: after nmsm_shutdown + nmsm_init a recovery is the first to need the table of G, so it
    builds it; ECDSA then verifies with the same table."""
    lib = nmsm._lib.load()
    lib.nmsm_shutdown()
    nmsm._lib.check(lib.nmsm_init(0))
    _recover_round(nmsm)
    _ecdsa_round(nmsm)
