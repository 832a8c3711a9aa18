"""P-384 ECDSA batch verification on the GPU (nmsm_p384_verify_batch): every verdict is compared per item with the
oracle (oracle.p384_ref.p384_ecdsa_verify, noble's p384.verify) and with OpenSSL for OpenSSL-signed batches."""
import random
import struct

import pytest

import ecdsa_cases as E
import p256_cases as C256
import p384_cases as C
from oracle import ecdsa_ref as ER
from oracle import p256_ref as PR256
from oracle import p384_ref as PR

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _verify(nmsm, items, **kw):
    return nmsm.p384_ecdsa_verify_batch([i[0] for i in items], [i[1] for i in items], [i[2] for i in items], **kw)


@pytest.mark.parametrize("prehash,lowS", C.FLAGS)
def test_edge_set_matches_oracle(nmsm, prehash, lowS):
    cases = C.edge_cases()
    got = _verify(nmsm, [c[1:] for c in cases], prehash=prehash, lowS=lowS)
    want = [PR.p384_ecdsa_verify(c[1], c[2], c[3], prehash=prehash, lowS=lowS) for c in cases]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    names = dict(zip((c[0] for c in cases), got))
    if not prehash:
        assert names["Rx>=n"] and names["u1G=u2Q"] and not names["R=O"] and not names["Rx>=n-r=x"]
    else:
        assert names["valid"] and names["valid-97"] and names["valid-negated-s"] == (not lowS)


def test_single_verify_defaults_and_empty_batch(nmsm):
    sig, msg, pk = C.edge_cases()[0][1:]
    assert nmsm.p384.verify(sig, msg, pk) is True
    assert nmsm.secp384r1.verify(sig, msg + b"!", pk) is False
    r, s = sig[:48], int.from_bytes(sig[48:], "big")
    high = r + C.be48(C.N - s)
    assert nmsm.p384.verify(high, msg, pk) is True  # noble's p384 default: lowS false
    assert nmsm.p384.verify(high, msg, pk, lowS=True) is False
    assert nmsm.p384_ecdsa_verify_batch([], [], []) == []


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097, 2**16 + 3])
def test_batches_with_scattered_invalid_items(nmsm, n):
    """OpenSSL-signed batches, compressed and uncompressed keys mixed, about one item in four corrupted.  The largest
    batch tiles 4099 unique signatures (OpenSSL signing in Python is the slow part), so tiles land in other warps."""
    pytest.importorskip("cryptography")
    uniq = C.corrupt(C.openssl_sign(min(n, 4099), seed=100 + n), seed=200 + n)
    want_u = {lowS: [C.openssl_verify(*i, prehash=True, lowS=lowS) for i in uniq] for lowS in (False, True)}
    items = (uniq * (n // len(uniq) + 1))[:n]
    for lowS in (False, True):
        got = _verify(nmsm, items, lowS=lowS)
        want = (want_u[lowS] * (n // len(uniq) + 1))[:n]
        assert got == want, [k for k in range(n) if got[k] != want[k]][:10]
        if n > 1:
            assert 0 < sum(got) < n  # valid and invalid items side by side
        for k in random.Random(n).sample(range(len(uniq)), min(len(uniq), 8)):  # oracle sample
            assert got[k] == PR.p384_ecdsa_verify(*items[k], prehash=True, lowS=lowS), k


def test_raw_digest_batch(nmsm):
    """prehash off: the caller passes its own 48-byte SHA-384 digests."""
    pytest.importorskip("cryptography")
    items = C.corrupt(C.openssl_sign(257, seed=7, prehash=False), seed=8)
    got = _verify(nmsm, items, prehash=False)
    assert got == [C.openssl_verify(*i, prehash=False) for i in items]
    assert 0 < sum(got) < len(items)


def test_packed_offsets_are_validated(nmsm):
    sig, msg, pk = C.edge_cases()[0][1:]
    off = lambda *v: struct.pack("<%dQ" % len(v), *v)  # noqa: E731
    with pytest.raises(ValueError, match="pk_off"):
        nmsm.p384_ecdsa_verify_batch_packed(sig, pk, off(1, 49), msg, off(0, len(msg)), 1)
    with pytest.raises(ValueError, match="msg_off"):
        nmsm.p384_ecdsa_verify_batch_packed(sig * 2, pk * 2, off(0, 49, 98), msg, off(0, len(msg), 0), 2)
    with pytest.raises(ValueError, match="unknown flag"):
        nmsm.p384_ecdsa_verify_batch_packed(sig, pk, off(0, 49), msg, off(0, len(msg)), 1, flags=4)
    # a valid packed call after the rejected ones
    assert nmsm.p384_ecdsa_verify_batch_packed(sig, pk, off(0, 49), msg, off(0, len(msg)), 1) == b"\x01"


def test_profiling_slots(nmsm):
    items = [c[1:] for c in C.edge_cases()] * 40
    nmsm.set_profiling(True)
    try:
        _verify(nmsm, items)
        t, _ = nmsm.last_timing()
    finally:
        nmsm.set_profiling(False)
    assert t["prepare"] > 0 and t["count"] > 0 and t["total"] >= max(t["prepare"], t["count"])


def test_interleaved_with_p256_and_secp256k1(nmsm):
    """secp256k1, P-256 and P-384 verifies alternate in one process with all three G tables resident: no verdict
    changes."""
    k1, r1, r3 = E.edge_cases(), C256.edge_cases(), C.edge_cases()
    want_k1 = [ER.secp256k1_ecdsa_verify(c[1], c[2], c[3]) for c in k1]
    want_r1 = [PR256.p256_ecdsa_verify(c[1], c[2], c[3]) for c in r1]
    want_r3 = [PR.p384_ecdsa_verify(c[1], c[2], c[3]) for c in r3]
    for _ in range(3):
        assert nmsm.ecdsa_verify_batch([c[1] for c in k1], [c[2] for c in k1], [c[3] for c in k1]) == want_k1
        assert _verify(nmsm, [c[1:] for c in r3]) == want_r3
        assert nmsm.p256_ecdsa_verify_batch([c[1] for c in r1], [c[2] for c in r1], [c[3] for c in r1]) == want_r1


def test_g_table_is_rebuilt_after_reinit(nmsm):
    """Last in this module: nmsm_shutdown frees the G table, the next nmsm_init + verify builds it again."""
    items = [c[1:] for c in C.edge_cases()]
    before = _verify(nmsm, items)
    lib = nmsm._lib.load()
    lib.nmsm_shutdown()
    nmsm._lib.check(lib.nmsm_init(0))
    after = _verify(nmsm, items)
    assert after == before and any(after)
