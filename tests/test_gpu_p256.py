"""P-256 ECDSA batch verification on the GPU (nmsm_p256_verify_batch): every verdict is compared per item with the
oracle (oracle.p256_ref.p256_ecdsa_verify, noble's p256.verify), with OpenSSL for OpenSSL-signed batches, and with the
EIP-7951 statement for P256VERIFY inputs."""
import random
import struct

import pytest

import ecdsa_cases as E
import p256_cases as C
from oracle import ecdsa_ref as ER
from oracle import p256_ref as PR

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _verify(nmsm, items, **kw):
    return nmsm.p256_ecdsa_verify_batch([i[0] for i in items], [i[1] for i in items], [i[2] for i in items], **kw)


@pytest.mark.parametrize("prehash,lowS", C.FLAGS)
def test_edge_set_matches_oracle(nmsm, prehash, lowS):
    cases = C.edge_cases()
    got = _verify(nmsm, [c[1:] for c in cases], prehash=prehash, lowS=lowS)
    want = [PR.p256_ecdsa_verify(c[1], c[2], c[3], prehash=prehash, lowS=lowS) for c in cases]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    names = dict(zip((c[0] for c in cases), got))
    if not prehash:
        assert names["Rx>=n"] and names["u1G=u2Q"] and not names["R=O"] and not names["Rx>=n-r=x"]
    else:
        assert names["valid"] and names["valid-negated-s"] == (not lowS)


def test_single_verify_defaults_and_empty_batch(nmsm):
    sig, msg, pk = C.edge_cases()[0][1:]
    assert nmsm.p256.verify(sig, msg, pk) is True
    assert nmsm.secp256r1.verify(sig, msg + b"!", pk) is False
    r, s = sig[:32], int.from_bytes(sig[32:], "big")
    high = r + C.be32(C.N - s)
    assert nmsm.p256.verify(high, msg, pk) is True  # noble's p256 default: lowS false
    assert nmsm.p256.verify(high, msg, pk, lowS=True) is False
    assert nmsm.p256_ecdsa_verify_batch([], [], []) == []


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097])
def test_batches_with_scattered_invalid_items(nmsm, n):
    pytest.importorskip("cryptography")
    items = C.corrupt(C.openssl_sign(n, seed=100 + n), seed=200 + n)
    for lowS in (False, True):
        got = _verify(nmsm, items, lowS=lowS)
        want = [C.openssl_verify(*i, prehash=True, lowS=lowS) for i in items]
        assert got == want, [k for k in range(n) if got[k] != want[k]][:10]
        if n > 1:
            assert 0 < sum(got) < n  # valid and invalid items side by side
        for k in random.Random(n).sample(range(n), min(n, 12)):  # oracle sample
            assert got[k] == PR.p256_ecdsa_verify(*items[k], prehash=True, lowS=lowS), k


def test_raw_digest_batch(nmsm):
    pytest.importorskip("cryptography")
    items = C.corrupt(C.openssl_sign(257, seed=7, prehash=False), seed=8)
    got = _verify(nmsm, items, prehash=False)
    assert got == [C.openssl_verify(*i, prehash=False) for i in items]
    assert 0 < sum(got) < len(items)


def test_precompile_batch_matches_eip7951_oracle(nmsm):
    cases = C.precompile_cases()
    want = [PR.p256verify_precompile(i) for _, i in cases]
    got = nmsm.p256verify_precompile_batch([i for _, i in cases])
    assert got == want, [n for (n, _), g, w in zip(cases, got, want) if g != w]
    assert any(want) and not all(want)
    packed = [i for _, i in cases if len(i) == 160]
    assert nmsm.p256verify_precompile_batch(b"".join(packed)) == [PR.p256verify_precompile(i) for i in packed]


def test_precompile_batch_from_openssl(nmsm):
    pytest.importorskip("cryptography")
    items = C.corrupt(C.openssl_sign(300, seed=41, prehash=False, compressed_ratio=0.0), seed=42)
    inputs = [m + s + pk[1:] for s, m, pk in items]  # hash || r || s || qx || qy (a corrupted 05 prefix is dropped)
    got = nmsm.p256verify_precompile_batch(inputs)
    assert got == [PR.p256verify_precompile(i) for i in inputs]
    assert 0 < sum(got) < len(inputs)


def test_packed_offsets_are_validated(nmsm):
    sig, msg, pk = C.edge_cases()[0][1:]
    off = lambda *v: struct.pack("<%dQ" % len(v), *v)  # noqa: E731
    with pytest.raises(ValueError, match="pk_off"):
        nmsm.p256_ecdsa_verify_batch_packed(sig, pk, off(1, 33), msg, off(0, len(msg)), 1)
    with pytest.raises(ValueError, match="msg_off"):
        nmsm.p256_ecdsa_verify_batch_packed(sig * 2, pk * 2, off(0, 33, 66), msg, off(0, len(msg), 0), 2)
    with pytest.raises(ValueError, match="unknown flag"):
        nmsm.p256_ecdsa_verify_batch_packed(sig, pk, off(0, 33), msg, off(0, len(msg)), 1, flags=4)


def test_profiling_slots(nmsm):
    items = [c[1:] for c in C.edge_cases()] * 40
    nmsm.set_profiling(True)
    try:
        _verify(nmsm, items)
        t, _ = nmsm.last_timing()
    finally:
        nmsm.set_profiling(False)
    assert t["prepare"] > 0 and t["count"] > 0 and t["total"] >= max(t["prepare"], t["count"])


def test_interleaved_with_secp256k1(nmsm):
    """secp256k1 and P-256 verifies alternate in one process with both G tables live: the secp256k1 verdicts do not
    change, and neither do P-256's."""
    k1 = E.edge_cases()
    r1 = C.edge_cases()
    k1_args = ([c[1] for c in k1], [c[2] for c in k1], [c[3] for c in k1])
    want_k1 = [ER.secp256k1_ecdsa_verify(c[1], c[2], c[3]) for c in k1]
    want_r1 = [PR.p256_ecdsa_verify(c[1], c[2], c[3]) for c in r1]
    for _ in range(3):
        assert nmsm.ecdsa_verify_batch(*k1_args) == want_k1
        assert _verify(nmsm, [c[1:] for c in r1]) == want_r1
    # a P-256 key handed to the secp256k1 entry point gets the secp256k1 verdict (it decodes there or not at all)
    sig, msg, pk = r1[0][1:]
    assert nmsm.ecdsa_verify_batch([sig], [msg], [pk], lowS=False) == [ER.secp256k1_ecdsa_verify(sig, msg, pk, lowS=False)]


def test_g_table_is_rebuilt_after_reinit(nmsm):
    """Last in this module: nmsm_shutdown frees the G table, the next nmsm_init + verify builds it again."""
    items = [c[1:] for c in C.edge_cases()]
    before = _verify(nmsm, items)
    lib = nmsm._lib.load()
    lib.nmsm_shutdown()
    nmsm._lib.check(lib.nmsm_init(0))
    after = _verify(nmsm, items)
    assert after == before and any(after)
