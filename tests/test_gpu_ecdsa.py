"""secp256k1 ECDSA batch verification on the GPU (nmsm_secp256k1_verify_batch): every verdict is compared per item with
the oracle (oracle.ecdsa_ref.secp256k1_ecdsa_verify, the reference's ecdsa().verify), and for OpenSSL-signed batches
with OpenSSL's verdict plus the lowS rule."""
import random

import pytest

import ecdsa_cases as E
from oracle import ecdsa_ref as ER
from oracle import noble_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


@pytest.mark.parametrize("prehash,lowS", E.FLAGS)
def test_edge_set_matches_oracle(nmsm, prehash, lowS):
    cases = E.edge_cases()
    got = nmsm.ecdsa_verify_batch([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases],
                                  prehash=prehash, lowS=lowS)
    want = [ER.secp256k1_ecdsa_verify(c[1], c[2], c[3], prehash=prehash, lowS=lowS) for c in cases]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    if not prehash:
        names = dict(zip((c[0] for c in cases), got))
        assert names["Rx>=n"] and names["u1G=u2Q"] and not names["R=O"]


def test_single_verify_and_empty_batch(nmsm):
    sig, msg, pk = E.edge_cases()[0][1:]
    assert nmsm.secp256k1.verify(sig, msg, pk) is True
    assert nmsm.secp256k1.verify(sig, msg + b"!", pk) is False
    assert nmsm.ecdsa_verify_batch([], [], []) == []


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097])
def test_batches_with_scattered_invalid_items(nmsm, n):
    pytest.importorskip("cryptography")
    items = E.corrupt(E.openssl_sign(n, seed=100 + n), seed=200 + n)
    for lowS in (True, False):
        got = nmsm.ecdsa_verify_batch([i[0] for i in items], [i[1] for i in items], [i[2] for i in items], lowS=lowS)
        want = [E.openssl_verify(*i, prehash=True, lowS=lowS) for i in items]
        assert got == want, [k for k in range(n) if got[k] != want[k]][:10]
        if n > 1:
            assert 0 < sum(got) < n  # valid and invalid items side by side
        for k in random.Random(n).sample(range(n), min(n, 12)):  # oracle sample
            assert got[k] == ER.secp256k1_ecdsa_verify(*items[k], prehash=True, lowS=lowS), k


def test_raw_digest_batch(nmsm):
    pytest.importorskip("cryptography")
    items = E.corrupt(E.openssl_sign(257, seed=7, prehash=False), seed=8)
    got = nmsm.ecdsa_verify_batch([i[0] for i in items], [i[1] for i in items], [i[2] for i in items], prehash=False,
                                  lowS=False)
    assert got == [E.openssl_verify(*i, prehash=False, lowS=False) for i in items]


def test_packed_offsets_are_validated(nmsm):
    import struct

    sig, msg, pk = E.edge_cases()[0][1:]
    off = lambda *v: struct.pack("<%dQ" % len(v), *v)  # noqa: E731
    with pytest.raises(ValueError, match="pk_off"):
        nmsm.ecdsa_verify_batch_packed(sig, pk, off(1, 33), msg, off(0, len(msg)), 1)
    with pytest.raises(ValueError, match="msg_off"):
        nmsm.ecdsa_verify_batch_packed(sig * 2, pk * 2, off(0, 33, 66), msg, off(0, len(msg), 0), 2)
    with pytest.raises(ValueError, match="unknown flag"):
        nmsm.ecdsa_verify_batch_packed(sig, pk, off(0, 33), msg, off(0, len(msg)), 1, flags=4)


def test_g_table_is_rebuilt_after_reinit(nmsm):
    """Last in this module: nmsm_shutdown frees the G table, the next nmsm_init + verify builds it again."""
    cases = E.edge_cases()
    before = nmsm.ecdsa_verify_batch([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
    lib = nmsm._lib.load()
    lib.nmsm_shutdown()
    nmsm._lib.check(lib.nmsm_init(0))
    after = nmsm.ecdsa_verify_batch([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
    assert after == before and any(after)
