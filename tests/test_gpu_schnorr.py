"""secp256k1 BIP340 Schnorr batch verification on the GPU (nmsm_secp256k1_schnorr_verify_batch): every verdict is
compared per item with the oracle (oracle.schnorr_ref.secp256k1_schnorr_verify, the reference's schnorr.verify) or with
the verdict known from how the batch was constructed."""
import random
import struct

import pytest

import ecdsa_cases as E
import schnorr_cases as S
from oracle import ecdsa_ref as ER
from oracle import schnorr_ref as SR

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _verify(nmsm, items):
    return nmsm.schnorr_verify_batch([i[0] for i in items], [i[1] for i in items], [i[2] for i in items])


def test_edge_set_matches_oracle(nmsm):
    cases = S.edge_cases()
    got = _verify(nmsm, [c[1:] for c in cases])
    want = [SR.secp256k1_schnorr_verify(*c[1:]) for c in cases]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    names = dict(zip((c[0] for c in cases), got))
    assert names["valid"] and names["msg-10000"] and not names["R=O"] and not names["odd-y"] and not names["sG=uP"]


def test_known_answer_rows_single_form_and_empty_batch(nmsm):
    for _, _, msg, pk, sig in S.KAT:
        assert nmsm.schnorr.verify(sig, msg, pk) is True
        assert nmsm.schnorr.verify(sig, msg[:-1] + bytes([msg[-1] ^ 1]), pk) is False
    assert _verify(nmsm, [(k[4], k[2], k[3]) for k in S.KAT]) == [True, True]
    assert nmsm.schnorr_verify_batch([], [], []) == []


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097])
def test_batches_with_scattered_invalid_items(nmsm, n):
    items, want = S.corrupt(S.signed_batch(n, seed=300 + n), seed=400 + n)
    got = _verify(nmsm, items)
    assert got == want, [k for k in range(n) if got[k] != want[k]][:10]
    for k in random.Random(n).sample(range(n), min(n, 12)):  # oracle sample
        assert got[k] == SR.secp256k1_schnorr_verify(*items[k]), k
    if n >= 32:  # valid and invalid items side by side within one warp
        assert any(0 < sum(got[w:w + 32]) < len(got[w:w + 32]) for w in range(0, n, 32))


def _ecdsa_round(nmsm):
    cases = E.edge_cases()
    got = nmsm.ecdsa_verify_batch([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
    assert got == [ER.secp256k1_ecdsa_verify(c[1], c[2], c[3]) for c in cases]
    assert any(got)


def _schnorr_round(nmsm):
    cases = S.edge_cases()
    got = _verify(nmsm, [c[1:] for c in cases])
    assert got == [SR.secp256k1_schnorr_verify(*c[1:]) for c in cases]
    assert any(got)


def test_ecdsa_and_schnorr_share_one_context(nmsm):
    _ecdsa_round(nmsm)
    _schnorr_round(nmsm)
    _ecdsa_round(nmsm)


def test_packed_offsets_are_validated(nmsm):
    sig, msg, pk = S.edge_cases()[0][1:]
    off = lambda *v: struct.pack("<%dQ" % len(v), *v)  # noqa: E731
    with pytest.raises(ValueError, match=r"msg_off\[0\] must be 0"):
        nmsm.schnorr_verify_batch_packed(sig, pk, msg, off(1, len(msg)), 1)
    with pytest.raises(ValueError, match=r"msg_off must be non-decreasing \(index 2\)"):
        nmsm.schnorr_verify_batch_packed(sig * 2, pk * 2, msg, off(0, len(msg), 0), 2)


def test_schnorr_builds_the_shared_table_after_reinit(nmsm):
    """Last in this module: after nmsm_shutdown + nmsm_init a Schnorr verify is the first to need the table of G, so it
    builds it; ECDSA then uses the same table."""
    lib = nmsm._lib.load()
    lib.nmsm_shutdown()
    nmsm._lib.check(lib.nmsm_init(0))
    _schnorr_round(nmsm)
    _ecdsa_round(nmsm)
