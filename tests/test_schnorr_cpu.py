"""secp256k1 BIP340 Schnorr verification without a GPU: the oracle against BIP340's known-answer rows, the device
bodies (the challenge hash, the prepare + check bodies) run on the host through tests/hostemu, and the host mirror's
argument checks."""
import hashlib
import random

import pytest

import nmsm
import schnorr_cases as S
from oracle import schnorr_ref as SR


def _flips(b: bytes):
    for k in range(len(b)):
        yield b[:k] + bytes([b[k] ^ 0x01]) + b[k + 1:]


def test_oracle_reproduces_known_answer_rows():
    for sk, aux, msg, pk, sig in S.KAT:
        assert SR.public_key(sk) == pk
        assert SR.schnorr_sign(sk, msg, aux) == sig
        assert SR.secp256k1_schnorr_verify(sig, msg, pk) is True


def test_oracle_rejects_every_single_byte_flip_of_known_answer_rows():
    for _, _, msg, pk, sig in S.KAT:
        for bad in _flips(sig):
            assert SR.secp256k1_schnorr_verify(bad, msg, pk) is False
        for bad in _flips(msg):
            assert SR.secp256k1_schnorr_verify(sig, bad, pk) is False
        for bad in _flips(pk):
            assert SR.secp256k1_schnorr_verify(sig, msg, bad) is False


def test_device_challenge_hash_matches_hashlib():
    """Lengths 0..200 and 1000 past the 128-byte prefix T || T || r || pk: the padding boundaries at 55, 56, 63, 64."""
    rnd = random.Random(9)
    tag = hashlib.sha256(b"BIP0340/challenge").digest()
    r32, pk32 = bytes(rnd.randrange(256) for _ in range(32)), bytes(rnd.randrange(256) for _ in range(32))
    for ln in list(range(201)) + [1000]:
        m = bytes(rnd.randrange(256) for _ in range(ln))
        assert S.emu_challenge(r32, pk32, m) == hashlib.sha256(tag + tag + r32 + pk32 + m).digest(), ln


def test_host_bodies_match_oracle_on_edge_set():
    cases = S.edge_cases()
    got = S.emu_verify([c[1:] for c in cases])
    want = [SR.secp256k1_schnorr_verify(*c[1:]) for c in cases]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    names = dict(zip((c[0] for c in cases), want))
    assert names["valid"] and names["kat-0"] and names["kat-1"]
    assert all(names["msg-%d" % ln] for ln in (0, 32, 55, 56, 119, 120, 10000))
    assert not any(v for k, v in names.items() if k.startswith(("key-", "r=", "s=")))
    assert not names["R=O"] and not names["odd-y"] and not names["sG=uP"]


def test_constructed_cases_reach_their_branches():
    """The oracle's view of the constructed signatures: R = O, x(R) == r with an odd y, and s G == u P."""
    G = S.E.PT.BASE
    for name, sig, msg, pk in S.constructed_cases():
        Pt = SR.lift_x(int.from_bytes(pk, "big"))
        s = int.from_bytes(sig[32:], "big")
        u = (S.N - SR.challenge(sig[:32], pk, msg)) % S.N
        sG, uP = G.multiply(s), Pt.multiply(u)
        R = sG.add(uP)
        if name == "R=O":
            assert R.is0()
        elif name == "odd-y":
            a = R.toAffine()
            assert a["x"] == int.from_bytes(sig[:32], "big") and a["y"] % 2 == 1
        else:
            assert sG.equals(uP) and R.equals(sG.double())


def test_host_bodies_match_oracle_on_signed_batch():
    items, want = S.corrupt(S.signed_batch(40, seed=3), seed=4)
    got = S.emu_verify(items)
    assert got == want
    assert got == [SR.secp256k1_schnorr_verify(*i) for i in items]
    assert 0 < sum(got) < len(items)


def test_mirror_argument_validation_without_device():
    sig, msg, pk = bytes(64), b"m", bytes(32)
    with pytest.raises(ValueError, match="equal length"):
        nmsm.schnorr_verify_batch([sig], [msg, msg], [pk])
    with pytest.raises(ValueError, match="length 64"):
        nmsm.schnorr_verify_batch([bytes(63)], [msg], [pk])
    with pytest.raises(ValueError, match="length 64"):
        nmsm.schnorr.verify(bytes(65), msg, pk)
    with pytest.raises(ValueError, match="length 32"):
        nmsm.schnorr.verify(sig, msg, bytes(33))
    with pytest.raises(TypeError, match="signature"):
        nmsm.schnorr_verify_batch(["00" * 64], [msg], [pk])
    with pytest.raises(TypeError, match="message"):
        nmsm.schnorr_verify_batch([sig], ["m"], [pk])
    with pytest.raises(TypeError, match="publicKey"):
        nmsm.schnorr_verify_batch([sig], [msg], [None])
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.schnorr_verify_batch_packed(bytes(64), pk, msg, bytes(8), 1)
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.schnorr_verify_batch_packed(bytes(64), bytes(33), msg, bytes(16), 1)
