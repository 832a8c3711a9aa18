"""secp256k1 public-key recovery and ecrecover without a GPU: the oracle's Keccak against hashlib's SHA3 and the known
answers, the oracle's recovered keys against the signer's and OpenSSL's keys, the device bodies (Keccak-256 of 64
bytes, the prepare + check bodies in both input layouts) run on the host through tests/hostemu, and the host mirror's
argument checks."""
import hashlib
import random

import pytest

import ecdsa_cases as E
import nmsm
import recover_cases as RC
from oracle import keccak_ref as K
from oracle import noble_ref as R
from oracle import recover_ref as RR


def test_oracle_keccak_sponge_is_sha3_under_sha3_padding():
    """Every length 0..300 crosses the 135 / 136 / 137 and 271 / 272 rate edges."""
    rnd = random.Random(1)
    for ln in range(301):
        data = bytes(rnd.randrange(256) for _ in range(ln))
        assert K.sponge(data, 0x06) == hashlib.sha3_256(data).digest(), ln


def test_oracle_keccak256_known_answers():
    assert K.keccak256(b"").hex() == "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"
    assert RR.eth_address(*RC.key_of(1)) == RC.KEY1_ADDRESS


def test_oracle_recovers_the_keys_known_from_construction():
    cases = RC.edge_cases()
    for name, sig, msg, prehash, want in cases:
        assert RR.secp256k1_recover_public_key(sig, msg, prehash=prehash) == want, name
    names = {c[0]: c[4] for c in cases}
    assert names["rec2-x=n+t"] and names["rec3-x=n+t"] and names["rec2-x=n+t"] != names["rec3-x=n+t"]
    assert names["u1G=u2R"] and names["Q=O"] is None and names["raw-8193"] is None and names["high-s"]
    for name, data, want in RC.ecrecover_cases():
        assert RR.eth_ecrecover(data) == want, name


def test_oracle_recovers_openssl_keys():
    """For OpenSSL signatures exactly one of rec 0 / 1 recovers OpenSSL's key, and that key verifies under OpenSSL."""
    pytest.importorskip("cryptography")
    for prehash, seed in ((True, 31), (False, 32)):
        for sig64, msg, pk in E.openssl_sign(40, seed=seed, prehash=prehash):
            want = R.secp256k1_decode_sec1(pk)
            keys = [RR.secp256k1_recover_public_key(bytes([rec]) + sig64, msg, prehash=prehash) for rec in (0, 1)]
            assert keys.count(want) == 1, (prehash, pk.hex())
            assert E.openssl_verify(sig64, msg, b"\x04" + E.be32(want[0]) + E.be32(want[1]), prehash=prehash,
                                    lowS=False)


def _check_emu_against_oracle(cases):
    for prehash in (True, False):
        sub = [c for c in cases if c[3] == prehash]
        xy, ok = RC.emu_recover([c[1] for c in sub], [c[2] for c in sub], prehash)
        bad = []
        for k, (name, sig, msg, _, _) in enumerate(sub):
            want = RR.secp256k1_recover_public_key(sig, msg, prehash=prehash)
            if ok[k] != (want is not None) or xy[64 * k:64 * k + 64] != RC.xy_bytes(want):
                bad.append(name)
        assert not bad, (prehash, bad)


def test_host_bodies_match_oracle_on_edge_set():
    _check_emu_against_oracle(RC.edge_cases())


def test_host_bodies_match_oracle_on_signed_batch():
    items, want_ok, keys = RC.corrupt(RC.signed_batch(40, seed=5), seed=6)
    xy, ok = RC.emu_recover([i[0] for i in items], [i[1] for i in items], True)
    assert [b == 1 for b in ok] == want_ok
    for k, (sig, msg) in enumerate(items):
        want = RR.secp256k1_recover_public_key(sig, msg)
        assert xy[64 * k:64 * k + 64] == RC.xy_bytes(want), k
        if keys[k] is not None:
            assert want == keys[k], k


def test_host_bodies_match_oracle_on_ecrecover_edge_set():
    cases = RC.ecrecover_cases()
    words, ok = RC.emu_ecrecover([c[1] for c in cases])
    got = [words[32 * k:32 * k + 32] if ok[k] else b"" for k in range(len(cases))]
    assert got == [RR.eth_ecrecover(c[1]) for c in cases], [c[0] for c, g in zip(cases, got) if g != RR.eth_ecrecover(c[1])]
    assert all(words[32 * k:32 * k + 32] == bytes(32) for k in range(len(cases)) if not ok[k])
    assert dict(zip((c[0] for c in cases), got))["key-1"] == bytes(12) + RC.KEY1_ADDRESS


def test_device_keccak256_64_matches_oracle():
    rnd = random.Random(7)
    for _ in range(64):
        data = bytes(rnd.randrange(256) for _ in range(64))
        assert RC.emu_keccak256_64(data) == K.keccak256(data)


def test_mirror_argument_validation_without_device():
    sig, msg = bytes(65), b"m"
    with pytest.raises(ValueError, match="equal length"):
        nmsm.ecdsa_recover_batch([sig], [msg, msg])
    with pytest.raises(ValueError, match="length 65"):
        nmsm.ecdsa_recover_batch([bytes(64)], [msg])
    with pytest.raises(ValueError, match="length 65"):
        nmsm.secp256k1.recoverPublicKey(bytes(66), msg)
    with pytest.raises(TypeError, match="signature"):
        nmsm.ecdsa_recover_batch(["00" * 65], [msg])
    with pytest.raises(TypeError, match="message"):
        nmsm.ecdsa_recover_batch([sig], ["m"])
    with pytest.raises(TypeError, match="input 0"):
        nmsm.eth_ecrecover_batch(["00" * 128])
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.ecdsa_recover_batch_packed(bytes(64), msg, bytes(16), 1, 0)
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.eth_ecrecover_batch_packed(bytes(127), 1)
    assert nmsm.eth_ecrecover_batch([]) == []
