"""secp256k1 ECDSA verification without a GPU: the oracle against OpenSSL, the device bodies (SHA-256, the 65-byte
key decoder, the prepare + check bodies) run on the host through tests/hostemu, and the host mirror's argument
checks."""
import ctypes
import hashlib
import random

import numpy as np
import pytest

import ecdsa_cases as E
import nmsm
from oracle import ecdsa_ref as ER
from oracle import noble_ref as R


def test_oracle_matches_openssl():
    pytest.importorskip("cryptography")
    high = accepted = 0
    for prehash, seed in ((True, 1), (False, 2)):  # prehash = False: 32-byte digests signed as given
        items = E.openssl_sign(120, seed=seed, prehash=prehash)
        for idx, (sig, msg, pk) in enumerate(items + E.corrupt(items, seed=seed + 10)):
            ossl = E.openssl_verify(sig, msg, pk, prehash=prehash, lowS=False)
            assert ER.secp256k1_ecdsa_verify(sig, msg, pk, prehash=prehash, lowS=False) == ossl, (prehash, idx)
            s = int.from_bytes(sig[32:], "big")
            high += s > E.N >> 1
            accepted += ossl
            want = ossl and s <= E.N >> 1
            assert ER.secp256k1_ecdsa_verify(sig, msg, pk, prehash=prehash, lowS=True) == want, (prehash, idx)
    assert high > 50 and accepted > 200  # OpenSSL does not normalise s: both halves are exercised


def _emu_sha256(data: bytes) -> bytes:
    out = ctypes.create_string_buffer(32)
    E.ecdsa_emu().emu_sha256(ctypes.c_char_p(data or b"\0"), ctypes.c_uint64(len(data)), out)
    return out.raw


def test_device_sha256_matches_hashlib():
    rnd = random.Random(5)
    for ln in (0, 1, 55, 56, 63, 64, 119, 120, 1000):
        data = bytes(rnd.randrange(256) for _ in range(ln))
        assert _emu_sha256(data) == hashlib.sha256(data).digest(), ln


def test_uncompressed_decoder_matches_oracle():
    rnd = random.Random(6)
    encs = []
    for _ in range(20):
        Q = E.PT.BASE.multiply(rnd.randrange(1, E.N))
        a = Q.toAffine()
        encs.append(E.uncompressed(Q))
        encs.append(b"\x04" + E.be32(a["x"]) + E.be32((a["y"] + 1) % E.P))
    encs += [b"\x04" + bytes(64), b"\x04" + E.be32(E.P) + bytes(32), b"\x04" + bytes(32) + E.be32(E.P),
             b"\x03" + encs[0][1:], b"\x04" + E.be32(R.SECP256K1_CURVE["Gx"]) + E.be32(E.P - R.SECP256K1_CURVE["Gy"])]
    lib = E.ecdsa_emu()
    for enc in encs:
        out = np.zeros(16, np.uint32)
        st = lib.emu_sec1_decode_uncompressed(ctypes.c_char_p(enc), out.ctypes.data_as(ctypes.c_void_p))
        try:
            x, y = R.secp256k1_decode_sec1(enc)
        except ValueError:
            assert st == 0, enc.hex()
            continue
        assert st == 1, enc.hex()
        assert int.from_bytes(out[:8].tobytes(), "little") == x and int.from_bytes(out[8:].tobytes(), "little") == y


def emu_verify(items, prehash, lowS):
    sigs, pks, pk_off, msgs, msg_off = E.pack([i[0] for i in items], [i[1] for i in items], [i[2] for i in items])
    out = ctypes.create_string_buffer(max(len(items), 1))
    flags = (nmsm.ECDSA_PREHASH if prehash else 0) | (nmsm.ECDSA_LOW_S if lowS else 0)
    cp = lambda b: ctypes.c_char_p(b or b"\0")  # noqa: E731
    rc = E.ecdsa_emu().emu_ecdsa_verify_batch(cp(sigs), cp(pks), cp(pk_off), cp(msgs), cp(msg_off), len(items), flags, out)
    assert rc == 0
    return [b == 1 for b in out.raw[:len(items)]]


@pytest.mark.parametrize("prehash,lowS", E.FLAGS)
def test_host_bodies_match_oracle_on_edge_set(prehash, lowS):
    cases = E.edge_cases()
    got = emu_verify([(c[1], c[2], c[3]) for c in cases], prehash, lowS)
    want = [ER.secp256k1_ecdsa_verify(c[1], c[2], c[3], prehash=prehash, lowS=lowS) for c in cases]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    names = {c[0]: w for c, w in zip(cases, want)}
    if not prehash:  # the constructed signatures carry their h as a raw 32-byte message
        assert names["Rx>=n"] and names["u1G=u2Q"] and names["h=n"] and names["empty-raw"]
        assert not names["R=O"] and not names["Rx>=n-r=x"] and not names["raw-8193"] and names["raw-8192"]
        assert names["s=%x" % (E.N >> 1)] and names["s=%x" % ((E.N >> 1) + 1)] == (not lowS)
    else:
        assert names["valid"] and names["valid-65"] and names["empty-prehash"]


def test_mirror_argument_validation_without_device():
    sig, msg, pk = bytes(64), b"m", bytes(33)
    with pytest.raises(ValueError, match="equal length"):
        nmsm.ecdsa_verify_batch([sig], [msg, msg], [pk])
    with pytest.raises(ValueError, match="length 64"):
        nmsm.ecdsa_verify_batch([bytes(63)], [msg], [pk])
    with pytest.raises(ValueError, match="length 64"):
        nmsm.secp256k1.verify(bytes(65), msg, pk)
    with pytest.raises(TypeError, match="signature"):
        nmsm.ecdsa_verify_batch(["00" * 64], [msg], [pk])
    with pytest.raises(TypeError, match="message"):
        nmsm.ecdsa_verify_batch([sig], ["m"], [pk])
    with pytest.raises(TypeError, match="publicKey"):
        nmsm.ecdsa_verify_batch([sig], [msg], [None])
    with pytest.raises(NotImplementedError, match="not part of the accelerated path"):
        nmsm.secp256k1.verify(sig, msg, pk, format="der")
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.ecdsa_verify_batch_packed(bytes(64), pk, bytes(8), msg, bytes(16), 1)
