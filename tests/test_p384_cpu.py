"""P-384 ECDSA verification without a GPU: the oracle against OpenSSL, the device bodies (SHA-384, the SEC1 decoders, the
a = -3 group law at 12 limbs, the windowed and table scalar multiplications with 12-word scalars, the prepare + check
bodies) run on the host through tests/hostemu, and the host mirror's argument checks."""
import ctypes
import hashlib
import random

import numpy as np
import pytest

import nmsm
import p384_cases as C
from oracle import p384_ref as PR

G = C.PT.BASE
W = 12


def _words(v: int, n: int = W) -> np.ndarray:
    return np.array([(v >> (32 * k)) & 0xFFFFFFFF for k in range(n)], np.uint32)


def _xy(Q) -> np.ndarray:
    if Q.is0():
        return np.zeros(2 * W, np.uint32)
    a = Q.toAffine()
    return np.concatenate([_words(a["x"]), _words(a["y"])])


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


def _point(out: np.ndarray, inf: int):
    if inf:
        return None
    return int.from_bytes(out[:W].tobytes(), "little"), int.from_bytes(out[W:].tobytes(), "little")


def _affine(Q):
    if Q.is0():
        return None
    a = Q.toAffine()
    return a["x"], a["y"]


def test_curve_constants():
    """G is on the curve, has order n, and the oracle's (n - 1) G is -G."""
    p, a, b = C.P, C.A, C.B
    gx, gy = PR.P384_CURVE["Gx"], PR.P384_CURVE["Gy"]
    assert (gy * gy - gx ** 3 - a * gx - b) % p == 0 and a == p - 3
    assert _affine(G.multiply(C.N - 1)) == _affine(G.negate()) and G.multiply(C.N - 1).add(G).is0()
    assert p % 4 == 3 and C.N >> 383 == 1 and p - C.N < 2**190


def test_oracle_matches_openssl():
    pytest.importorskip("cryptography")
    high = accepted = 0
    for prehash, seed in ((True, 1), (False, 2)):  # prehash = False: 48-byte digests signed as given
        items = C.openssl_sign(60, seed=seed, prehash=prehash)
        for idx, (sig, msg, pk) in enumerate(items + C.corrupt(items, seed=seed + 10)):
            ossl = C.openssl_verify(sig, msg, pk, prehash=prehash)
            assert PR.p384_ecdsa_verify(sig, msg, pk, prehash=prehash) == ossl, (prehash, idx)
            high += int.from_bytes(sig[48:], "big") > C.N >> 1
            accepted += ossl
    assert high > 25 and accepted > 100  # OpenSSL does not normalise s: both halves are exercised


def test_sha384_matches_hashlib():
    lib = C.p384_emu()
    rnd = random.Random(3)
    out = ctypes.create_string_buffer(48)
    for ln in range(0, 301):
        m = bytes(rnd.randrange(256) for _ in range(ln))
        lib.emu_sha384(ctypes.c_char_p(m or b"\0"), ctypes.c_uint64(ln), out)
        assert out.raw == hashlib.sha384(m).digest(), ln


def emu_verify(items, prehash, lowS):
    sigs, pks, pk_off, msgs, msg_off = C.pack([i[0] for i in items], [i[1] for i in items], [i[2] for i in items])
    out = ctypes.create_string_buffer(max(len(items), 1))
    flags = (nmsm.ECDSA_PREHASH if prehash else 0) | (nmsm.ECDSA_LOW_S if lowS else 0)
    cp = lambda b: ctypes.c_char_p(b or b"\0")  # noqa: E731
    rc = C.p384_emu().emu_p384_verify_batch(cp(sigs), cp(pks), cp(pk_off), cp(msgs), cp(msg_off), len(items), flags, out)
    assert rc == 0
    return [b == 1 for b in out.raw[:len(items)]]


@pytest.mark.parametrize("prehash,lowS", C.FLAGS)
def test_host_bodies_match_oracle_on_edge_set(prehash, lowS):
    cases = C.edge_cases()
    got = emu_verify([(c[1], c[2], c[3]) for c in cases], prehash, lowS)
    want = [PR.p384_ecdsa_verify(c[1], c[2], c[3], prehash=prehash, lowS=lowS) for c in cases]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    names = {c[0]: w for c, w in zip(cases, want)}
    if not prehash:  # the constructed signatures carry their h as a raw 48-byte message
        assert names["Rx>=n"] and names["u1G=u2Q"] and names["h=n"] and names["empty-raw"]
        assert not names["R=O"] and not names["Rx>=n-r=x"] and not names["raw-8193"] and names["raw-8192"]
        assert names["raw-47"] and names["raw-48"] and names["raw-49"]
        assert names["s=%x" % (C.N >> 1)] and names["s=%x" % ((C.N >> 1) + 1)] == (not lowS)
        assert names["u1=0"] or lowS
    else:
        assert names["valid"] and names["valid-97"] and names["empty-prehash"]
        assert all(names["prehash-%d" % ln] for ln in (111, 112, 127, 128, 239))
        assert names["valid-negated-s"] == (not lowS)
    assert not any(w for k, w in names.items() if k.startswith("key-"))


def test_host_bodies_match_openssl():
    pytest.importorskip("cryptography")
    for prehash, seed in ((True, 31), (False, 32)):
        items = C.corrupt(C.openssl_sign(40, seed=seed, prehash=prehash), seed=seed + 1)
        for lowS in (False, True):
            want = [C.openssl_verify(*i, prehash=prehash, lowS=lowS) for i in items]
            assert emu_verify(items, prehash, lowS) == want
            assert 0 < sum(want) < len(items)


def test_decoders_match_oracle():
    rnd = random.Random(6)
    encs = []
    for _ in range(20):
        Q = G.multiply(rnd.randrange(1, C.N))
        a = Q.toAffine()
        encs += [C.compressed(Q), C.uncompressed(Q), b"\x04" + C.be48(a["x"]) + C.be48((a["y"] + 1) % C.P)]
    encs += [c[3] for c in C.edge_cases() if c[0].startswith("key-")]
    lib = C.p384_emu()
    for enc in encs:
        out = np.zeros(2 * W, np.uint32)
        st = lib.emu_p384_decode(ctypes.c_char_p(enc or b"\0"), ctypes.c_uint64(len(enc)), _ptr(out))
        try:
            x, y = PR.p384_decode_sec1(enc)
        except (ValueError, IndexError):
            assert st == 0, enc.hex()
            continue
        assert st == 1, enc.hex()
        assert _point(out, 0) == (x, y)


def _group_op(op, p, q, lam_p=0, lam_q=0):
    out = np.zeros(2 * W, np.uint32)
    a, b, lp, lq = _xy(p), _xy(q), _words(lam_p), _words(lam_q)
    inf = C.p384_emu().emu_p384_group_op(op, _ptr(a), _ptr(lp), _ptr(b), _ptr(lq), _ptr(out))
    return _point(out, inf)


def test_group_law_matches_oracle():
    """The a = -3 dbl, dbl_affine, madd and add at 12 limbs against the oracle's complete formulas, on random points
    with random projective factors and on P + P, P + (-P), O + P and P + O."""
    rnd = random.Random(9)
    O = G.multiply(1).subtract(G)
    for _ in range(16):
        p, q = G.multiply(rnd.randrange(1, C.N)), G.multiply(rnd.randrange(1, C.N))
        lp, lq = rnd.randrange(1, C.P), rnd.randrange(1, C.P)
        assert _group_op(0, p, q, lp, lq) == _affine(p.add(q))
        assert _group_op(1, p, q, lp) == _affine(p.add(q))
        assert _group_op(2, p, p, lp) == _affine(p.double())
        assert _group_op(3, p, p) == _affine(p.double())
        for op in (0, 1):  # the exceptional cases of the additions
            assert _group_op(op, p, p, lp, lq) == _affine(p.double()), op
            assert _group_op(op, p, p.negate(), lp, lq) is None, op
            assert _group_op(op, O, p, 0, lq) == _affine(p), op
            assert _group_op(op, p, O, lp, 0) == _affine(p), op
        assert _group_op(2, O, O) is None


def test_scalar_mul_with_12_word_scalars():
    rnd = random.Random(10)
    lib = C.p384_emu()
    out = np.zeros(2 * W, np.uint32)
    g = _xy(G)
    assert lib.emu_p384_mul(_ptr(g), _ptr(_words(C.N)), _ptr(out)) == 1  # n G = O
    assert lib.emu_p384_mul(_ptr(g), _ptr(_words(C.N - 1)), _ptr(out)) == 0
    assert _point(out, 0) == _affine(G.negate())
    for k in [1, 2, 3, 15, 16, 17, C.N >> 1, 2**383, 2**256 + 1, 2**320 - 1] + [rnd.randrange(1, C.N) for _ in range(6)]:
        Q = G.multiply(rnd.randrange(1, C.N))
        inf = lib.emu_p384_mul(_ptr(_xy(Q)), _ptr(_words(k)), _ptr(out))
        assert _point(out, inf) == _affine(Q.multiply(k)), k


def test_table_mul_with_12_word_scalars():
    """table_mul_body over a table of G with 8-bit digits: every digit of a 12-word scalar is read, the top level
    carries, and scalars >= n are rejected."""
    rnd = random.Random(11)
    lib = C.p384_emu()
    out = np.zeros(2 * W, np.uint32)
    assert lib.emu_p384_table_mul(_ptr(_words(0)), _ptr(out)) == 1
    assert lib.emu_p384_table_mul(_ptr(_words(C.N)), _ptr(out)) == -1
    assert lib.emu_p384_table_mul(_ptr(_words(2**384 - 1)), _ptr(out)) == -1
    for k in [1, 0x80, 0x81, C.N - 1, C.N >> 1, 2**383, 2**352 + 2**320, int("80" * 48, 16) % C.N] + \
            [rnd.randrange(1, C.N) for _ in range(8)]:
        inf = lib.emu_p384_table_mul(_ptr(_words(k)), _ptr(out))
        assert _point(out, inf) == _affine(G.multiply(k)), hex(k)


def test_mirror_argument_validation_without_device():
    sig, msg, pk = bytes(96), b"m", bytes(49)
    with pytest.raises(ValueError, match="equal length"):
        nmsm.p384_ecdsa_verify_batch([sig], [msg, msg], [pk])
    with pytest.raises(ValueError, match="length 96"):
        nmsm.p384_ecdsa_verify_batch([bytes(64)], [msg], [pk])
    with pytest.raises(ValueError, match="length 96"):
        nmsm.p384.verify(bytes(95), msg, pk)
    with pytest.raises(TypeError, match="signature"):
        nmsm.p384_ecdsa_verify_batch(["00" * 96], [msg], [pk])
    with pytest.raises(TypeError, match="message"):
        nmsm.p384_ecdsa_verify_batch([sig], ["m"], [pk])
    with pytest.raises(TypeError, match="publicKey"):
        nmsm.secp384r1.verify(sig, msg, None)
    with pytest.raises(NotImplementedError, match="not part of the accelerated path"):
        nmsm.p384.verify(sig, msg, pk, format="der")
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.p384_ecdsa_verify_batch_packed(bytes(64), pk, bytes(16), msg, bytes(16), 1)
    assert nmsm.secp384r1 is nmsm.p384 and "p384" not in nmsm.CURVES
    assert nmsm.p384 is not nmsm.p256
