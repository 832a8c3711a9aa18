"""P-256 ECDSA verification without a GPU: the oracle against OpenSSL, the device bodies (SEC1 decoders, the a = -3
group law, the windowed scalar multiplication, the prepare + check bodies) run on the host through tests/hostemu, and
the host mirror's argument checks."""
import ctypes
import random

import numpy as np
import pytest

import nmsm
import p256_cases as C
from oracle import p256_ref as PR

G = C.PT.BASE


def _words(v: int, n: int = 8) -> np.ndarray:
    return np.array([(v >> (32 * k)) & 0xFFFFFFFF for k in range(n)], np.uint32)


def _xy(Q) -> np.ndarray:
    if Q.is0():
        return np.zeros(16, np.uint32)
    a = Q.toAffine()
    return np.concatenate([_words(a["x"]), _words(a["y"])])


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


def _point(out: np.ndarray, inf: int):
    if inf:
        return None
    return int.from_bytes(out[:8].tobytes(), "little"), int.from_bytes(out[8:].tobytes(), "little")


def _affine(Q):
    if Q.is0():
        return None
    a = Q.toAffine()
    return a["x"], a["y"]


def test_oracle_matches_openssl():
    pytest.importorskip("cryptography")
    high = accepted = 0
    for prehash, seed in ((True, 1), (False, 2)):  # prehash = False: 32-byte digests signed as given
        items = C.openssl_sign(120, seed=seed, prehash=prehash)
        for idx, (sig, msg, pk) in enumerate(items + C.corrupt(items, seed=seed + 10)):
            ossl = C.openssl_verify(sig, msg, pk, prehash=prehash)
            assert PR.p256_ecdsa_verify(sig, msg, pk, prehash=prehash) == ossl, (prehash, idx)
            s = int.from_bytes(sig[32:], "big")
            high += s > C.N >> 1
            accepted += ossl
    assert high > 50 and accepted > 200  # OpenSSL does not normalise s: both halves are exercised


def test_precompile_oracle_agrees_with_verify():
    """P256VERIFY is p256.verify without prehash and lowS on the key 04 || qx || qy (or False for a bad length)."""
    for name, inp in C.precompile_cases():
        want = PR.p256verify_precompile(inp)
        if len(inp) != 160:
            assert want is False, name
            continue
        got = PR.p256_ecdsa_verify(inp[32:96], inp[:32], b"\x04" + inp[96:], prehash=False, lowS=False)
        assert got == want, name


def emu_verify(items, prehash, lowS):
    sigs, pks, pk_off, msgs, msg_off = C.pack([i[0] for i in items], [i[1] for i in items], [i[2] for i in items])
    out = ctypes.create_string_buffer(max(len(items), 1))
    flags = (nmsm.ECDSA_PREHASH if prehash else 0) | (nmsm.ECDSA_LOW_S if lowS else 0)
    cp = lambda b: ctypes.c_char_p(b or b"\0")  # noqa: E731
    rc = C.p256_emu().emu_p256_verify_batch(cp(sigs), cp(pks), cp(pk_off), cp(msgs), cp(msg_off), len(items), flags, out)
    assert rc == 0
    return [b == 1 for b in out.raw[:len(items)]]


@pytest.mark.parametrize("prehash,lowS", C.FLAGS)
def test_host_bodies_match_oracle_on_edge_set(prehash, lowS):
    cases = C.edge_cases()
    got = emu_verify([(c[1], c[2], c[3]) for c in cases], prehash, lowS)
    want = [PR.p256_ecdsa_verify(c[1], c[2], c[3], prehash=prehash, lowS=lowS) for c in cases]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w]
    names = {c[0]: w for c, w in zip(cases, want)}
    if not prehash:  # the constructed signatures carry their h as a raw 32-byte message
        assert names["Rx>=n"] and names["u1G=u2Q"] and names["h=n"] and names["empty-raw"]
        assert not names["R=O"] and not names["Rx>=n-r=x"] and not names["raw-8193"] and names["raw-8192"]
        assert names["s=%x" % (C.N >> 1)] and names["s=%x" % ((C.N >> 1) + 1)] == (not lowS)
        assert names["u1=0"] or lowS
    else:
        assert names["valid"] and names["valid-65"] and names["empty-prehash"]
        assert names["valid-negated-s"] == (not lowS)


def test_host_bodies_match_oracle_on_precompile_inputs():
    cases = [(n, i) for n, i in C.precompile_cases() if len(i) == 160]
    items = [(i[32:96], i[:32], b"\x04" + i[96:]) for _, i in cases]
    got = emu_verify(items, prehash=False, lowS=False)
    want = [PR.p256verify_precompile(i) for _, i in cases]
    assert got == want, [n for (n, _), g, w in zip(cases, got, want) if g != w]


def test_host_bodies_match_openssl():
    pytest.importorskip("cryptography")
    for prehash, seed in ((True, 31), (False, 32)):
        items = C.corrupt(C.openssl_sign(40, seed=seed, prehash=prehash), seed=seed + 1)
        assert emu_verify(items, prehash, False) == [C.openssl_verify(*i, prehash=prehash) for i in items]


def test_decoders_match_oracle():
    rnd = random.Random(6)
    encs = []
    for _ in range(20):
        Q = G.multiply(rnd.randrange(1, C.N))
        a = Q.toAffine()
        encs += [C.compressed(Q), C.uncompressed(Q), b"\x04" + C.be32(a["x"]) + C.be32((a["y"] + 1) % C.P)]
    encs += [c[3] for c in C.edge_cases() if c[0].startswith("key-")]
    lib = C.p256_emu()
    for enc in encs:
        out = np.zeros(16, np.uint32)
        st = lib.emu_p256_decode(ctypes.c_char_p(enc or b"\0"), ctypes.c_uint64(len(enc)), _ptr(out))
        try:
            x, y = PR.p256_decode_sec1(enc)
        except (ValueError, IndexError):
            assert st == 0, enc.hex()
            continue
        assert st == 1, enc.hex()
        assert _point(out, 0) == (x, y)


def _group_op(op, p, q, lam_p=0, lam_q=0):
    out = np.zeros(16, np.uint32)
    a, b, lp, lq = _xy(p), _xy(q), _words(lam_p), _words(lam_q)
    inf = C.p256_emu().emu_p256_group_op(op, _ptr(a), _ptr(lp), _ptr(b), _ptr(lq), _ptr(out))
    return _point(out, inf)


def test_group_law_matches_oracle():
    """The a = -3 dbl, dbl_affine, madd and add against the oracle's complete formulas, on random points with random
    projective factors and on P + P, P + (-P), O + P and P + O."""
    rnd = random.Random(9)
    O = G.multiply(1).subtract(G)
    for _ in range(24):
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


def test_scalar_mul_and_group_order_in_host_emulation():
    rnd = random.Random(10)
    lib = C.p256_emu()
    out = np.zeros(16, np.uint32)
    g = _xy(G)
    assert lib.emu_p256_mul(_ptr(g), _ptr(_words(C.N)), _ptr(out)) == 1  # n G = O
    assert lib.emu_p256_mul(_ptr(g), _ptr(_words(C.N - 1)), _ptr(out)) == 0
    assert _point(out, 0) == _affine(G.negate())
    for k in [1, 2, 3, 15, 16, 17, C.N >> 1, 2**255] + [rnd.randrange(1, C.N) for _ in range(8)]:
        Q = G.multiply(rnd.randrange(1, C.N))
        q = _xy(Q)
        inf = lib.emu_p256_mul(_ptr(q), _ptr(_words(k)), _ptr(out))
        assert _point(out, inf) == _affine(Q.multiply(k)), k


def test_mirror_argument_validation_without_device():
    sig, msg, pk = bytes(64), b"m", bytes(33)
    with pytest.raises(ValueError, match="equal length"):
        nmsm.p256_ecdsa_verify_batch([sig], [msg, msg], [pk])
    with pytest.raises(ValueError, match="length 64"):
        nmsm.p256_ecdsa_verify_batch([bytes(63)], [msg], [pk])
    with pytest.raises(ValueError, match="length 64"):
        nmsm.p256.verify(bytes(63), msg, pk)
    with pytest.raises(TypeError, match="signature"):
        nmsm.p256_ecdsa_verify_batch(["00" * 64], [msg], [pk])
    with pytest.raises(TypeError, match="message"):
        nmsm.p256_ecdsa_verify_batch([sig], ["m"], [pk])
    with pytest.raises(TypeError, match="publicKey"):
        nmsm.secp256r1.verify(sig, msg, None)
    with pytest.raises(NotImplementedError, match="not part of the accelerated path"):
        nmsm.p256.verify(sig, msg, pk, format="der")
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.p256_ecdsa_verify_batch_packed(bytes(64), pk, bytes(8), msg, bytes(16), 1)
    with pytest.raises(TypeError, match="P256VERIFY"):
        nmsm.p256verify_precompile_batch(["00" * 160])
    with pytest.raises(ValueError, match="multiple of 160"):
        nmsm.p256verify_precompile_batch(bytes(161))
    # wrong lengths are False without reaching the library
    assert nmsm.p256verify_precompile_batch([b"", bytes(159), bytes(161)]) == [False, False, False]
    assert nmsm.p256verify_precompile_batch(b"") == []
    assert nmsm.secp256r1 is nmsm.p256 and "p256" not in nmsm.CURVES
