"""ed25519 per-signature verification on the GPU (nmsm_ed25519_verify_each): every verdict is compared per item with
the oracle (oracle.noble_ref.ed25519_verify, the reference's ed25519.verify) in both decoding modes, or with the verdict
known from how the batch was constructed."""
import ctypes
import random
import struct

import pytest

import ecdsa_cases as E
import ed25519_cases as C
from oracle import ecdsa_ref as ER
from oracle import noble_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


@pytest.fixture(scope="module")
def cases():
    return C.all_cases()


@pytest.fixture(scope="module")
def openssl_4096():
    pytest.importorskip("cryptography")
    return C.openssl_sign(4096, seed=41)


def _verify(nmsm, items, zip215=True):
    return nmsm.ed25519_verify_each([i[0] for i in items], [i[1] for i in items], [i[2] for i in items], zip215=zip215)


@pytest.mark.parametrize("zip215", C.MODES)
def test_all_cases_match_oracle_in_one_batch(nmsm, cases, zip215):
    items = [c[1:] for c in cases]
    got = _verify(nmsm, items, zip215)
    want = [R.ed25519_verify(*i, zip215=zip215) for i in items]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w][:20]
    names = dict(zip((c[0] for c in cases), got))
    assert names["valid"] and names["tors-R-7"] and names["msg-1000"]
    assert names["raw-R"] == zip215 and names["small-A-0"] == zip215 and not names["raw-R-canonical-k"]


@pytest.mark.parametrize("zip215", C.MODES)
def test_single_form_on_golden_sets(nmsm, zip215):
    for name, sig, msg, pk in C.rfc_vectors()[::3] + C.zip215_cases() + C.strict_edge_cases():
        assert nmsm.ed25519.verify(sig, msg, pk, zip215=zip215) is R.ed25519_verify(sig, msg, pk, zip215), name


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097, (1 << 16) + 3])
def test_batches_with_scattered_invalid_items(nmsm, openssl_4096, n):
    base = [openssl_4096[i % len(openssl_4096)] for i in range(n)]
    items, want = C.corrupt(base, seed=500 + n)
    for zip215 in C.MODES:
        got = _verify(nmsm, items, zip215)
        assert got == want, [k for k in range(n) if got[k] != want[k]][:10]
    for k in random.Random(n).sample(range(n), min(n, 12)):  # oracle sample
        assert got[k] == R.ed25519_verify(*items[k], zip215=False), k
    if n >= 32:  # valid and invalid items side by side within one warp
        assert any(0 < sum(got[w:w + 32]) < len(got[w:w + 32]) for w in range(0, n, 32))


def test_openssl_batch_all_accepted(nmsm, openssl_4096):
    for zip215 in C.MODES:
        assert _verify(nmsm, openssl_4096, zip215) == [True] * len(openssl_4096)


def _batch_equation(nmsm, items, seed):
    z = random.Random(seed).randbytes(16 * len(items))
    return nmsm.ed25519_verify_batch([i[0] for i in items], [i[1] for i in items], [i[2] for i in items], z)


def test_agrees_with_the_batch_equation(nmsm, openssl_4096):
    """All valid: the batch equation holds and every verdict is 1.  One decodable forgery: the batch equation fails
    without an index, and exactly that signature gets a 0 verdict."""
    items = list(openssl_4096)
    assert _batch_equation(nmsm, items, 1) == (True, -1)
    assert _verify(nmsm, items) == [True] * len(items)
    idx = 1234
    sig, msg, pk = items[idx]
    items[idx] = (sig[:32] + C.le32((int.from_bytes(sig[32:], "little") + 1) % C.L), msg, pk)
    assert _batch_equation(nmsm, items, 2) == (False, -1)
    got = _verify(nmsm, items)
    assert [k for k, v in enumerate(got) if not v] == [idx]


def _ecdsa_round(nmsm):
    cases = E.edge_cases()
    got = nmsm.ecdsa_verify_batch([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
    assert got == [ER.secp256k1_ecdsa_verify(c[1], c[2], c[3]) for c in cases]


def _each_round(nmsm, cases):
    items = [c[1:] for c in cases]
    assert _verify(nmsm, items) == [R.ed25519_verify(*i) for i in items]


def test_interleaved_with_ecdsa_and_the_batch_equation(nmsm, cases, openssl_4096):
    """The three share the verification scratch: each call must leave the next one's inputs alone."""
    short = cases[::5]
    for _ in range(2):
        _each_round(nmsm, short)
        _ecdsa_round(nmsm)
        assert _batch_equation(nmsm, openssl_4096[:300], 3) == (True, -1)
        _each_round(nmsm, short)


def test_table_of_b_survives_repeated_calls(nmsm, openssl_4096):
    items, want = C.corrupt(openssl_4096[:500], seed=77)
    for _ in range(5):
        assert _verify(nmsm, items) == want
        assert _verify(nmsm, items, zip215=False) == want


def test_error_codes_and_empty_batch(nmsm):
    lib = nmsm._lib.load()
    ERR = nmsm._lib.ERR_ARG
    sig, msg, pk = C.sign_with(5, 7, b"error codes")
    off = lambda *v: struct.pack("<%dQ" % len(v), *v)  # noqa: E731
    out = ctypes.create_string_buffer(b"\xaa" * 4, 4)
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p) if b is not None else None  # noqa: E731
    call = lambda s, p, m, mo, n, fl: lib.nmsm_ed25519_verify_each(cp(s), cp(p), cp(m), cp(mo), n, fl, out)  # noqa: E731
    assert call(None, None, None, None, 0, 0) == 0 and out.raw == b"\xaa" * 4  # n == 0 writes nothing
    assert call(sig, pk, msg, off(0, len(msg)), 1, 0) == 0 and out.raw[0] == 1
    assert call(sig, pk, msg, off(0, len(msg)), 1, 1) == 0 and out.raw[0] == 1
    assert call(sig, pk, msg, off(0, len(msg)), 1, 2) == ERR  # unknown flag bit
    assert call(sig, pk, msg, off(0, len(msg)), 1, -1) == ERR
    assert call(None, pk, msg, off(0, len(msg)), 1, 0) == ERR
    assert call(sig, None, msg, off(0, len(msg)), 1, 0) == ERR
    assert call(sig, pk, msg, None, 1, 0) == ERR
    assert call(sig, pk, None, off(0, len(msg)), 1, 0) == (ERR if msg else 0)
    assert call(sig, pk, None, off(0, 0), 1, 0) == 0  # an empty message needs no message buffer
    assert call(sig, pk, msg, off(0, len(msg)), 1 << 31, 0) == ERR  # before msg_off[n] is read
    assert call(sig, pk, msg, off(1, len(msg)), 1, 0) == ERR
    assert "msg_off[0] must be 0" in nmsm._lib.load().nmsm_last_error().decode()
    assert call(sig * 2, pk * 2, msg, off(0, len(msg), 0), 2, 0) == ERR
    assert "non-decreasing (index 2)" in nmsm._lib.load().nmsm_last_error().decode()
    assert nmsm.ed25519_verify_each([], [], []) == []


def test_profiling_slots(nmsm, openssl_4096):
    nmsm.set_profiling(True)
    try:
        _verify(nmsm, openssl_4096)
        ms = nmsm.last_timing()[0]
    finally:
        nmsm.set_profiling(False)
    # slot 0: k_ed_verify_prepare, slot 1: k_ed_verify_check (include/nmsm.h)
    prep, check = list(ms.values())[:2]
    assert prep > 0 and check > 0 and ms["total"] >= prep + check - 1e-3


def test_table_is_rebuilt_after_reinit(nmsm, cases):
    """Last in this module: nmsm_shutdown frees the table of B and the next call after nmsm_init builds it again."""
    lib = nmsm._lib.load()
    lib.nmsm_shutdown()
    nmsm._lib.check(lib.nmsm_init(0))
    _each_round(nmsm, cases[::7])
    _ecdsa_round(nmsm)
