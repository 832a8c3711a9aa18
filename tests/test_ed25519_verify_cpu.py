"""ed25519 per-signature verification without a GPU: the device bodies (prepare + check, ed25519_verify.cuh) run on the
host through tests/hostemu against the oracle (oracle.noble_ref.ed25519_verify, the reference's ed25519.verify) in
both decoding modes, and the host mirror's argument checks."""
import pytest

import ed25519_cases as C
import nmsm
from oracle import noble_ref as R


@pytest.fixture(scope="module")
def cases():
    return C.all_cases()


@pytest.mark.parametrize("zip215", C.MODES)
def test_host_bodies_match_oracle_item_by_item(cases, zip215):
    items = [c[1:] for c in cases]
    got = C.emu_verify(items, zip215)
    want = [R.ed25519_verify(*i, zip215=zip215) for i in items]
    assert got == want, [c[0] for c, g, w in zip(cases, got, want) if g != w][:20]
    names = dict(zip((c[0] for c in cases), got))
    assert all(names["rfc-%d" % j] for j in range(128))
    assert not any(v for k, v in names.items() if k.startswith("rfc-") and k.endswith(("s^1", "msg^")))
    assert names["valid"] and all(names["msg-%d" % ln] for ln in C.MSG_LENS)
    assert all(names["tors-%s-%d" % (w, j)] for w in ("R", "A", "RA") for j in range(8))
    assert not any(names["s=" + s] for s in ("l", "l+1", "2^253", "2^256-1", "l-ident"))
    assert not names["raw-R-canonical-k"]
    zip_only = ["s=0", "s=l-1", "raw-R", "x0-sign-R", "x0-sign-A"] + ["small-A-%d" % j for j in range(8)]
    assert all(names[k] == zip215 for k in zip_only), {k: names[k] for k in zip_only}


def test_zip215_set_matches_its_own_labels():
    """The golden ZIP-215 cases carry the verdict ZIP-215 rules give; the host bodies reproduce each."""
    cases = C.zip215_cases()
    got = C.emu_verify([c[1:] for c in cases], True)
    from conftest import load_golden

    assert got == [v["valid_zip215"] for v in load_golden("ed25519.json")["zip215"]]


def test_host_bodies_on_openssl_signed_batch():
    pytest.importorskip("cryptography")
    items, want = C.corrupt(C.openssl_sign(60, seed=5), seed=6)
    for zip215 in C.MODES:
        got = C.emu_verify(items, zip215)
        assert got == want
        assert got == [C.openssl_verify(*i) for i in items]
    assert 0 < sum(want) < len(items)


def test_mirror_argument_validation_without_device():
    sig, msg, pk = bytes(64), b"m", bytes(32)
    with pytest.raises(ValueError, match="equal length"):
        nmsm.ed25519_verify_each([sig], [msg, msg], [pk])
    with pytest.raises(ValueError, match="length 64"):
        nmsm.ed25519_verify_each([bytes(63)], [msg], [pk])
    with pytest.raises(ValueError, match="length 64"):
        nmsm.ed25519.verify(bytes(65), msg, pk)
    with pytest.raises(ValueError, match="length 32"):
        nmsm.ed25519.verify(sig, msg, bytes(33), zip215=False)
    with pytest.raises(TypeError, match="signature"):
        nmsm.ed25519_verify_each(["00" * 64], [msg], [pk])
    with pytest.raises(TypeError, match="message"):
        nmsm.ed25519_verify_each([sig], ["m"], [pk])
    with pytest.raises(TypeError, match="publicKey"):
        nmsm.ed25519.verify(sig, msg, None)
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.ed25519_verify_each_packed(bytes(64), pk, msg, bytes(8), 1)
    with pytest.raises(ValueError, match="packed arrays"):
        nmsm.ed25519_verify_each_packed(bytes(64), bytes(33), msg, bytes(16), 1)
