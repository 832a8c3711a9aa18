"""EIP-4844 KZG proof verification without a GPU: the oracle (oracle.kzg_ref) against the spec's constants and against
independent restatements (the inverse NTT of oracle/noble_fft.py, hashlib, the pairing), and the device bodies of
kzg.cuh run on the host through tests/hostemu against the oracle: the challenge, the blob evaluation, Fr inversion,
the prepare body's pairs and the serial verdicts of a mixed batch."""
import hashlib
import random

import pytest

import kzg_cases as C
from oracle import hash_to_g1_ref as H
from oracle import kzg_ref as K
from oracle import noble_fft

R = K.BLS_MODULUS
OMEGA = 0x564C0A11A0F704F4FC3E8ACFE0F8245F0AD1347B378FBF96E206DA11A5D36306


# ---- the oracle --------------------------------------------------------------------------------------------------
def test_constants():
    assert R == H.N  # the BLS12-381 group order
    assert K.FIELD_ELEMENTS_PER_BLOB == 4096 and K.BYTES_PER_BLOB == 131072
    assert K.ROOTS_OF_UNITY[1] == OMEGA == pow(7, (R - 1) // 4096, R)


def test_omega_has_order_exactly_4096():
    assert pow(OMEGA, 4096, R) == 1 and pow(OMEGA, 2048, R) != 1
    assert len(set(K.ROOTS_OF_UNITY)) == 4096


def test_bit_reversal_of_the_domain():
    brp = K.BRP_ROOTS_OF_UNITY
    w = K.ROOTS_OF_UNITY
    assert (brp[0], brp[1], brp[2], brp[3]) == (w[0], w[2048], w[1024], w[3072])
    assert brp[4095] == w[4095] and brp[1 << 11] == w[1]
    assert noble_fft.reverse_bits(6, 12) == 0b011000000000


def test_barycentric_equals_coefficient_form():
    """the blob as evaluations over the bit-reversed domain, interpolated by the reference's inverse NTT, evaluated by
    Horner at random z: the same value as the spec's barycentric formula"""
    blob = C.random_blob(3)
    poly = K.blob_to_polynomial(blob)
    fft = noble_fft.FFT(noble_fft.RootsOfUnity(R, 7))
    coeffs = fft.inverse(noble_fft.bit_reversal_permutation(poly))
    rnd = random.Random(5)
    for _ in range(3):
        z = rnd.randrange(R)
        assert K.evaluate_polynomial_in_evaluation_form(poly, z) == noble_fft.eval_poly(R, coeffs, z)


def test_z_on_the_domain_returns_the_element():
    poly = K.blob_to_polynomial(C.random_blob(4))
    for k in (0, 1, 2048, 4095):
        assert K.evaluate_polynomial_in_evaluation_form(poly, K.BRP_ROOTS_OF_UNITY[k]) == poly[k]


def test_challenge_transcript_layout():
    blob, c = C.random_blob(6), C.blob_item(1)[1]
    t = K.challenge_transcript(blob, c)
    assert len(t) == 16 + 16 + 131072 + 48
    assert t[:16] == b"FSBLOBVERIFY_V1_"
    assert t[16:32] == bytes(14) + b"\x10\x00"
    assert t[32:32 + 131072] == blob and t[-48:] == c
    assert K.compute_challenge(blob, c) == int.from_bytes(hashlib.sha256(t).digest(), "big") % R


def test_oracle_pairing_accepts_honest_and_rejects_changed_y():
    rnd = random.Random(7)
    c, z, y, pi = C.proof_item(rnd)
    assert K.verify_kzg_proof(c, C.be(z), C.be(y), pi, C.SETUP)
    assert not K.verify_kzg_proof(c, C.be(z), C.be((y + 1) % R), pi, C.SETUP)
    assert not K.verify_kzg_proof(c, C.be(z), C.be(y), pi, C.OTHER_SETUP)
    blob, bc, bpi, _, _ = C.blob_item(1)
    assert K.verify_blob_kzg_proof(blob, bc, bpi, C.SETUP)


def test_zero_blob_and_identities():
    assert K.verify_blob_kzg_proof(C.ZERO_BLOB, C.IDENTITY, C.IDENTITY, C.SETUP)
    assert not K.verify_blob_kzg_proof(C.ZERO_BLOB, C.NON_CANONICAL_IDENTITY, C.IDENTITY, C.SETUP)


def test_precompile_return_bytes():
    item = C.proof_item(random.Random(8))
    out = K.point_evaluation_precompile(C.precompile_input(item), C.SETUP)
    assert out == (4096).to_bytes(32, "big") + R.to_bytes(32, "big")
    assert out.hex().endswith("73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001")
    assert out[:32] == bytes(30) + b"\x10\x00"
    bad = b"\x00" + C.precompile_input(item)[1:]
    assert K.point_evaluation_precompile(bad, C.SETUP) is None
    assert K.point_evaluation_precompile(C.precompile_input(item)[:191], C.SETUP) is None


def test_mirror_constants():
    import nmsm

    assert nmsm.KZG_FIELD_ELEMENTS_PER_BLOB == 4096 and nmsm.KZG_BYTES_PER_BLOB == 131072
    assert nmsm.POINT_EVALUATION_OUTPUT == (4096).to_bytes(32, "big") + R.to_bytes(32, "big")


def test_mirror_argument_checks():
    import nmsm

    with pytest.raises(ValueError):
        nmsm.kzg_verify_proof_batch([b"\0" * 47], [0], [0], [C.IDENTITY], C.SETUP)
    with pytest.raises(ValueError):
        nmsm.kzg_verify_proof_batch([C.IDENTITY], [1 << 256], [0], [C.IDENTITY], C.SETUP)
    with pytest.raises(ValueError):
        nmsm.kzg_verify_blob_proof_batch([b"\0" * 100], [C.IDENTITY], [C.IDENTITY], C.SETUP)
    with pytest.raises(ValueError):
        nmsm.eth_point_evaluation_batch(b"\0" * 100, C.SETUP)
    with pytest.raises(ValueError):
        nmsm.kzg_verify_proof_batch([C.IDENTITY], [0], [0], [C.IDENTITY], C.SETUP[:95])


# ---- host emulation of the device bodies --------------------------------------------------------------------------
def test_emu_roots_are_the_bit_reversed_domain():
    assert C.emu_roots() == K.BRP_ROOTS_OF_UNITY


def test_emu_challenge_matches_hashlib():
    items = [C.blob_item(s) for s in (1, 2)]
    blobs = [i[0] for i in items] + [C.ZERO_BLOB, bytes([0xFF]) * K.BYTES_PER_BLOB]
    cs = [i[1] for i in items] + [C.IDENTITY, C.off_curve_g1()]
    want = [int.from_bytes(hashlib.sha256(K.challenge_transcript(b, c)).digest(), "big") % R for b, c in zip(blobs, cs)]
    assert C.emu_challenge(blobs, cs) == want


def test_emu_eval_matches_oracle():
    blob = C.random_blob(9)
    poly = K.blob_to_polynomial(blob)
    brp = K.BRP_ROOTS_OF_UNITY
    rnd = random.Random(10)
    cases = [(blob, rnd.randrange(R)), (blob, brp[0]), (blob, brp[4095]), (blob, brp[77]), (C.ZERO_BLOB, 12345)]
    got = C.emu_eval([b for b, _ in cases], [z for _, z in cases])
    for (b, z), (y, ok) in zip(cases, got):
        assert ok and y == K.evaluate_polynomial_in_evaluation_form(K.blob_to_polynomial(b), z)
    assert got[1][0] == poly[0] and got[2][0] == poly[4095]


@pytest.mark.parametrize("index", [0, 4095])
@pytest.mark.parametrize("value", [R, (1 << 256) - 1])
def test_emu_eval_rejects_an_element_out_of_range(index, value):
    blob = C.blob_with(C.random_blob(11), index, value)
    ((_, ok),) = C.emu_eval([blob], [5])
    assert not ok


def test_emu_fr_inverse():
    rnd = random.Random(12)
    for a in [1, 2, R - 1, 4096] + [rnd.randrange(1, R) for _ in range(20)]:
        assert C.emu_fr_inv(a) == pow(a, -1, R)


def test_emu_prepare_pairs():
    rnd = random.Random(13)
    c, z, y, pi = C.proof_item(rnd)
    items = [(c, z, y, pi), (C.IDENTITY, 0, 0, C.IDENTITY), (c, R, y, pi)]
    pairs, pre = C.emu_prepare(items)
    assert pre == [1, 1, 0]
    # Q = C - y G1 + z pi
    cpt, pipt = K.g1_decode(c), K.g1_decode(pi)
    q = H.point_add(H.point_add(cpt, H.point_neg(K.g1_mul(y, K.G1_GEN))), K.g1_mul(z, pipt))
    g1, g2 = pairs[0]
    assert g1 == H.g1_packed(q) + H.g1_packed(pipt)
    neg_g2 = K.B.affine(K.B.G2.BASE.negate())
    tau = K.B.affine(K.setup_g2_point(C.TAU))
    pack2 = lambda p: b"".join(v.to_bytes(48, "little") for v in (p[0][0], p[0][1], p[1][0], p[1][1]))  # noqa: E731
    assert g2 == pack2(neg_g2) + pack2(tau)
    assert pairs[1][0] == bytes(192)  # Q = O and pi = O: identity pairs, accepted
    assert pairs[2] == (bytes(192), bytes(384))


def test_emu_setup_rejections():
    items = [C.proof_item(random.Random(14))]
    for bad in (b"\xc0" + bytes(95), bytes(96), C.SETUP[:1] + bytes([C.SETUP[1] ^ 1]) + C.SETUP[2:]):
        c, z, y, pi = C.pack_proofs(items)
        import ctypes

        g1, g2, pre = (ctypes.create_string_buffer(k) for k in (192, 384, 1))
        assert C.kzg_emu().emu_kzg_prepare(c, z, y, pi, None, None, 1, bad, g1, g2, pre) == -1


def test_emu_serial_verdicts_match_oracle():
    rnd = random.Random(15)
    good = [C.proof_item(rnd) for _ in range(3)]
    c, z, y, pi = good[0]
    items = good + [
        (c, z, (y + 1) % R, pi),
        (c, (z + 1) % R, y, pi),
        (c, z, y, good[1][3]),
        (C.off_curve_g1(), z, y, pi),
        (c, z, y, C.small_order_g1()),
        (C.NON_CANONICAL_IDENTITY, z, y, pi),
        (C.uncompressed_flag(c), z, y, pi),
        (C.IDENTITY, 0, 0, C.IDENTITY),
        (C.IDENTITY, 5, 0, C.IDENTITY),
    ]
    want = [True] * 3 + [False] * 7 + [True, True]
    assert C.emu_verify(items) == want
    vhs = [C.versioned_hash(i[0]) for i in items[:3]]
    vhs[1] = b"\x00" + vhs[1][1:]
    vhs[2] = vhs[2][:31] + bytes([vhs[2][31] ^ 1])
    assert C.emu_verify(items[:3], vhs=vhs) == [True, False, False]
