"""EIP-4844 KZG proof verification on the GPU (nmsm_bls12_381_kzg_verify_proof_batch, nmsm_bls12_381_kzg_verify_blob_batch
and the Python mirror): honest items from the oracle's test prover verify at several sizes (the blob path across its
1024-blob chunk boundary), each corruption is False without touching its neighbours, the blob path agrees with the
proof path fed the oracle's (z, y), and a sample agrees with the oracle's own pairing verdicts."""
import random

import pytest

import bls_cases as BC
import kzg_cases as C
import torsion_cases as TC
from oracle import bls_pairing_ref as B
from oracle import kzg_ref as K

pytestmark = pytest.mark.gpu
R = C.R


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _proofs(nmsm, items, setup=C.SETUP, vhs=None):
    c, z, y, pi = C.pack_proofs(items)
    out = nmsm.kzg_verify_proof_batch_packed(c, z, y, pi, b"".join(vhs) if vhs is not None else None, len(items),
                                             setup)
    return [b == 1 for b in out]


def _blobs(nmsm, blobs, cs, pis, setup=C.SETUP):
    out = nmsm.kzg_verify_blob_proof_batch_packed(b"".join(blobs), b"".join(cs), b"".join(pis), len(blobs), setup)
    return [b == 1 for b in out]


def _blob_items(count, distinct=4):
    base = [C.blob_item(s) for s in range(1, 1 + min(count, distinct))]
    return [base[k % len(base)] for k in range(count)]


@pytest.mark.parametrize("n", [1, 33, 300, 4096])
def test_honest_proofs_verify(nmsm, n):
    items = C.proof_items(n)
    assert _proofs(nmsm, items) == [True] * n
    vhs = [C.versioned_hash(i[0]) for i in items]
    assert _proofs(nmsm, items, vhs=vhs) == [True] * n


@pytest.mark.parametrize("n", [1, 3, 64, 1025])
def test_honest_blobs_verify(nmsm, n):
    items = _blob_items(n)
    assert _blobs(nmsm, [i[0] for i in items], [i[1] for i in items], [i[2] for i in items]) == [True] * n


def test_zero_blob_with_identities(nmsm):
    blob, c, pi, _, _ = C.blob_item(1)
    got = _blobs(nmsm, [C.ZERO_BLOB, blob, C.ZERO_BLOB], [C.IDENTITY, c, C.NON_CANONICAL_IDENTITY],
                 [C.IDENTITY, pi, C.IDENTITY])
    assert got == [True, True, False]


def _small(q):
    return B.g1_encode(TC.small_order_point("bls12_381_G1", q, random.Random(q)))


def test_proof_corruptions(nmsm):
    good = C.proof_items(8, distinct=8, seed=21)
    c, z, y, pi = good[0]
    bad = [
        (c, z, (y + 1) % R, pi),
        (c, (z + 1) % R, y, pi),
        (c, z, y, good[1][3]),
        (c, R, y, pi),
        (c, z, R, pi),
        (C.off_curve_g1(), z, y, pi),
        (c, z, y, C.off_curve_g1()),
        (_small(3), z, y, pi),
        (c, z, y, _small(11)),
        (C.NON_CANONICAL_IDENTITY, z, y, pi),
        (c, z, y, C.NON_CANONICAL_IDENTITY),
        (C.uncompressed_flag(c), z, y, pi),
        (c, z, y, C.uncompressed_flag(pi)),
    ]
    items, want = [], []
    for k, b in enumerate(bad):  # every corruption between two honest neighbours
        items += [good[k % 8], b]
        want += [True, False]
    items.append(good[7])
    want.append(True)
    assert _proofs(nmsm, items) == want


def test_versioned_hash_corruptions(nmsm):
    items = C.proof_items(5, distinct=5, seed=22)
    vhs = [C.versioned_hash(i[0]) for i in items]
    vhs[1] = b"\x00" + vhs[1][1:]
    vhs[3] = vhs[3][:20] + bytes([vhs[3][20] ^ 0x40]) + vhs[3][21:]
    assert _proofs(nmsm, items, vhs=vhs) == [True, False, True, False, True]


def test_blob_corruptions(nmsm):
    items = _blob_items(3, distinct=3)
    (b0, c0, p0, _, _), (b1, c1, p1, _, _), (b2, c2, p2, _, _) = items
    cases = [
        (b0, c0, p0, True),
        (C.blob_with(b1, 0, R), c1, p1, False),
        (b2, c2, p2, True),
        (C.blob_with(b0, 4095, R), c0, p0, False),
        (b1, c1, p1, True),
        (C.blob_with(b2, 17, int.from_bytes(b2[544:576], "big") ^ 1), c2, p2, False),  # a changed element
        (b0, c0, p1, False),  # another blob's proof
        (b1, C.off_curve_g1(), p1, False),
        (b2, c2, _small(3), False),
        (b0, c0, C.uncompressed_flag(p0), False),
        (b1, c1, p1, True),
    ]
    got = _blobs(nmsm, [x[0] for x in cases], [x[1] for x in cases], [x[2] for x in cases])
    assert got == [x[3] for x in cases]


def test_other_tau_rejects_everything(nmsm):
    items = C.proof_items(40)
    assert _proofs(nmsm, items, setup=C.OTHER_SETUP) == [False] * 40
    blobs = _blob_items(2)
    assert _blobs(nmsm, [i[0] for i in blobs], [i[1] for i in blobs], [i[2] for i in blobs],
                  setup=C.OTHER_SETUP) == [False, False]


def test_invalid_setup_raises_arg_error(nmsm):
    from nmsm._lib import ERR_ARG, NmsmError

    x, y = BC.g2_off_subgroup(random.Random(23))
    flipped = bytearray(C.SETUP)
    flipped[40] ^= 1
    items = C.proof_items(2)
    for bad in (b"\xc0" + bytes(95), bytes(96), bytes(flipped), B.g2_encode(B.G2.fromAffine({"x": x, "y": y}))):
        with pytest.raises(NmsmError) as e:
            _proofs(nmsm, items, setup=bad)
        assert e.value.code == ERR_ARG
    with pytest.raises(NmsmError) as e:
        _blobs(nmsm, [C.ZERO_BLOB], [C.IDENTITY], [C.IDENTITY], setup=b"\xc0" + bytes(95))
    assert e.value.code == ERR_ARG
    assert _proofs(nmsm, items) == [True, True]  # the context is still usable


def test_blob_path_agrees_with_proof_path(nmsm):
    items = _blob_items(6, distinct=3)
    got_blob = _blobs(nmsm, [i[0] for i in items], [i[1] for i in items], [i[2] for i in items])
    got_proof = _proofs(nmsm, [(i[1], i[3], i[4], i[2]) for i in items])
    assert got_blob == got_proof == [True] * 6
    # a proof for (z, y) of a different blob verifies on the proof path and not on the blob path
    b0, c0, p0, z0, y0 = items[0]
    alt = C.blob_with(b0, 5, 1234)
    assert _proofs(nmsm, [(c0, z0, y0, p0)]) == [True]
    assert _blobs(nmsm, [alt], [c0], [p0]) == [False]


def test_mirror_agrees_with_packed(nmsm):
    items = C.proof_items(6, distinct=6, seed=24)
    items[2] = (items[2][0], items[2][1], (items[2][2] + 1) % R, items[2][3])
    want = [True, True, False, True, True, True]
    cs, zs, ys, pis = zip(*items)
    assert nmsm.kzg_verify_proof_batch(list(cs), list(zs), [C.be(y) for y in ys], list(pis), C.SETUP) == want
    assert nmsm.kzg_verify_proof_batch(list(cs), list(zs), list(ys), list(pis), C.SETUP) == want
    inputs = [C.precompile_input(i) for i in items]
    inputs.insert(1, inputs[0][:191])  # wrong length: False
    assert nmsm.eth_point_evaluation_batch(inputs, C.SETUP) == [True, False] + want[1:]
    assert nmsm.eth_point_evaluation_batch(b"".join(C.precompile_input(i) for i in items), C.SETUP) == want
    blobs = _blob_items(2)
    assert nmsm.kzg_verify_blob_proof_batch([b[0] for b in blobs], [b[1] for b in blobs], [b[2] for b in blobs],
                                            C.SETUP) == [True, True]
    assert nmsm.kzg_verify_proof_batch([], [], [], [], C.SETUP) == []


def test_sample_agrees_with_oracle_pairing(nmsm):
    rnd = random.Random(25)
    good = C.proof_items(3, distinct=3, seed=26)
    c, z, y, pi = good[0]
    sample = good + [(c, z, rnd.randrange(R), pi), (good[1][0], good[1][1], good[1][2], pi),
                     (C.IDENTITY, rnd.randrange(R), 0, C.IDENTITY)]
    want = [K.verify_kzg_proof(c, C.be(z), C.be(y), pi, C.SETUP) for c, z, y, pi in sample]
    assert want == [True, True, True, False, False, True]
    assert _proofs(nmsm, sample) == want
    blob, bc, bpi, _, _ = C.blob_item(2)
    assert _blobs(nmsm, [blob], [bc], [bpi]) == [K.verify_blob_kzg_proof(blob, bc, bpi, C.SETUP)]
