"""The EIP-4844 prover's comb (k_kzg_lincomb, k_kzg_lincomb_finish) at every lane count S that the chunk-size policy
reaches on this device, and every proof call across a chunk boundary: commitments of distinct blobs in each S regime
and over two and three chunks; compute_kzg_proof and compute_blob_kzg_proof over two chunks, with the cases where the
spec raises at chunk and warp edges; blobs of 8-bit digit edges at S = 4096 and S = 128; and blobs whose two partial
sums are equal or opposite where the shuffle tree, shared memory, the finish's partials or one lane's walk first add
them.  Every output, every item, is compared byte for byte with the fast exact reference (kzg_prove_fast_ref), with
None exactly where the spec raises."""
import itertools
import random

import pytest

import kzg_cases as C
import kzg_prove_fast_ref as F
import kzg_prove_ref as KP

pytestmark = pytest.mark.gpu
R = C.R
CHUNK = F.CHUNK
# z on the domain at the lane edges of k_kzg_eval and k_kzg_quotient (element t + 256 j is lane t's j-th) and of the comb
LANE_EDGE_INDICES = (0, 1, 31, 32, 127, 128, 255, 256, 511, 512, 1023, 1024, 2047, 2048, 3840, 4095)


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


@pytest.fixture(scope="module")
def lagrange():
    return KP.setup_g1_lagrange(C.TAU)  # ~17 s in the oracle


@pytest.fixture(scope="module")
def setup(nmsm, lagrange):
    s = nmsm.KzgSetup(lagrange)
    yield s
    s.close()


@pytest.fixture(scope="module")
def sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def pool():
    return F.Pool()


def _mismatches(got, want):
    assert len(got) == len(want)
    return [k for k, (g, w) in enumerate(zip(got, want)) if g != w]


def test_commitments_of_distinct_blobs_at_every_lane_count(setup, sms, pool):
    """one call at the largest chunk of each S regime, then 1024, 1025, 1024 + 33 and 2 * 1024 + 264 blobs"""
    counts = F.regime_counts(sms)
    reached = set()
    for off, n in enumerate(sorted(set(counts.values()) | {CHUNK, CHUNK + 1, CHUNK + 33, 2 * CHUNK + 264})):
        idx = pool.indices(n, offset=97 * off)
        got = setup.blob_to_kzg_commitment_batch([pool.blobs[i] for i in idx])
        assert _mismatches(got, [pool.commitments[i] for i in idx]) == [], (n, F.chunk_lanes(n, sms))
        reached |= set(F.chunk_lanes(n, sms))
    assert reached == set(counts), (sms, sorted(reached))


def test_compute_kzg_proof_across_chunks(setup, sms, pool):
    """distinct (blob, z) over two chunks, the second at a middle S: random z, z on the domain at lane edges, z = 0,
    and z >= r at the first and last item of each chunk"""
    n = CHUNK + 140
    assert 128 < F.chunk_lanes(n, sms)[-1] < 4096
    rnd = random.Random(90)
    idx = pool.indices(n, offset=500)
    edges = itertools.cycle(LANE_EDGE_INDICES)
    zs = []
    for k in range(n):
        kind = k % 3
        zs.append(rnd.randrange(R) if kind == 0 else F.BRP[next(edges)] if kind == 1 else 0 if k % 6 == 2 else
                  rnd.randrange(R))
    for k, z in zip((0, CHUNK - 1, CHUNK, n - 1), (R, R + 1, (1 << 256) - 1, 1 << 255)):
        zs[k] = z
    got = setup.compute_kzg_proof_batch([pool.blobs[i] for i in idx], zs)
    want = [F.kzg_proof(pool.blobs[i], z) for i, z in zip(idx, zs)]
    assert [k for k, w in enumerate(want) if w is None] == [0, CHUNK - 1, CHUNK, n - 1]
    assert _mismatches(got, want) == []


def test_compute_blob_kzg_proof_across_chunks(nmsm, setup, sms, pool):
    """two chunks, the second at a middle S, with invalid commitments and out-of-range elements in the second chunk at
    its first and last items and at the edges of a finish warp, and the identity as a valid commitment of a non-zero
    blob; then the verifier accepts every valid item"""
    n = CHUNK + 70
    assert 128 < F.chunk_lanes(n, sms)[-1] < 4096
    idx = pool.indices(n, offset=200)
    blobs = [pool.blobs[i] for i in idx]
    cs = [pool.commitments[i] for i in idx]
    c1, last = CHUNK, n - 1
    cs[c1] = C.off_curve_g1()
    cs[c1 + 32] = C.small_order_g1()
    cs[last - 1] = C.NON_CANONICAL_IDENTITY
    cs[c1 + 1] = C.uncompressed_flag(cs[c1 + 1])
    blobs[c1 + 1] = C.blob_with(blobs[c1 + 1], 0, R)
    blobs[c1 + 31] = C.blob_with(blobs[c1 + 31], 4095, R)
    blobs[c1 + 63] = C.blob_with(blobs[c1 + 63], 4095, (1 << 256) - 1)
    blobs[last] = C.blob_with(blobs[last], 4095, R)
    cs[3] = cs[c1 + 5] = C.IDENTITY
    want = [F.blob_proof(b, c) for b, c in zip(blobs, cs)]
    assert [k for k, w in enumerate(want) if w is None] == sorted(
        {c1, c1 + 1, c1 + 31, c1 + 32, c1 + 63, last - 1, last})
    got = setup.compute_blob_kzg_proof_batch(blobs, cs)
    assert _mismatches(got, want) == []
    honest = [k for k in range(n) if want[k] is not None and cs[k] == pool.commitments[idx[k]]]
    assert len(honest) == n - 9
    verdicts = nmsm.kzg_verify_blob_proof_batch([blobs[k] for k in honest], [cs[k] for k in honest],
                                                [got[k] for k in honest], C.SETUP)
    assert [k for k, v in zip(honest, verdicts) if not v] == []


def test_digit_edge_blobs_at_4096_and_128_lanes(setup, sms, pool):
    """commitments and proofs of the digit-edge blobs alone (S = 4096) and inside a full chunk (S = 128)"""
    edges = F.digit_edge_blobs()
    rnd = random.Random(91)
    ez = [rnd.randrange(R), 0, F.BRP[4095], F.BRP[128], rnd.randrange(R), rnd.randrange(R)]
    assert len(ez) == len(edges) and F.chunk_lanes(len(edges), sms) == [4096]
    assert _mismatches(setup.blob_to_kzg_commitment_batch(edges), [F.commitment(b) for b in edges]) == []
    assert _mismatches(setup.compute_kzg_proof_batch(edges, ez), [F.kzg_proof(b, z) for b, z in zip(edges, ez)]) == []

    assert F.chunk_lanes(CHUNK, sms) == [128]
    idx = pool.indices(CHUNK, offset=300)
    blobs = [pool.blobs[i] for i in idx]
    cs = [pool.commitments[i] for i in idx]
    zs = [F.BRP[k % 4096] for k in range(CHUNK)]  # on the domain: a cheap reference for the filler blobs
    for pos, b, z in zip((0, 31, 32, 500, CHUNK - 2, CHUNK - 1), edges, ez):
        blobs[pos], cs[pos], zs[pos] = b, F.commitment(b), z
    assert _mismatches(setup.blob_to_kzg_commitment_batch(blobs), cs) == []
    assert _mismatches(setup.compute_kzg_proof_batch(blobs, zs), [F.kzg_proof(b, z) for b, z in zip(blobs, zs)]) == []


def _collision_calls(S, n, pool):
    """calls of n blobs (so the comb runs at S lanes) holding every collision case of F.collisions(S): identities at
    items 0, 31 and n - 1, and for n >= 64 the whole finish warp 32 ... 63; when n < 64 one more call of 32 identities.
    The other items are the remaining cases, then distinct pool blobs.  [[(blob, expected commitment)]]"""
    cases = F.collisions(S)
    minus = itertools.cycle([(b, w) for b, _, w, _ in cases if w == C.IDENTITY])
    rest = [(b, w) for b, _, w, _ in cases]
    filler = ((pool.blobs[i], pool.commitments[i]) for i in itertools.cycle(range(len(pool.blobs))))
    ident = {0, 31, n - 1} | (set(range(32, 64)) if n >= 64 else set())
    calls = []
    while rest:
        calls.append([next(minus) if k in ident else rest.pop() if rest else next(filler) for k in range(n)])
    if n < 64:
        calls.append([next(minus) for _ in range(32)])
    return calls


def test_collisions_at_the_lane_count_of_the_call(setup, sms, pool):
    """two equal or opposite partial sums at every meeting distance of the comb, at each S the device reaches"""
    counts = F.regime_counts(sms)
    for S, n in sorted(counts.items()):
        for call in _collision_calls(S, n, pool):
            assert F.chunk_lanes(len(call), sms) == [S]
            got = setup.blob_to_kzg_commitment_batch([b for b, _ in call])
            assert _mismatches(got, [w for _, w in call]) == [], S
