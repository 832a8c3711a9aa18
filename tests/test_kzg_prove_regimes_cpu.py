"""The inputs and the fast reference of tests/test_gpu_kzg_prove_regimes.py, without a GPU: the reference agrees with
the spec oracle on commitments, proofs and y, and None exactly where the spec raises; the lane policy is the one the
tests target; each builder does what it claims, in scalars (the digit walk of every edge element, the equal or opposite
partial sums of every collision blob and the stage of the comb where they meet); and the host build of the comb
(kzg_lincomb_serial through tests/hostemu) gets the collisions right against the oracle."""
import random

import pytest

import kzg_cases as C
import kzg_prove_cases as P
import kzg_prove_fast_ref as F
from oracle import kzg_ref as K

R = K.BLS_MODULUS
LANE_COUNTS = (4096, 2048, 1024, 512, 256, 128)


# ---- the reference against the oracle --------------------------------------------------------------------------------
def _ref_blobs():
    blobs = [C.random_blob(60 + k) for k in range(6)] + [F.pool_blob(0)] + F.digit_edge_blobs()[:1]
    assert len(set(blobs)) == 8
    return blobs


@pytest.mark.parametrize("k", range(8))
def test_fast_reference_matches_the_oracle(k):
    """commitment and compute_kzg_proof at random z, z on the domain at indices 0, 1, 2048 and 4095, and z = 0"""
    blob = _ref_blobs()[k]
    assert F.commitment(blob) == K.commit_value(P.f_tau(blob))
    for name, z in P.z_cases(seed=70 + k):
        proof, y = P.expected_proof(blob, z)
        assert F.kzg_proof(blob, z) == (proof, C.be(y)), name


def test_fast_blob_proof_matches_the_oracle():
    """compute_blob_kzg_proof with the blob's own commitment and with the identity, which the spec accepts and
    hashes into the challenge like any other commitment"""
    for blob in _ref_blobs()[:2]:
        for c in (F.commitment(blob), C.IDENTITY):
            assert F.blob_proof(blob, c) == P.expected_proof(blob, K.compute_challenge(blob, c))[0]


def test_fast_reference_is_none_where_the_spec_raises():
    blob = C.random_blob(60)
    c = F.commitment(blob)
    for bad in (C.off_curve_g1(), C.small_order_g1(), C.NON_CANONICAL_IDENTITY, C.uncompressed_flag(c)):
        assert F.blob_proof(blob, bad) is None
    for z in (R, R + 1, (1 << 256) - 1):
        assert F.kzg_proof(blob, z) is None
    for index, value in ((0, R), (4095, R), (7, (1 << 256) - 1)):
        bad = C.blob_with(blob, index, value)
        assert F.commitment(bad) is None and F.kzg_proof(bad, 5) is None and F.blob_proof(bad, c) is None


# ---- the lane policy -------------------------------------------------------------------------------------------------
def test_lane_policy_on_a_132_sm_h100():
    want = {4096: (1, 32), 2048: (33, 65), 1024: (66, 131), 512: (132, 263), 256: (264, 527), 128: (528, 1024)}
    for S, (lo, hi) in want.items():
        assert {F.lincomb_lanes(n, 132) for n in range(lo, hi + 1)} == {S}
    assert F.regime_counts(132) == {S: hi for S, (_, hi) in want.items()}
    assert F.chunk_lanes(2 * 1024 + 264, 132) == [128, 128, 256]
    assert F.chunk_lanes(1025, 132) == [128, 4096]


# ---- the builders ----------------------------------------------------------------------------------------------------
def test_pool_blobs_are_distinct_and_in_range():
    blobs = [F.pool_blob(k) for k in range(F.POOL_SIZE)]
    assert len(set(blobs)) == F.POOL_SIZE > F.CHUNK
    tops = {b[k] for b in blobs[:8] for k in range(0, K.BYTES_PER_BLOB, 32)}
    assert tops == set(range(0x73))  # every top byte below r's
    assert all(max(F.elements(b)) < R for b in blobs[:50])


def test_digit_edges_cover_every_digit_with_and_without_carry():
    edges = F.digit_edge_elements()
    assert max(edges) < R
    seen = set()
    for e in edges:
        walk = F.signed_digits(e)
        assert sum(v << (8 * w) for w, (_, _, v) in enumerate(walk)) == e  # the walk is a signed-digit recoding
        assert all(-127 <= v <= 128 for _, _, v in walk)
        seen |= {(w, raw, cin) for w, (raw, cin, _) in enumerate(walk)}
    for w in range(F.LEVELS):
        for v in F.EDGE_DIGITS:
            for cin in ((0,) if w == 0 else (0, 1)):
                if (v << (8 * w)) < R:
                    assert (w, v, cin) in seen, (w, v, cin)
    # a run of 0xFF from level 0 carries into every level above it
    assert [cin for _, cin, _ in F.signed_digits((1 << 248) - 1)] == [0] + [1] * 31
    assert {1 << k for k in range(255)} | {(1 << k) - 1 for k in range(255)} <= set(edges)
    assert {R - 1, R - 2, (R - 1) // 2} <= set(edges)
    blobs = F.digit_edge_blobs()
    assert set(edges) <= set(F.elements(blobs[0]))
    assert all(max(F.elements(b)) < R for b in blobs)


def _lane_scalars(f, S):
    out = {}
    for p, v in f.items():
        out[p % S] = (out.get(p % S, 0) + v * F.LB[p]) % R
    return out


@pytest.mark.parametrize("S", LANE_COUNTS)
def test_collision_blobs_meet_where_they_claim(S):
    ds = F.collision_distances(S)
    assert {1, 2, 4, 8, 16, 32, 64} <= set(ds)
    assert [d for d in ds if 128 <= d < S][:1] == ([128] if S > 128 else []) and (S in ds) == (S < 4096)
    if S <= 1024:
        assert {d for d in ds if 128 <= d < S} == set(range(128, S, 128))
    cases = F.collisions(S)
    stages = set()
    for blob, el, want, stage in cases:
        (p1, f1), (p2, a) = sorted(el.items())
        d = p2 - p1
        assert F.elements(blob) == [el.get(p, 0) for p in range(4096)]
        assert 1 <= a <= 128 and F.signed_digits(a)[0] == (a, 0, a)  # a single digit: one table entry
        t1, t2 = f1 * F.LB[p1] % R, a * F.LB[p2] % R
        assert t1 in (t2, R - t2)
        if t1 == t2:
            assert want == K.commit_value(2 * t2) and F.f_tau(F.elements(blob)) == 2 * t2 % R
        else:
            assert want == C.IDENTITY and F.f_tau(F.elements(blob)) == 0
        if d < 32:
            assert stage == ("shuffle", d)
        elif d < 128:
            assert stage == ("shared", None)
        elif d < S:
            assert stage == ("finish", None) and d % 128 == 0
        else:
            assert d == S and stage == ("lane", S)
        if stage[0] == "lane":  # the lane's sum after p1 is +- the entry a P_p2 that its walk adds next
            assert _lane_scalars(el, S) == {p1 % S: (t1 + t2) % R}
        else:  # two lanes whose sums are equal or opposite, every other lane 0
            assert _lane_scalars(el, S) == {p1 % S: t1, p2 % S: t2}
        stages.add(stage[0] if stage[0] != "shuffle" else stage)
        assert F.meeting(p1, p2, S) == stage
    want_stages = {("shuffle", d) for d in (1, 2, 4, 8, 16)} | {"shared"}
    want_stages |= {"finish"} if S > 128 else set()
    want_stages |= {"lane"} if S < 4096 else set()
    assert stages == want_stages
    assert {w == C.IDENTITY for _, _, w, _ in cases} == {True, False}


@pytest.mark.parametrize("S", LANE_COUNTS)
def test_collision_expectations_match_the_fast_reference(S):
    for blob, _, want, _ in F.collisions(S)[::5]:
        assert F.commitment(blob) == want


def test_emu_lincomb_on_collisions():
    """the host comb (5 points, 4-bit digits) on two equal or opposite terms, in one lane's walk and across lanes"""
    rnd = random.Random(80)
    logs = [rnd.randrange(1, R) for _ in range(5)]
    points = [K.commit_value(s) for s in logs]
    rows, want = [], []
    for d in (1, 2, 4):
        for p1 in range(5 - d):
            for a in (1, 8, 5):  # single 4-bit digits: 8 is the table's largest entry
                for sign in (1, -1):
                    row = [0] * 5
                    row[p1 + d], row[p1] = a, sign * a * logs[p1 + d] * pow(logs[p1], -1, R) % R
                    rows.append(row)
                    want.append(K.commit_value(sum(v * s for v, s in zip(row, logs))))
    assert C.IDENTITY in want
    for lanes in (1, 2, 4):
        assert P.emu_lincomb(points, rows, lanes) == [(w, True) for w in want]
