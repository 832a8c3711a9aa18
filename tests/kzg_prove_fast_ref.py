"""A fast exact reference of the EIP-4844 prover under the seeded tau, and the inputs of the prover's regime tests
(tests/test_gpu_kzg_prove_regimes.py).

The reference uses what a test knows and a prover does not: tau.  A commitment is [f(tau)] G1 with
f(tau) = sum_p f_p L_brp(p)(tau), a proof is [(f(tau) - y) / (tau - z)] G1, and y = f(z) takes the barycentric formula
with one batched inversion.  That is about 5 ms per item instead of the spec oracle's 50 ms per f(z) evaluation, and
test_kzg_prove_regimes_cpu.py checks it against the oracle (kzg_prove_cases.expected_proof, f_tau, kzg_ref.commit_value).

The inputs, all seeded:
  - a pool of distinct random blobs (POOL_SIZE > KZG_CHUNK, so no chunk holds a blob twice);
  - digit-edge elements: every 8-bit digit value the comb's signed walk treats specially, with and without a carry in,
    at every level, runs of 0xFF that carry through every level, 2^k, 2^k - 1, r - 1, r - 2 and (r - 1) / 2;
  - collision blobs: two non-zero elements whose partial sums in k_kzg_lincomb are equal (the addition doubles) or
    opposite (the commitment of a non-zero blob is the identity), placed so that the kernel first adds them at a chosen
    stage: the shuffle tree, shared memory, k_kzg_lincomb_finish's partials, or one lane's sequential walk."""
import random

import numpy as np

import kzg_cases as C
from oracle import kzg_ref as K
import kzg_prove_ref as KP

R = K.BLS_MODULUS
N = K.FIELD_ELEMENTS_PER_BLOB
BRP = K.BRP_ROOTS_OF_UNITY
BRP_INDEX = {w: i for i, w in enumerate(BRP)}
CHUNK = 1024  # blobs per upload and comb launch of the prover (KZG_CHUNK in inst_kzg.cu)
COMB_BITS = 8  # digit width of the setup table (KZG_COMB_BITS in kzg.cuh)
LEVELS = 32  # digits per scalar: point_table_levels<KzgCv, 8>() = ceil(256 / 8)
# LB[p] = L_brp(p)(tau): the discrete log of point p of the comb's table, which is in bit-reversed order
LB = KP.bit_reversal_permutation(KP.setup_g1_lagrange_scalars(C.TAU))
_INV_N = pow(N, -1, R)


# ---- the lane policy of the comb -------------------------------------------------------------------------------------
def lincomb_lanes(cnt: int, sms: int) -> int:
    """S, the lanes per blob of k_kzg_lincomb for a chunk of cnt blobs on a device of `sms` SMs: halved from 4096 while
    cnt * S / 2 >= 512 * sms.  A restatement of kzg_lincomb_lanes in inst_kzg.cu; if that policy changes, the expected
    values of the tests stay right and only the choice of which S each call reaches weakens."""
    S = N
    while S > 1 and cnt * (S // 2) >= 512 * sms:
        S //= 2
    return S


def chunk_lanes(n: int, sms: int):
    """S of each chunk of a call over n blobs"""
    return [lincomb_lanes(min(CHUNK, n - c0), sms) for c0 in range(0, n, CHUNK)]


def regime_counts(sms: int):
    """{S: the largest chunk size with that S} over every S that chunks of 1 ... KZG_CHUNK blobs reach"""
    out = {}
    for cnt in range(1, CHUNK + 1):
        out[lincomb_lanes(cnt, sms)] = cnt
    return out


# ---- the reference -----------------------------------------------------------------------------------------------------
def elements(blob: bytes):
    return [int.from_bytes(blob[k:k + 32], "big") for k in range(0, K.BYTES_PER_BLOB, 32)]


def f_tau(f) -> int:
    """sum_p f_p L_brp(p)(tau): the discrete log of blob_to_kzg_commitment (kzg_prove_cases.lincomb_scalar)"""
    return sum(a * b for a, b in zip(f, LB)) % R


def evaluate(f, z: int) -> int:
    """f(z) for the polynomial in evaluation form over the bit-reversed domain (0 <= z < r): the element itself when z
    is on the domain, else (z^N - 1) / N sum_i f_i w_i / (z - w_i) with one inversion (Montgomery's trick)"""
    i = BRP_INDEX.get(z)
    if i is not None:
        return f[i]
    d = [(z - w) % R for w in BRP]
    pre, acc = [0] * N, 1
    for k in range(N):
        pre[k] = acc
        acc = acc * d[k] % R
    inv, s = pow(acc, -1, R), 0  # inv = 1 / (d_0 ... d_k) going down
    for k in range(N - 1, -1, -1):
        s += f[k] * BRP[k] % R * (inv * pre[k] % R)
        inv = inv * d[k] % R
    return s % R * (pow(z, N, R) - 1) % R * _INV_N % R


def commitment(blob: bytes):
    """blob_to_kzg_commitment, None where the spec raises (an element >= r)"""
    f = elements(blob)
    if max(f) >= R:
        return None
    return K.commit_value(f_tau(f))


def _open(f, z: int):
    y = evaluate(f, z)
    return K.prove_value(f_tau(f), z, y, C.TAU), y


def kzg_proof(blob: bytes, z: int):
    """compute_kzg_proof: (proof, y as 32 big-endian bytes), None where the spec raises (z or an element >= r)"""
    f = elements(blob)
    if z >= R or max(f) >= R:
        return None
    proof, y = _open(f, z)
    return proof, C.be(y)


def blob_proof(blob: bytes, commitment48: bytes):
    """compute_blob_kzg_proof, None where the spec raises (a commitment that fails validate_kzg_g1, an element >= r).
    The challenge hashes the commitment given, which need not be the blob's."""
    try:
        K.g1_decode(commitment48)
    except ValueError:
        return None
    f = elements(blob)
    if max(f) >= R:
        return None
    return _open(f, K.compute_challenge(blob, commitment48))[0]


# ---- distinct random blobs -------------------------------------------------------------------------------------------
POOL_SIZE = 1100


def pool_blob(k: int) -> bytes:
    """distinct random blob k of the pool: uniform bytes with the top byte of each element folded below 0x73, so every
    element is < r (r = 0x73ed...) and its top digit takes every value below r's"""
    a = np.frombuffer(random.Random(100_000 + k).randbytes(K.BYTES_PER_BLOB), np.uint8).reshape(N, 32).copy()
    top = a[:, 0] & 0x7F
    top[top >= 0x73] -= 0x40
    a[:, 0] = top
    return a.tobytes()


class Pool:
    """POOL_SIZE distinct blobs with their commitments, computed once; item k of a call is pool[(offset + k) % size]"""

    def __init__(self, size: int = POOL_SIZE):
        self.blobs = [pool_blob(k) for k in range(size)]
        self.commitments = [K.commit_value(f_tau(elements(b))) for b in self.blobs]

    def indices(self, n: int, offset: int = 0):
        return [(offset + k) % len(self.blobs) for k in range(n)]


# ---- digit-edge elements ---------------------------------------------------------------------------------------------
EDGE_DIGITS = (0, 1, 127, 128, 129, 255)


def signed_digits(s: int):
    """[(raw digit, carry in, signed digit)] of table_walk_acc's walk over s (msm_body.cuh), level 0 first"""
    out, carry = [], 0
    for w in range(LEVELS):
        raw = (s >> (COMB_BITS * w)) & 0xFF
        v, cin = raw + carry, carry
        carry = 0
        if v > 128:
            v, carry = v - 256, 1
        out.append((raw, cin, v))
    return out


def digit_edge_elements():
    """elements < r: each EDGE_DIGITS value at each level with no carry in (the level below holds 5) and with a carry in
    (the level below holds 200), runs of 0xFF from every level up to the top, 2^k and 2^k - 1 for k < 255, r - 1,
    r - 2 and (r - 1) / 2"""
    out = []
    for w in range(LEVELS):
        for v in EDGE_DIGITS:
            for below in ((None,) if w == 0 else (5, 200)):
                e = v << (COMB_BITS * w)
                if below is not None:
                    e |= below << (COMB_BITS * (w - 1))
                if e < R:
                    out.append(e)
    top = 0x72 << (COMB_BITS * (LEVELS - 1))  # the largest top digit below r's 0x73 under a run of 0xFF
    for lo in range(LEVELS - 1):
        run = (1 << (COMB_BITS * (LEVELS - 1))) - (1 << (COMB_BITS * lo))  # 0xFF at levels lo ... 30
        out += [run, top | run, top | run | 0x80]
    for k in range(255):
        out += [1 << k, (1 << k) - 1]
    out += [R - 1, R - 2, (R - 1) // 2]
    return out


def digit_edge_blobs():
    """blobs of digit-edge elements: four that lay the list out over every position at different offsets and strides,
    every element r - 1 (f(tau) = -1, since sum_p L_p = 1), and every element a run of 0xFF from level 0"""
    edges = digit_edge_elements()
    m = len(edges)
    blobs = [b"".join(C.be(edges[(off + stride * p) % m]) for p in range(N))
             for off, stride in ((0, 1), (17, 1), (5, 7), (m // 2, 13))]
    blobs.append(C.be(R - 1) * N)
    blobs.append(C.be((0x72 << 248) | ((1 << 248) - 1)) * N)
    return blobs


# ---- collision blobs -------------------------------------------------------------------------------------------------
def meeting(p1: int, p2: int, S: int):
    """where k_kzg_lincomb and k_kzg_lincomb_finish first add the partial sums of points p1 < p2 when no other element
    is non-zero: ("lane", S) the sequential walk of one lane, ("shuffle", d) the warp shuffle tree's step d,
    ("shared", None) the block's warp partials, ("finish", None) the per-blob block partials"""
    t1, t2 = p1 % S, p2 % S
    if t1 == t2:
        return "lane", S
    W = min(S, 32)
    if t1 // W == t2 // W:
        # after the step of shift d, lane k < d holds the lanes = k mod d: two lanes first share a sum at the largest
        # power of two that divides their distance
        x = abs(t2 - t1)
        return "shuffle", x & -x
    if t1 // 128 == t2 // 128:
        return "shared", None
    return "finish", None


def collision_distances(S: int):
    """the distances d = p2 - p1 at which two lanes' sums meet at each stage of the comb at S lanes: 1 ... 16 in the
    shuffle tree, 32 and 64 in shared memory, multiples of 128 below S between block partials (all of them up to 1024,
    then the powers of two, 384 and S - 128), and S itself, one lane's two points, when S < 4096"""
    ds = [1, 2, 4, 8, 16, 32, 64]
    mult = [128 * k for k in range(1, S // 128)]
    ds += mult if S <= 1024 else sorted({d for d in mult if d & (d - 1) == 0} | {384, S - 128})
    if S < N:
        ds.append(S)
    return ds


def collision_first_point(d: int, S: int, rnd):
    """a p1 such that p1 and p1 + d meet at the stage that collision_distances assigns to d: within one warp's lanes
    for d < 32, one block's for d < 128, one blob's for d < S, any lane for d = S"""
    span = 32 if d < 32 else 128 if d < 128 else S if d < S else N
    base = rnd.randrange(0, (N - d) // span) * span if span < N else 0
    return base + rnd.randrange(0, span - d) if d < span else rnd.randrange(0, N - d)


def collision_elements(p1: int, d: int, a: int, sign: int):
    """{p1: sign a L_brp(p2)(tau) / L_brp(p1)(tau), p2: a}, p2 = p1 + d: the two points' terms are equal (sign 1) or
    opposite (sign -1), and with a single digit a <= 128 the second term is a table entry itself"""
    p2 = p1 + d
    return {p1: sign * a * LB[p2] * pow(LB[p1], -1, R) % R, p2: a}


def blob_of(elems) -> bytes:
    f = bytearray(K.BYTES_PER_BLOB)
    for p, v in elems.items():
        f[32 * p:32 * p + 32] = C.be(v)
    return bytes(f)


def collisions(S: int, seed: int = 0):
    """[(blob, elements, expected commitment, meeting stage)] for a call at S lanes: every collision distance, both signs,
    a in (1, 128) and one random single digit"""
    rnd = random.Random(seed * 8191 + S)
    out = []
    for d in collision_distances(S):
        for a in (1, 128, rnd.randrange(2, 128)):
            for sign in (1, -1):
                p1 = collision_first_point(d, S, rnd)
                el = collision_elements(p1, d, a, sign)
                want = C.IDENTITY if sign < 0 else K.commit_value(2 * a * LB[p1 + d] % R)
                out.append((blob_of(el), el, want, meeting(p1, p1 + d, S)))
    return out
