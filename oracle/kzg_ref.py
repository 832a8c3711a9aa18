"""EIP-4844 KZG proof verification oracle — TEST INFRASTRUCTURE ONLY, never imported by the product.

A line-by-line restatement of the consensus specs' Deneb polynomial-commitments.md functions the library batches
(compute_challenge, evaluate_polynomial_in_evaluation_form, validate_kzg_g1, verify_kzg_proof_impl, verify_kzg_proof,
verify_blob_kzg_proof) and of the EIP-4844 point-evaluation precompile, on the plain-integer G1 arithmetic of
oracle/hash_to_g1_ref.py, the G2 points of oracle/noble_ref.py and the pairing of oracle/bls_pairing_ref.py.  Where the
spec raises on malformed input, these return False (the library's verdict).

The trusted setup is a parameter: `setup_g2(tau)` makes [tau] G2 for a test tau, and `commit` / `prove` are a test-only
prover with that known tau (commitment [f(tau)] G1 with f(tau) by the same barycentric formula, proof
[(f(tau) - y) / (tau - z)] G1), which needs no Lagrange setup."""
from __future__ import annotations

import hashlib

from oracle import bls_pairing_ref as B
from oracle import hash_to_g1_ref as H
from oracle import noble_fft

BLS_MODULUS = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
FIELD_ELEMENTS_PER_BLOB = 4096
BYTES_PER_FIELD_ELEMENT = 32
BYTES_PER_BLOB = BYTES_PER_FIELD_ELEMENT * FIELD_ELEMENTS_PER_BLOB
FIAT_SHAMIR_PROTOCOL_DOMAIN = b"FSBLOBVERIFY_V1_"
PRIMITIVE_ROOT_OF_UNITY = 7
VERSIONED_HASH_VERSION_KZG = b"\x01"
G1_POINT_AT_INFINITY = b"\xc0" + bytes(47)
r = BLS_MODULUS


def compute_roots_of_unity(order: int):
    """[omega^i for i < order], omega = 7^((r - 1) / order)"""
    assert (r - 1) % order == 0
    omega = pow(PRIMITIVE_ROOT_OF_UNITY, (r - 1) // order, r)
    out, cur = [], 1
    for _ in range(order):
        out.append(cur)
        cur = cur * omega % r
    return out


ROOTS_OF_UNITY = compute_roots_of_unity(FIELD_ELEMENTS_PER_BLOB)
BRP_ROOTS_OF_UNITY = noble_fft.bit_reversal_permutation(ROOTS_OF_UNITY)


def bytes_to_bls_field(b: bytes) -> int:
    """raises (here: ValueError) for a value >= r"""
    v = int.from_bytes(b, "big")
    if v >= r:
        raise ValueError("field element out of range")
    return v


def hash_to_bls_field(data: bytes) -> int:
    return int.from_bytes(hashlib.sha256(data).digest(), "big") % r


def blob_to_polynomial(blob: bytes):
    if len(blob) != BYTES_PER_BLOB:
        raise ValueError("blob length")
    return [bytes_to_bls_field(blob[32 * i:32 * i + 32]) for i in range(FIELD_ELEMENTS_PER_BLOB)]


def challenge_transcript(blob: bytes, commitment: bytes) -> bytes:
    degree_poly = FIELD_ELEMENTS_PER_BLOB.to_bytes(16, "big")
    return FIAT_SHAMIR_PROTOCOL_DOMAIN + degree_poly + blob + commitment


def compute_challenge(blob: bytes, commitment: bytes) -> int:
    return hash_to_bls_field(challenge_transcript(blob, commitment))


def evaluate_polynomial_in_evaluation_form(polynomial, z: int) -> int:
    width = len(polynomial)
    assert width == FIELD_ELEMENTS_PER_BLOB
    inverse_width = pow(width, -1, r)
    roots_of_unity_brp = BRP_ROOTS_OF_UNITY
    if z in roots_of_unity_brp:
        return polynomial[roots_of_unity_brp.index(z)]
    result = 0
    for i in range(width):
        a = polynomial[i] * roots_of_unity_brp[i] % r
        b = (z - roots_of_unity_brp[i]) % r
        result += a * pow(b, -1, r)
    return result * (pow(z, width, r) - 1) * inverse_width % r


# ---- G1 / G2 ------------------------------------------------------------------------------------------------------
def g1_decode(b: bytes):
    """validate_kzg_g1 and decompression: the affine point, None for the identity; ValueError when rejected"""
    if len(b) != 48:
        raise ValueError("G1 length")
    if b == G1_POINT_AT_INFINITY:
        return None
    x, y = B.R.bls12_381_g1_decode(b)  # compressed-only: a 48-byte input with the uncompressed flag fails its length
    if (x, y) == (0, 0) or not H.in_g1((x, y)):
        raise ValueError("not a point of G1")
    return x, y


def g1_mul(k: int, pt):
    return H.scalar_mul(k % r, pt)


G1_GEN = B.affine(B.G1.BASE)


def setup_g2_point(tau: int):
    return B.G2.BASE.multiply(tau % r)


def setup_g2(tau: int) -> bytes:
    """[tau] G2, 96-byte compressed (the role of KZG_SETUP_G2_MONOMIAL[1])"""
    return B.g2_encode(setup_g2_point(tau))


def verify_kzg_proof_impl(commitment, z: int, y: int, proof, setup_g2_pt) -> bool:
    """e(P - y G1, -G2) e(proof, [tau] G2 - z G2) == 1 with the G2 points of the spec (the library computes it through
    Q = P - y G1 + z proof; this states the spec's form)"""
    X_minus_z = setup_g2_pt.add(B.G2.BASE.multiply(z).negate()) if z % r else setup_g2_pt
    P_minus_y = H.point_add(commitment, H.point_neg(g1_mul(y, G1_GEN)))
    neg_g2 = B.affine(B.G2.BASE.negate())
    x_minus_z = (B.Z2, B.Z2) if X_minus_z.is0() else B.affine(X_minus_z)
    pairs = [(P_minus_y or (0, 0), neg_g2), (proof or (0, 0), x_minus_z)]
    return B.pairing_check(pairs)


def verify_kzg_proof(commitment_bytes: bytes, z_bytes: bytes, y_bytes: bytes, proof_bytes: bytes, setup: bytes) -> bool:
    try:
        commitment = g1_decode(commitment_bytes)
        proof = g1_decode(proof_bytes)
        z, y = bytes_to_bls_field(z_bytes), bytes_to_bls_field(y_bytes)
    except ValueError:
        return False
    return verify_kzg_proof_impl(commitment, z, y, proof, setup_point(setup))


def verify_blob_kzg_proof(blob: bytes, commitment_bytes: bytes, proof_bytes: bytes, setup: bytes) -> bool:
    try:
        commitment = g1_decode(commitment_bytes)
        polynomial = blob_to_polynomial(blob)
        proof = g1_decode(proof_bytes)
    except ValueError:
        return False
    z = compute_challenge(blob, commitment_bytes)
    y = evaluate_polynomial_in_evaluation_form(polynomial, z)
    return verify_kzg_proof_impl(commitment, z, y, proof, setup_point(setup))


def setup_point(setup: bytes):
    x, y = B.R.bls12_381_g2_decode(setup)
    return B.G2.fromAffine({"x": x, "y": y})


def kzg_to_versioned_hash(commitment: bytes) -> bytes:
    return VERSIONED_HASH_VERSION_KZG + hashlib.sha256(commitment).digest()[1:]


def point_evaluation_precompile(data: bytes, setup: bytes):
    """EIP-4844 point_evaluation_precompile: the 64 output bytes, or None where it fails"""
    if len(data) != 192:
        return None
    versioned_hash, z, y, commitment, proof = data[:32], data[32:64], data[64:96], data[96:144], data[144:192]
    if kzg_to_versioned_hash(commitment) != versioned_hash:
        return None
    if not verify_kzg_proof(commitment, z, y, proof, setup):
        return None
    return FIELD_ELEMENTS_PER_BLOB.to_bytes(32, "big") + BLS_MODULUS.to_bytes(32, "big")


# ---- a test-only prover with a known tau --------------------------------------------------------------------------
def commit_value(f_tau: int) -> bytes:
    return H.g1_encode(g1_mul(f_tau, G1_GEN))


def prove_value(f_tau: int, z: int, y: int, tau: int) -> bytes:
    """[(f(tau) - y) / (tau - z)] G1 (tau != z)"""
    return H.g1_encode(g1_mul((f_tau - y) * pow(tau - z, -1, r), G1_GEN))


def blob_commit_and_prove(blob: bytes, tau: int):
    """(commitment, proof, z, y) for the blob's polynomial under the test tau"""
    poly = blob_to_polynomial(blob)
    f_tau = evaluate_polynomial_in_evaluation_form(poly, tau)
    commitment = commit_value(f_tau)
    z = compute_challenge(blob, commitment)
    y = evaluate_polynomial_in_evaluation_form(poly, z)
    return commitment, prove_value(f_tau, z, y, tau), z, y
