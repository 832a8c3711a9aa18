"""The EIP-4844 prover's spec functions — TEST INFRASTRUCTURE ONLY, never imported by the product.

A line-by-line restatement of the consensus specs' Deneb polynomial-commitments.md prover (g1_lincomb,
blob_to_kzg_commitment, compute_quotient_eval_within_domain, compute_kzg_proof_impl, compute_kzg_proof,
compute_blob_kzg_proof) on the verifier oracle's integers (oracle/kzg_ref.py), and the test setup
KZG_SETUP_G1_LAGRANGE of a known tau.  Where the spec raises, these raise ValueError."""
from oracle import hash_to_g1_ref as H
from oracle import noble_fft
from oracle.kzg_ref import (BRP_ROOTS_OF_UNITY, FIELD_ELEMENTS_PER_BLOB, G1_GEN, ROOTS_OF_UNITY, blob_to_polynomial,
                            bytes_to_bls_field, compute_challenge, evaluate_polynomial_in_evaluation_form, g1_decode,
                            g1_mul, r)


def setup_g1_lagrange_scalars(tau: int):
    """L_i(tau) for the Lagrange basis over the natural-order domain omega^i (tau off the domain):
    L_i(tau) = (tau^N - 1) / N * omega^i / (tau - omega^i)"""
    n = FIELD_ELEMENTS_PER_BLOB
    c = (pow(tau, n, r) - 1) * pow(n, -1, r) % r
    return [c * w * pow(tau - w, -1, r) % r for w in ROOTS_OF_UNITY]


def setup_g1_lagrange(tau: int):
    """KZG_SETUP_G1_LAGRANGE of the test tau: the 4096 compressed points [L_i(tau)] G1 in natural order"""
    return [H.g1_encode(g1_mul(s, G1_GEN)) for s in setup_g1_lagrange_scalars(tau)]


# ---- the spec's prover (Deneb polynomial-commitments.md) over an explicit setup ---------------------------------------
def bit_reversal_permutation(sequence):
    return noble_fft.bit_reversal_permutation(list(sequence))


def g1_lincomb(points, scalars) -> bytes:
    """BLS multi-scalar multiplication over compressed points (plain sum of products; the spec's g1_lincomb)"""
    assert len(points) == len(scalars)
    result = None
    for x, a in zip(points, scalars):
        pt = g1_decode(x)
        if pt is not None and a % r:
            result = H.point_add(result, g1_mul(a, pt))
    return H.g1_encode(result)


def blob_to_kzg_commitment(blob: bytes, setup_g1_lagrange_points) -> bytes:
    return g1_lincomb(bit_reversal_permutation(setup_g1_lagrange_points), blob_to_polynomial(blob))


def compute_quotient_eval_within_domain(z: int, polynomial, y: int) -> int:
    """sum over omega_i != z of (f_i - y) omega_i / (z (z - omega_i))"""
    width = len(polynomial)
    roots_of_unity_brp = BRP_ROOTS_OF_UNITY
    result = 0
    for i in range(width):
        omega_i = roots_of_unity_brp[i]
        if omega_i == z:
            continue
        f_i = (polynomial[i] - y) % r
        numerator = f_i * omega_i % r
        denominator = z * (z - omega_i) % r
        result += numerator * pow(denominator, -1, r)
    return result % r


def compute_quotient(polynomial, z: int, y: int):
    """the quotient polynomial of compute_kzg_proof_impl in evaluation form"""
    roots_of_unity_brp = BRP_ROOTS_OF_UNITY
    polynomial_shifted = [(p - y) % r for p in polynomial]
    denominator_poly = [(x - z) % r for x in roots_of_unity_brp]
    quotient_polynomial = [0] * FIELD_ELEMENTS_PER_BLOB
    for i, (a, b) in enumerate(zip(polynomial_shifted, denominator_poly)):
        if b == 0:
            quotient_polynomial[i] = compute_quotient_eval_within_domain(roots_of_unity_brp[i], polynomial, y)
        else:
            quotient_polynomial[i] = a * pow(b, -1, r) % r
    return quotient_polynomial


def compute_kzg_proof_impl(polynomial, z: int, setup_g1_lagrange_points):
    """(proof, y)"""
    y = evaluate_polynomial_in_evaluation_form(polynomial, z)
    quotient_polynomial = compute_quotient(polynomial, z, y)
    return g1_lincomb(bit_reversal_permutation(setup_g1_lagrange_points), quotient_polynomial), y


def compute_kzg_proof(blob: bytes, z_bytes: bytes, setup_g1_lagrange_points):
    """(proof, y as 32 big-endian bytes); raises ValueError where the spec raises"""
    polynomial = blob_to_polynomial(blob)
    proof, y = compute_kzg_proof_impl(polynomial, bytes_to_bls_field(z_bytes), setup_g1_lagrange_points)
    return proof, y.to_bytes(32, "big")


def compute_blob_kzg_proof(blob: bytes, commitment_bytes: bytes, setup_g1_lagrange_points) -> bytes:
    """raises ValueError where the spec raises"""
    g1_decode(commitment_bytes)  # bytes_to_kzg_commitment: validate_kzg_g1
    polynomial = blob_to_polynomial(blob)
    evaluation_challenge = compute_challenge(blob, commitment_bytes)
    proof, _ = compute_kzg_proof_impl(polynomial, evaluation_challenge, setup_g1_lagrange_points)
    return proof
