"""BLS12-381 aggregate verification in Python integers: the contract of include/nmsm.h
nmsm_bls12_381_aggregate_verify_batch, one check at a time.  It covers Ethereum's FastAggregateVerify (one group) and
noble's bls.verifyBatch(signature, messages, publicKeys) (abstract/bls.ts: keys of pairs with equal messages summed).

Built on bls_pairing_ref (decode, torsion_free, pairing_check) and hash_to_curve_ref (hash_to_g2).  Keys are affine G1
tuples that the caller has decoded and subgroup-checked; (0, 0) is the identity.  They are not subgroup-checked here,
so a key outside G1 gives whatever the group law and the pairing give."""
import functools

from oracle import bls_pairing_ref as B
from oracle import hash_to_curve_ref as H
from oracle import noble_ref as R

G1, G2 = B.G1, B.G2


@functools.lru_cache(maxsize=None)
def hashed(msg: bytes, dst: bytes):
    """H(m) as an affine G2 tuple ((x0, x1), (y0, y1)), the identity as B.ID2-style zeros"""
    pt = H.hash_to_g2(bytes(msg), bytes(dst))
    return ((0, 0), (0, 0)) if pt is None else pt


def key_sum(keys):
    """sum of affine G1 keys by the group law (a repeated key doubles, P + (-P) is the identity)"""
    s = G1.ZERO
    for k in keys:
        if not B.is_identity_g1(k):
            s = s.add(G1.fromAffine({"x": k[0], "y": k[1]}))
    return s


def aggregate_verify(sig96: bytes, groups, dst: bytes) -> bool:
    """groups: [(message bytes, [affine G1 keys])].  True iff
    1. the signature decodes, is not the identity and lies in G2 (the rules of bls_pairing_ref.bls_verify);
    2. there is at least one group, and every group has at least one key;
    3. no key is the identity;
    4. no group's key sum S_g is the identity;
    5. e(-G1, sig) prod_g e(S_g, H(m_g)) == 1."""
    try:
        sig = R.bls12_381_g2_decode(sig96)
    except ValueError:
        return False
    if len(sig96) != 96 or B.is_identity_g2(sig) or not B.torsion_free(G2.fromAffine({"x": sig[0], "y": sig[1]})):
        return False
    if not groups or any(len(keys) == 0 for _, keys in groups):
        return False
    if any(B.is_identity_g1(k) for _, keys in groups for k in keys):
        return False
    pairs = []
    for msg, keys in groups:
        s = key_sum(keys)
        if s.is0():
            return False
        pairs.append((B.affine(s), hashed(msg, dst)))
    pairs.append((B.affine(G1.BASE.negate()), sig))
    return B.pairing_check(pairs)
