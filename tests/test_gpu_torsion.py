"""Subgroup checks and the point kernels on the GPU on points of small and mixed order (torsion_cases.py), against
mul_any.  These are the inputs an attacker chooses: a point outside the prime-order subgroup that a subgroup check
accepts breaks soundness for everything built on it, and the torsion parts drive the kernels through their exceptional
branches (P = +-Q, identity table entries, warps whose results are all O, bucket sums that cancel)."""
import hashlib
import random

import pytest

import helpers as H
import torsion_cases as TC
from conftest import load_golden
from oracle import noble_ref as R

pytestmark = pytest.mark.gpu

NMSM_ERR_POINT = -3
MUL_IDS = [1, 3, 4, 5, 6, 7]
MSM_IDS = [1, 3, 6, 7]


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


def _unpack_all(name, out, infs, n):
    pb = len(out) // n
    return [(*H.unpack_point(name, out[i * pb:(i + 1) * pb]), infs[i]) for i in range(n)]


def _torsion_want(name):
    r = TC.r_of(name)
    return [1 if TC.mul_any(p, r).is0() else 0 for _, p, _ in TC.points(name)]


@pytest.mark.parametrize("cid", range(8))
def test_torsion_free_lists_and_ragged_tiles(nmsm, cid):
    """torsion_free_packed on the lists (r P == O by mul_any; ids 4 / 6 and 5 / 7 agree; ids 0 and 2 pass every
    on-curve point), then the lists tiled to a ragged size across warps and blocks, every flag checked."""
    name = TC.NAME_OF_ID[cid]
    pl = TC.points(name)
    want = _torsion_want(name)
    if cid in (0, 2):
        assert want == [1] * len(pl)
    pb = H.pack_points(name, [p for _, p, _ in pl])
    got = list(nmsm.torsion_free_packed(cid, pb, len(pl)))
    assert got == want, [(kind, q) for (kind, _, q), g, w in zip(pl, got, want) if g != w]
    other = {4: 6, 6: 4, 5: 7, 7: 5}.get(cid)
    if other is not None:
        assert list(nmsm.torsion_free_packed(other, pb, len(pl))) == got
    n = 100003 if "G2" not in name else (1 << 14) + 3
    reps = -(-n // len(pl))
    tiled = (pb * reps)[: n * (len(pb) // len(pl))]
    got = nmsm.torsion_free_packed(cid, tiled, n)
    assert list(got) == (want * reps)[:n]


@pytest.mark.parametrize("cid", range(8))
def test_torsion_free_reports_smallest_bad_index(nmsm, cid):
    """Out-of-range coordinates in two different blocks: NMSM_ERR_POINT with the smaller index, also when the smaller
    one is out of range only in the last coordinate part (y.c1 of a G2 point)."""
    name = TC.NAME_OF_ID[cid]
    pl = TC.points(name)
    n = 1500
    pb = bytearray((H.pack_points(name, [p for _, p, _ in pl]) * (n // len(pl) + 1))[: n * 2 * H.FP_BYTES[name]
                                                                                     * H.PARTS[name]])
    step = len(pb) // n
    fb = H.FP_BYTES[name]
    bad = R.CURVES[name].Fp.ORDER if H.PARTS[name] == 1 else R.CURVES[name].Fp.Fp.ORDER
    for lo, hi in ((300, 1100), (1100, 300)):
        b = bytearray(pb)
        b[lo * step + step - fb: (lo + 1) * step] = bad.to_bytes(fb, "little")  # last part of y only
        b[hi * step: hi * step + fb] = bad.to_bytes(fb, "little")               # first part of x
        with pytest.raises(ValueError, match="invalid point at index %d" % min(lo, hi)) as e:
            nmsm.torsion_free_packed(cid, bytes(b), n)
        assert e.value.__cause__.code == NMSM_ERR_POINT and e.value.__cause__.index == min(lo, hi)


def _mul_batch_case(name, rnd):
    """mul_cases(name) followed by aligned groups of 32 items: zero scalars (allow_zero), multiples of q on points of
    order q (all O), and ordinary results, so that both kernel forms see whole warps of identities next to warps of
    ordinary results."""
    cases = list(TC.mul_cases(name))
    cases += [(None, 0)] * (-len(cases) % 32)
    r = TC.r_of(name)
    small = TC.small_points(name)
    sub = [p for kind, p, _ in TC.points(name) if kind == "subgroup"]
    for j in range(4):
        cases += [(rnd.choice(sub + [T for T, _ in small]), 0) for _ in range(32)]
        T, q = small[j % len(small)]
        cases += [(T, q * rnd.randrange(1, r // q)) for _ in range(32)]
        cases += [(rnd.choice(sub), rnd.randrange(1, r)) for _ in range(32)]
    ident = R.CURVES[name].ZERO
    return [(p if p is not None else ident, k) for p, k in cases]


@pytest.mark.parametrize("form", ["quad", "serial"])
@pytest.mark.parametrize("cid", MUL_IDS)
def test_mul_batch_small_and_mixed_order(nmsm, cid, form, monkeypatch):
    """nmsm_mul_batch (independent of the subgroup for every id) on the lists with the scalars of scalars_for, in the
    quad form (one item per quad of lanes) and the serial form (NMSM_MUL_QUAD_MAX=0), then one batch above the quad
    threshold (132 SMs x 48 items on an H100)."""
    if form == "serial":
        monkeypatch.setenv("NMSM_MUL_QUAD_MAX", "0")
    name = TC.NAME_OF_ID[cid]
    cases = _mul_batch_case(name, random.Random("mul-%d" % cid))
    pb = H.pack_points(name, [p for p, _ in cases])
    sb = H.pack_scalars([k for _, k in cases])
    out, infs = nmsm.mul_batch_packed(cid, pb, sb, len(cases), True)
    got = _unpack_all(name, out, infs, len(cases))
    bad = [(i, hex(k)) for i, (p, k) in enumerate(cases) if got[i] != TC.expected(name, p, k)]
    assert not bad, bad[:8]
    if form == "quad":
        n = 132 * 48 + 77
        reps = -(-n // len(cases))
        out, infs = nmsm.mul_batch_packed(cid, (pb * reps)[: n * (len(pb) // len(cases))], (sb * reps)[: n * 32], n,
                                          True)
        assert _unpack_all(name, out, infs, n) == (got * reps)[:n]


@pytest.mark.parametrize("name", ["ed25519", "bls12_381_G1"])
def test_object_api_cofactor_helpers(nmsm, name):
    """Point.clearCofactor / isSmallOrder / isTorsionFree on the lists equal their definitions h P, h P == O and
    r P == O by mul_any; clearCofactor(P) passes the GPU subgroup check."""
    C = nmsm.CURVES[name]
    h, r = TC.COFACTOR[name], TC.r_of(name)
    cleared = []
    for kind, p, q in TC.points(name):
        cp = C.fromAffine(p.toAffine())
        hp = TC.expected(name, p, h)
        cc = cp.clearCofactor()
        assert (cc.x, cc.y, 1 if cc.is0() else 0) == hp, (kind, q)
        assert cp.isSmallOrder() == bool(hp[2]), (kind, q)
        assert cp.isTorsionFree() == bool(TC.expected(name, p, r)[2]), (kind, q)
        assert cc.isTorsionFree(), (kind, q)
        cleared.append(cc.to_packed())
    cid = {"ed25519": 1, "bls12_381_G1": 6}[name]
    assert set(nmsm.torsion_free_packed(cid, b"".join(cleared), len(cleared))) == {1}


@pytest.mark.parametrize("cid", MUL_IDS)
def test_point_table_small_order_base(nmsm, cid):
    """nmsm_point_table_* with a small-order base (identity entries at digits d = 0 mod q, and for ed25519 every level
    j >= 1 once 2^16 T = O), a mixed base and a base outside the subgroup of large order, with scalars whose 16-bit
    digits land on those entries.  table_base_body / table_mul_body only add the prepared point itself (the
    endomorphism image k_prepare stores next to it is never read), so ids 4 and 5 take the same points."""
    name = TC.NAME_OF_ID[cid]
    rnd = random.Random("gpu-table-%d" % cid)
    pl = TC.points(name)
    small = TC.small_points(name)
    bases = small[:2] + [(p, q) for kind, p, q in pl if kind == "mixed"][:1]
    bases += [(p, 0) for kind, p, _ in pl if kind == "random"][:1]
    for base, q in bases:
        ks = TC.table_scalars(name, q if q > 1 else 3, 16, rnd, count=10) + [0]
        tbl = nmsm.PointTable(cid, H.point_bytes(name, base))
        try:
            out, infs = tbl.mul_batch(H.pack_scalars(ks), len(ks), True)
        finally:
            tbl.close()
        got = _unpack_all(name, out, infs, len(ks))
        for k, g in zip(ks, got):
            assert g == TC.expected(name, base, k), (q, hex(k))


@pytest.mark.parametrize("cid", MSM_IDS)
def test_msm_and_fixed_base_small_and_mixed_order(nmsm, cid):
    """MSMs and fixed-base point sets (ids 1, 3, 6, 7; ids 4 and 5 exclude such points by contract) on mixed sets,
    sets whose torsion parts cancel and all-small-order sets summing to O, over the window sizes 2, 3, 5, 8, 13."""
    name = TC.NAME_OF_ID[cid]
    try:
        for label, pts, sc in TC.msm_sets(name):
            want = TC.expected_sum(name, pts, sc)
            pb, sb = H.pack_points(name, pts), H.pack_scalars(sc)
            for c in (0, 2, 3, 5, 8, 13):
                nmsm.set_window_bits(c)
                out, inf = nmsm.msm_packed(cid, pb, sb, len(pts))
                assert (*H.unpack_point(name, out), inf) == want, (label, c)
            nmsm.set_window_bits(0)
            for c in (0, 4, 8, 13):
                ps = nmsm.PointSet(cid, pb, len(pts))
                try:
                    ps.precompute(c)
                    out, inf = ps.msm(sb, len(pts))
                finally:
                    ps.close()
                assert (*H.unpack_point(name, out), inf) == want, (label, "table", c)
    finally:
        nmsm.set_window_bits(0)


def test_msm_ed25519_large_tiled(nmsm):
    """2^16 + 1 terms on ed25519 tiled from the mixed, small-order and random points: expected
    sum_j (sum_{i: P_i = P_j} s_i) P_j with the inner sum taken as an integer."""
    name = "ed25519"
    pl = [p for _, p, _ in TC.points(name)]
    n = (1 << 16) + 1
    rnd = random.Random(65537)
    r = TC.r_of(name)
    pts = [pl[i % len(pl)] for i in range(n)]
    sc = [rnd.randrange(r) for _ in range(n)]
    want = TC.expected_sum(name, pts, sc)
    pb = b"".join(H.point_bytes(name, p) for p in pl)
    step = len(pb) // len(pl)
    pbig = b"".join(pb[(i % len(pl)) * step:(i % len(pl) + 1) * step] for i in range(n))
    out, inf = nmsm.msm_packed(1, pbig, H.pack_scalars(sc), n)
    assert (*H.unpack_point(name, out), inf) == want
    ps = nmsm.PointSet(1, pbig, n)
    try:
        ps.precompute(0)
        out, inf = ps.msm(H.pack_scalars(sc), n)
    finally:
        ps.close()
    assert (*H.unpack_point(name, out), inf) == want


def _ed_sign_with_torsion(rnd, T_R, T_A, msg):
    """R = rB + T_R, A = aB + T_A, s = r + k a mod l with k = SHA-512(R || A || M): cofactored verification accepts."""
    ED = R.CURVES["ed25519"]
    ell = ED.Fn.ORDER
    a, rr = rnd.randrange(1, ell), rnd.randrange(1, ell)
    Rp = ED.BASE.multiply(rr).add(T_R)
    Ap = ED.BASE.multiply(a).add(T_A)
    rb, ab = Rp.toBytes(), Ap.toBytes()
    k = int.from_bytes(hashlib.sha512(rb + ab + msg).digest(), "little") % ell
    s = (rr + k * a) % ell
    return rb + s.to_bytes(32, "little"), ab


def test_ed25519_batch_verify_with_torsion_components(nmsm):
    """Signatures whose R and A carry torsion components of order 2, 4 and 8: the reference's cofactored verify
    accepts each; batches of 1, 33 and 4097 mixed with plain signatures accept; one wrong s at index 0, 31, 32 or the
    last gives False with bad_index -1; an undecodable R gives its index."""
    rnd = random.Random(25519)
    ED = R.CURVES["ed25519"]
    ell = ED.Fn.ORDER
    small = [T for T, _ in TC.small_points("ed25519")] + [ED.ZERO]
    tors = []
    for i in range(24):
        msg = bytes([i]) * (i % 7)
        sig, pk = _ed_sign_with_torsion(rnd, small[i % len(small)], small[(3 * i + 1) % len(small)], msg)
        assert R.ed25519_verify(sig, msg, pk)
        tors.append((sig, msg, pk))
    plain = [(bytes.fromhex(v["sig"]), bytes.fromhex(v["msg"]), bytes.fromhex(v["pk"]))
             for v in load_golden("ed25519.json")["vectors"][:40]]
    mixed = [x for pair in zip(tors, plain) for x in pair] + plain[len(tors):]

    def run(items, seed):
        z = random.Random(seed).randbytes(16 * len(items))
        return nmsm.ed25519_verify_batch([s for s, _, _ in items], [m for _, m, _ in items], [p for _, _, p in items], z)

    for sig, msg, pk in tors:
        assert run([(sig, msg, pk)], 1) == (True, -1)
    for n in (1, 33, 4097):
        items = [mixed[i % len(mixed)] for i in range(n)]
        assert run(items, n) == (True, -1), n
    items = [mixed[i % len(mixed)] for i in range(4097)]
    for idx in (0, 31, 32, 4096):
        bad = list(items)
        sig, msg, pk = bad[idx]
        s = (int.from_bytes(sig[32:], "little") + 1) % ell
        bad[idx] = (sig[:32] + s.to_bytes(32, "little"), msg, pk)
        assert not R.ed25519_verify(*bad[idx])
        assert run(bad, idx) == (False, -1), idx
    y = next(y for y in range(2, 100) if _undecodable(y))
    for idx in (0, 33, 4096):
        bad = list(items)
        sig, msg, pk = bad[idx]
        bad[idx] = (y.to_bytes(32, "little") + sig[32:], msg, pk)
        assert run(bad, idx) == (False, idx), idx


def _undecodable(y):
    try:
        R.ed25519_point_from_bytes(y.to_bytes(32, "little"), True)
        return False
    except ValueError:
        return True
