"""The device arithmetic on the GPU, bit for bit: tests/devemu runs the parts every kernel is built from (the eight
Montgomery fields, the double-width pieces of the lazy reduction, Fp2, both Fp12 towers and pairings, the serial and
lane-parallel group law, warp_batch_inverse) one case per thread, quad or warp, on arith_cases' carry-edge inputs.

Each result is compared with Python integers or the oracles, and the same input words are given to tests/hostemu, the
g++ build of the same headers with an emulated carry flag that the CPU suite relies on: equal words there confirm that
model on the hardware.  The field and Fp2 parts run in both builds: with the product's out-of-line multiplications
(-DNMSM_MUL_NOINLINE, mul_call / sqr_call / fp2_mul_call) and inlined (`make EXTRA=`)."""
import ctypes
import random

import numpy as np
import pytest

import arith_cases as A
import helpers as H
from oracle import noble_ref as R

pytestmark = pytest.mark.gpu

VARIANTS = ["", "_inl"]  # dev_* entry points of the NMSM_MUL_NOINLINE build and of the inlined build


@pytest.fixture(scope="module")
def dev():
    return H.devemu()


def _arr(ws):
    return np.ascontiguousarray(np.array(ws, np.uint32))


def _cp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _run(fn, *ints_args, bufs, out_words):
    """call fn(*ints_args, *bufs, out) with uint32 buffers; returns the output words"""
    out = np.zeros(max(out_words, 1), np.uint32)
    rc = fn(*ints_args, *[_cp(b) for b in bufs], _cp(out))
    assert rc == 0, "device call failed: cudaError_t %d" % rc
    return out[:out_words]


# ---- fields ------------------------------------------------------------------------------------------------------
def _field(lib, prefix, suffix, field, op, avals, bvals=None):
    n = A.FIELDS[field][2]
    a = _arr(A.words(avals, n))
    b = _arr(A.words(bvals if bvals is not None else [0] * len(avals), n))
    fn = getattr(lib, prefix + suffix)
    return A.ints(_run(fn, field, op, len(avals), bufs=[a, b], out_words=len(avals) * n), n)


def _check_field(dev, suffix, field, op, avals, bvals, want):
    """device == want (Python) and device words == hostemu words on the same inputs"""
    label = "%s op %d%s" % (A.FIELDS[field][0], op, " (inlined build)" if suffix else "")
    ops = list(zip(avals, bvals)) if bvals is not None else avals
    got = _field(dev, "dev_field", suffix, field, op, avals, bvals)
    A.assert_same(label + " vs Python", got, want, ops)
    host = _field(H.hostemu(), "emu_field_n", "", field, op, avals, bvals)
    A.assert_same(label + " vs hostemu", got, host, ops)


@pytest.mark.parametrize("suffix", VARIANTS)
@pytest.mark.parametrize("field", sorted(A.FIELDS))
def test_field_ops(dev, field, suffix):
    _, p, n = A.FIELDS[field]
    Rm = 1 << (32 * n)
    Ri = pow(Rm, -1, p)
    pairs = A.binary_pairs(field, seed=1)
    a = [x for x, _ in pairs]
    b = [y for _, y in pairs]
    _check_field(dev, suffix, field, A.MUL, a, b, [x * y * Ri % p for x, y in pairs])
    _check_field(dev, suffix, field, A.ADD, a, b, [(x + y) % p for x, y in pairs])
    _check_field(dev, suffix, field, A.SUB, a, b, [(x - y) % p for x, y in pairs])
    vals = A.field_values(field, seed=1, randoms=256)
    _check_field(dev, suffix, field, A.SQR, vals, None, [x * x * Ri % p for x in vals])
    _check_field(dev, suffix, field, A.NEG, vals, None, [(-x) % p for x in vals])
    _check_field(dev, suffix, field, A.FROM_MONT_IN, vals, None, [x * Rm % p for x in vals])
    mont = [x * Rm % p for x in vals]
    _check_field(dev, suffix, field, A.TO_CANON, mont, None, vals)
    near = [x for x in vals + [p, p + 1, p + 2, Rm - 1, p | 0xFFFFFFFF, p + (1 << 32)] if x < Rm]
    # canonical_in_range writes its verdict to word 0 and zeros elsewhere
    _check_field(dev, suffix, field, A.IN_RANGE, near, None, [1 if x < p else 0 for x in near])


@pytest.mark.parametrize("suffix", VARIANTS)
@pytest.mark.parametrize("field", sorted(A.FIELDS))
def test_field_inversions(dev, field, suffix):
    _, p, n = A.FIELDS[field]
    Rm = 1 << (32 * n)
    vals = A.inverse_values(field, seed=1)
    _check_field(dev, suffix, field, A.INV_WORDS, vals, None, [pow(x, -1, p) for x in vals])
    xm = [x * Rm % p for x in vals] + [0]
    want = [pow(x, -1, p) * Rm % p for x in vals] + [0]
    for op in (A.INV, A.DIVSTEPS, A.INV_XGCD):
        _check_field(dev, suffix, field, op, xm, None, want)


# ---- double-width pieces and Fp2 -----------------------------------------------------------------------------------
def _wide(lib, name, field, op, avals, bvals):
    n = A.FIELDS[field][2]
    wa, wr = (n, 2 * n) if op == 0 else (2 * n, n)
    a = _arr(A.words(avals, wa))
    b = _arr(A.words(bvals, n))
    return A.ints(_run(getattr(lib, name), field, op, len(avals), bufs=[a, b], out_words=len(avals) * wr), wr)


@pytest.mark.parametrize("suffix", VARIANTS)
@pytest.mark.parametrize("field", [2, 3])
def test_mul_wide_and_mont_reduce_wide(dev, field, suffix):
    _, p, n = A.FIELDS[field]
    Ri = pow(1 << (32 * n), -1, p)
    pairs = A.wide_pairs(field)
    a = [x for x, _ in pairs]
    b = [y for _, y in pairs]
    got = _wide(dev, "dev_wide" + suffix, field, 0, a, b)
    A.assert_same("%s mul_wide" % A.FIELDS[field][0], got, [x * y for x, y in pairs], pairs)
    A.assert_same("%s mul_wide vs hostemu" % A.FIELDS[field][0], got, _wide(H.hostemu(), "emu_wide_n", field, 0, a, b), pairs)
    ts = A.reduce_wide_inputs(field)
    got = _wide(dev, "dev_wide" + suffix, field, 1, ts, [0] * len(ts))
    A.assert_same("%s mont_reduce_wide" % A.FIELDS[field][0], got, [t * Ri % p for t in ts], ts)
    A.assert_same("%s mont_reduce_wide vs hostemu" % A.FIELDS[field][0], got,
                  _wide(H.hostemu(), "emu_wide_n", field, 1, ts, [0] * len(ts)), ts)


FP2_FORMS = {0: "three multiplications", 1: "mul_lazy", 2: "operator*", 3: "sqr", 4: "inv"}


@pytest.mark.parametrize("suffix", VARIANTS)
@pytest.mark.parametrize("field", [2, 3])
def test_fp2_ops(dev, field, suffix):
    _, p, n = A.FIELDS[field]
    Ri = pow(1 << (32 * n), -1, p)
    cases = A.fp2_pairs(field, seed=1)
    a = A.words([c for (x, _) in cases for c in x], n)
    b = A.words([c for (_, y) in cases for c in y], n)

    def want(form, x, y):
        (a0, a1), (b0, b1) = x, y
        if form <= 2:
            return ((a0 * b0 - a1 * b1) * Ri % p, (a0 * b1 + a1 * b0) * Ri % p)
        if form == 3:
            return ((a0 * a0 - a1 * a1) * Ri % p, 2 * a0 * a1 * Ri % p)
        # inverse of (a0 + a1 u) R^-1 in Montgomery form: conj / norm, 0 -> 0
        x0, x1 = a0 * Ri % p, a1 * Ri % p
        nrm = (x0 * x0 + x1 * x1) % p
        if nrm == 0:
            return (0, 0)
        i = pow(nrm, -1, p)
        Rm = 1 << (32 * n)
        return (x0 * i * Rm % p, (-x1) * i * Rm % p)

    for form, name in FP2_FORMS.items():
        got = A.ints(_run(getattr(dev, "dev_fp2" + suffix), field, form, len(cases), bufs=[_arr(a), _arr(b)],
                          out_words=len(cases) * 2 * n), n)
        got = list(zip(got[0::2], got[1::2]))
        label = "%s Fp2 %s%s" % (A.FIELDS[field][0], name, " (inlined build)" if suffix else "")
        A.assert_same(label, got, [want(form, x, y) for x, y in cases], cases)
        host = A.ints(_run(H.hostemu().emu_fp2_n, field, form, len(cases), bufs=[_arr(a), _arr(b)],
                           out_words=len(cases) * 2 * n), n)
        A.assert_same(label + " vs hostemu", got, list(zip(host[0::2], host[1::2])), cases)


# ---- Fp12 towers and pairings ------------------------------------------------------------------------------------
def _tower(tower):
    if tower == 0:
        import bls_cases as C
        from oracle import bls_pairing_ref as B
        return C, B, 12, B.X_ABS, "BLS12-381"
    import bn254_pairing_cases as C
    from oracle import bn254_pairing_ref as B
    return C, B, 8, B.U, "bn254"


def _f12_words(B, n, elems):
    return A.words([c for e in elems for c in B.flat(e)], n)


def _f12_elems(B, n, ws):
    v = A.ints(ws, n)
    return [B.unflat(v[12 * i:12 * i + 12]) for i in range(len(v) // 12)]


@pytest.mark.parametrize("tower", [0, 1])
def test_fp12_ops(dev, tower):
    C, B, n, xexp, label = _tower(tower)
    p = B.P
    rnd = random.Random(40 + tower)
    r12 = lambda: B.unflat([rnd.randrange(p) for _ in range(12)])  # noqa: E731
    edge = [B.unflat([p - 1] * 12), B.unflat([1] * 12), B.unflat([(1 << (32 * n)) % p] * 12), B.O12]
    xs = edge + [r12() for _ in range(12)]
    ys = list(reversed(edge)) + [r12() for _ in range(12)]
    easy = (p ** 6 - 1) * (p ** 2 + 1)
    cyc = [B.f12_pow(x, easy) for x in xs[4:8]]
    sparse = lambda f: (((f[0][0], f[0][1], (0, 0)), ((0, 0), f[0][2], (0, 0))) if tower == 0  # noqa: E731
                        else ((f[0][0], (0, 0), (0, 0)), (f[0][1], f[0][2], (0, 0))))
    cases = {
        0: (xs, ys, [B.f12_mul(x, y) for x, y in zip(xs, ys)]),
        1: (xs, xs, [B.f12_sqr(x) for x in xs]),
        2: (cyc, cyc, [B.f12_sqr(c) for c in cyc]),
        3: (xs, xs, [B.f12_inv(x) for x in xs]),
        4: (xs, xs, [B.f12_frobenius(x, 1) for x in xs]),
        5: (xs, xs, [B.f12_frobenius(x, 2) for x in xs]),
        6: (xs, xs, [B.f12_frobenius(x, 3) for x in xs]),
        7: (xs, xs, [B.f12_conj(x) for x in xs]),
        8: (cyc, cyc, [B.f12_pow(c, xexp) for c in cyc]),
        9: (xs[:6], xs[:6], [B.final_exp(x) for x in xs[:6]]),
        10: (xs, ys, [B.f12_mul(x, sparse(y)) for x, y in zip(xs, ys)]),
    }
    for op, (a, b, want) in cases.items():
        aw, bw = _arr(_f12_words(B, n, a)), _arr(_f12_words(B, n, b))
        got = _f12_elems(B, n, _run(dev.dev_fp12, tower, op, len(a), bufs=[aw, bw], out_words=len(a) * 12 * n))
        A.assert_same("%s Fp12 op %d" % (label, op), got, want, list(zip(a, b)))
        host = [C.emu_fp12(op, x, y) for x, y in zip(a, b)]
        A.assert_same("%s Fp12 op %d vs hostemu" % (label, op), got, host, list(zip(a, b)))


@pytest.mark.parametrize("tower", [0, 1])
def test_pairing_values(dev, tower):
    """the pairing VALUE of one pair per thread (Miller loop + final exponentiation), not only a verdict"""
    C, B, n, _, label = _tower(tower)
    rnd = random.Random(50 + tower)
    pairs = [(C.g1_mul(1), C.g2_mul(1)), (C.ID1, C.g2_mul(3)), (C.g1_mul(5), C.ID2)]
    pairs += [(C.g1_mul(rnd.randrange(1, B.N)), C.g2_mul(rnd.randrange(1, B.N))) for _ in range(5)]
    pairs += [(C.g1_mul(-1), C.g2_mul(B.N - 1))]
    pairs += [(C.g1_mul(2), C.g2_off_subgroup(rnd))]
    if tower == 0:
        pairs += [(C.g1_off_subgroup(rnd), C.g2_mul(7))]
    g1 = _arr(A.words([c for pt, _ in pairs for c in pt], n))
    g2 = _arr(A.words([c for _, q in pairs for co in q for c in co], n))
    got = _f12_elems(B, n, _run(dev.dev_pairing, tower, len(pairs), bufs=[g1, g2], out_words=len(pairs) * 12 * n))
    A.assert_same("%s pairing value" % label, got, [B.pairing_product([pr]) for pr in pairs], pairs)
    A.assert_same("%s pairing value vs hostemu" % label, got, [C.emu_pairing([pr]) for pr in pairs], pairs)


# ---- group law -----------------------------------------------------------------------------------------------------
GROUP_OPS = {0: "add", 1: "madd", 2: "dbl", 3: "dbl_affine", 4: "par_add per quad", 5: "par_dbl per quad",
             6: "par_add per warp", 7: "par_dbl per warp"}


def _coord_words(c, n):
    return A.words(list(c) if isinstance(c, tuple) else [c], n)


@pytest.mark.parametrize("curve", sorted(A.GROUP_CURVES))
def test_group_law(dev, curve):
    name = A.GROUP_CURVES[curve]
    P = R.CURVES[name]
    n = 12 if "bls" in name else 8
    parts = 2 if "G2" in name else 1
    acc_words = 4 * parts * n
    in_words = 2 * parts * n
    cases = A.group_cases(curve)

    def acc(pt, lam):
        return [w for c in A.acc_coords(name, pt, lam) for w in _coord_words(c, n)]

    def aff(pt):
        a = pt.toAffine()
        ws = _coord_words(a["x"], n) + _coord_words(a["y"], n)
        return ws + [0] * (acc_words - len(ws))

    for op, opname in GROUP_OPS.items():
        if op == 3 and name == "ed25519":
            continue
        pw, qw, want = [], [], []
        for kind, p, lp, q, lq in cases:
            pw += aff(p) if op == 3 else acc(p, lp)
            qw += aff(q) if op == 1 else acc(q, lq)
            r = p.double() if op in (2, 3, 5, 7) else p.add(q)
            want.append(H.expected_tuple(name, r))
        k = len(cases)
        inf = np.zeros(k, np.uint32)
        xy = np.zeros(k * in_words, np.uint32)
        rc = dev.dev_group(curve, op, k, _cp(_arr(pw)), _cp(_arr(qw)), _cp(xy), _cp(inf))
        assert rc == 0, "device call failed: cudaError_t %d" % rc
        got = [H.unpack_point(name, xy[i * in_words:(i + 1) * in_words].tobytes()) + (int(inf[i]),) for i in range(k)]
        A.assert_same("%s %s" % (name, opname), got, want, [(c[0], c[1].toAffine(), c[3].toAffine()) for c in cases])


# ---- warp-shared inversion -----------------------------------------------------------------------------------------
# dev_warp_inv field id -> (label, p, limbs, coordinates): every field type the kernels call warp_batch_inverse with
WARP_INV_FIELDS = {0: ("secp256k1 Fp / SchF", R.SECP256K1_CURVE["p"], 8, 1), 1: ("ed25519 Fp", R.ED25519_CURVE["p"], 8, 1),
                   2: ("bn254 Fp", R.BN254_G1_CURVE["p"], 8, 1), 3: ("bn254 Fp2", R.BN254_G1_CURVE["p"], 8, 2),
                   4: ("BLS12-381 Fp", R.BLS12_381_G1_CURVE["p"], 12, 1),
                   5: ("BLS12-381 Fp2", R.BLS12_381_G1_CURVE["p"], 12, 2),
                   6: ("secp256k1 Fn (EcS)", R.SECP256K1_CURVE["n"], 8, 1)}


@pytest.mark.parametrize("field", sorted(WARP_INV_FIELDS))
def test_warp_batch_inverse(dev, field):
    label, p, n, parts = WARP_INV_FIELDS[field]
    Rm = (1 << (32 * n)) % p
    if parts == 1:
        specials = [1, p - 1, Rm, p - 2]
        rand = lambda rnd: rnd.randrange(1, p)  # noqa: E731
        inv = lambda x: pow(x, -1, p)  # noqa: E731
        flat = lambda x: [x]  # noqa: E731
    else:
        F2 = R.Field2(R.Field(p))
        specials = [(1, 0), (p - 1, 0), (Rm, 0), (0, 1), (p - 1, p - 1), (Rm, Rm)]
        rand = lambda rnd: (rnd.randrange(p), rnd.randrange(1, p))  # noqa: E731
        inv = F2.inv
        flat = list
    for batch in A.warp_inverse_batches(specials, rand, seed=field):
        z = _arr(A.words([c for x in batch for c in flat(x)], n))
        got = A.ints(_run(dev.dev_warp_inv, field, len(batch), bufs=[z], out_words=len(batch) * parts * n), n)
        if parts == 2:
            got = list(zip(got[0::2], got[1::2]))
        A.assert_same("%s warp_batch_inverse n=%d" % (label, len(batch)), got, [inv(x) for x in batch], batch)
