"""The MSM pipeline in the regimes the rest of the suite does not reach: several MSMs in flight on the four slots with
distinct inputs, the synchronous entry points running on slot 0 beside them, and sizes above 2^20, up to the 2^26
BLS12-381 G1 terms one H100 holds (DESIGN §3).

Exact reference at every size (the scalar-in-exponent identity of test_gpu_parity.py): points P_i = k_i G, generated on
the GPU through the fixed-point table of G (nmsm_point_table_mul_batch, itself tested against the oracle) and
spot-checked against the oracle, and scalars s_i, so that sum s_i P_i = (sum k_i s_i mod r) G.  The dot product is
taken in 8-bit limbs as float64 matrix products (LimbDot: exact, every partial sum is an integer below 2^53), the last
multiplication by the oracle.  Inputs are fixed-seed byte arrays below r with planted edge scalars (0, 1, r - 1, a run
of equal scalars) and edge points (G, -G, one point twice).
"""
import ctypes

import numpy as np
import pytest
import torch

import helpers as H
from conftest import load_golden
from oracle import noble_ref as R

gpu = pytest.mark.gpu

CHUNK = 1 << 22  # points generated per table-multiply call (bounds host memory at every size)
SPOT_CHECKS = 64  # generated points compared with the oracle per case
SLOT0_MSG = "slot 0 holds an MSM that has not been collected: collect it before a synchronous call"
BUSY_MSG = "slot busy: collect the previous MSM first"
SPLIT = {"secp256k1": 2, "ed25519": 1, "bn254_G1": 2, "bn254_G2": 1, "bls12_381_G1": 2, "bls12_381_G2": 4}


# ------------------------------------------------------------------------------------------------
# exact reference: scalars as byte rows, sum k_i s_i mod r through 8-bit limb matrix products
# ------------------------------------------------------------------------------------------------
def draw_below(rng, m, order):
    """m fixed-seed scalars below `order` as an (m, 32) uint8 array of little-endian rows: uniform low bytes, the top
    byte uniform below order's top byte (so every value is < (order >> 248) * 2^248 <= order)."""
    a = rng.integers(0, 256, size=(m, 32), dtype=np.uint8)
    a[:, 31] = rng.integers(0, order >> 248, size=m, dtype=np.uint8)
    return a


def row_int(row) -> int:
    return int.from_bytes(row.tobytes(), "little")


def set_row(a, i, v: int) -> None:
    a[i] = np.frombuffer(v.to_bytes(32, "little"), dtype=np.uint8)


class LimbDot:
    """sum_i k_i s_i over byte-row scalars, accumulated chunk by chunk.  With k = sum_a K_a 2^(8a) and s likewise,
    sum_i k_i s_i = sum_(a,b) M[a, b] 2^(8(a+b)) where M = K^T S is a 32 x 32 matrix of integers <= rows * 255^2.  The
    products are float64 matrix products: exact while every partial sum stays below 2^53, i.e. for fewer than 2^37
    rows (2^26 rows reach 2^42)."""

    def __init__(self, rows_per_product=1 << 18):
        self.m = np.zeros((32, 32), dtype=np.float64)
        self.rows = 0
        self.step = rows_per_product

    def add(self, K, S):
        assert K.shape == S.shape and K.shape[1] == 32
        for lo in range(0, len(K), self.step):
            self.m += K[lo:lo + self.step].T.astype(np.float64) @ S[lo:lo + self.step].astype(np.float64)
        self.rows += len(K)
        assert self.rows < 1 << 37, "float64 limb sums would no longer be exact"

    def value(self, order: int) -> int:
        return sum(int(self.m[a, b]) << (8 * (a + b)) for a in range(32) for b in range(32)) % order


def test_limb_dot_matches_python_integers():
    """The reference routine itself against plain Python integers at 2^12 terms, on every scalar field, with ragged
    product chunks and the planted edge rows; draw_below stays below r."""
    rng = np.random.default_rng(12)
    n = 1 << 12
    for name in ("bls12_381_G1", "bn254_G1", "secp256k1", "ed25519"):
        order = R.CURVES[name].Fn.ORDER
        K, S = draw_below(rng, n, order), draw_below(rng, n, order)
        for i, v in ((0, 0), (1, 1), (2, order - 1), (n - 1, order - 1)):
            set_row(S, i, v)
            set_row(K, n - 1 - i, v)
        S[100:300] = S[99]
        ks, ss = [row_int(r) for r in K], [row_int(r) for r in S]
        assert max(ks + ss) < order
        dot = LimbDot(rows_per_product=1000)
        dot.add(K[:3001], S[:3001])
        dot.add(K[3001:], S[3001:])
        assert dot.rows == n
        assert dot.value(order) == sum(k * s for k, s in zip(ks, ss)) % order, name
    # all limbs 0xff: the largest limb products, still exact
    F = np.full((n, 32), 255, dtype=np.uint8)
    dot = LimbDot()
    dot.add(F, F)
    assert dot.value(2**1024) == n * (2**256 - 1) ** 2


# ------------------------------------------------------------------------------------------------
# input buffers and cases
# ------------------------------------------------------------------------------------------------
def lib():
    from nmsm import _lib

    return _lib.load()


def check(rc):
    from nmsm import _lib

    _lib.check(rc)


class Buf:
    """Bytes in pageable host memory (numpy), pinned host memory (nmsm_host_alloc) or device memory (torch)."""

    def __init__(self, kind, nbytes):
        self.kind, self.nbytes = kind, nbytes
        self.a = self.t = None
        if kind == "device":
            self.t = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
            self.ptr = self.t.data_ptr()
        elif kind == "pinned":
            self.ptr = lib().nmsm_host_alloc(nbytes)
            assert self.ptr, "nmsm_host_alloc(%d) failed" % nbytes
            self.a = np.ctypeslib.as_array((ctypes.c_uint8 * nbytes).from_address(self.ptr))
        else:
            assert kind == "pageable"
            self.a = np.empty(nbytes, dtype=np.uint8)
            self.ptr = self.a.ctypes.data

    @property
    def on_device(self):
        return 1 if self.kind == "device" else 0

    def write(self, off, src):
        """src: a contiguous uint8 numpy array"""
        src = src.reshape(-1)
        if self.t is not None:
            self.t[off:off + len(src)].copy_(torch.from_numpy(src))
        else:
            self.a[off:off + len(src)] = src

    def tobytes(self) -> bytes:
        return self.t.cpu().numpy().tobytes() if self.t is not None else self.a.tobytes()

    def free(self):
        if self.kind == "pinned" and self.ptr:
            self.a = None
            lib().nmsm_host_free(self.ptr)
        self.ptr, self.a, self.t = 0, None, None


class Case:
    """n points k_i G and scalars s_i in buffers of one kind, and the expected (x, y, is_inf) of their MSM."""

    def __init__(self, name, n, pts, sc, total, K=None):
        P = R.CURVES[name]
        self.name, self.n, self.cid, self.pts, self.sc, self.K = name, n, H.CURVE_IDS[name], pts, sc, K
        self.exp = H.expected_tuple(name, H.expected_from_total(P, total))
        self.label = "%s n=%d %s" % (name, n, pts.kind)

    def free(self):
        self.pts.free()
        self.sc.free()
        self.K = None


_G_TABLES = {}


def g_table(cid):
    """nmsm_point_table handle of the generator (kept for the module; tables live outside the slot workspaces)"""
    import nmsm

    if cid not in _G_TABLES:
        name = [k for k, v in H.CURVE_IDS.items() if v == cid][0]
        _G_TABLES[cid] = nmsm.PointTable(cid, H.point_bytes(name, R.CURVES[name].BASE))
    return _G_TABLES[cid]


def point_bytes_of(name):
    return 2 * H.FP_BYTES[name] * H.PARTS[name]


def make_case(name, n, seed, kind, keep_k=False):
    """Points k_i G (on the GPU, CHUNK at a time) and scalars s_i into `kind` buffers.  Planted: s = 0, 1, r - 1 at
    indices 0, 1, 2 and r - 1 at n - 1, a run of min(4096, n / 8) equal scalars from n / 2; k = 1 and r - 1 (G, -G) at
    indices 3, 4 and k_6 = k_5 (the same point twice).  64 generated points are compared with the oracle."""
    P = R.CURVES[name]
    order = P.Fn.ORDER
    cid = H.CURVE_IDS[name]
    pb = point_bytes_of(name)
    rng = np.random.default_rng(seed)
    pts, sc = Buf(kind, n * pb), Buf(kind, n * 32)
    stage = np.empty(min(n, CHUNK) * pb, dtype=np.uint8) if kind == "device" else None
    infs = np.empty(min(n, CHUNK), dtype=np.uint8)
    run_lo, run_len = n // 2, min(4096, n // 8)
    run_val = row_int(draw_below(rng, 1, order)[0])
    s_edges = {0: 0, 1: 1, 2: order - 1, n - 1: order - 1}
    k_edges = {3: 1, 4: order - 1}
    spots = sorted(set(range(8)) | set(np.linspace(8, n - 1, SPOT_CHECKS - 8).astype(np.int64).tolist()))
    dot, Ks, seen = LimbDot(), [], []
    handle = g_table(cid).handle
    for lo in range(0, n, CHUNK):
        m = min(CHUNK, n - lo)
        K, S = draw_below(rng, m, order), draw_below(rng, m, order)
        for i, v in s_edges.items():
            if lo <= i < lo + m:
                set_row(S, i - lo, v)
        a, b = max(run_lo, lo), min(run_lo + run_len, lo + m)
        for i in range(a, b):
            set_row(S, i - lo, run_val)
        if lo == 0:
            for i, v in k_edges.items():
                set_row(K, i, v)
            K[6] = K[5]
        K[~K.any(axis=1), 0] = 1  # the table multiply takes 1 <= k < r
        dst = stage if stage is not None else pts.a[lo * pb:(lo + m) * pb]
        check(lib().nmsm_point_table_mul_batch(handle, K.ctypes.data, m, 0, dst.ctypes.data, infs.ctypes.data))
        assert not infs[:m].any()
        if stage is not None:
            pts.write(lo * pb, stage[:m * pb])
        sc.write(lo * 32, S)
        dot.add(K, S)
        if keep_k:
            Ks.append(K)
        for i in spots:
            if lo <= i < lo + m:
                seen.append((i, row_int(K[i - lo]), dst[(i - lo) * pb:(i - lo + 1) * pb].tobytes()))
    if kind == "device":
        torch.cuda.synchronize()
    assert len(seen) == SPOT_CHECKS
    for i, k, xy in seen:
        assert H.unpack_point(name, xy) == R.affine_tuple(P, P.BASE.multiply(k)), (name, n, "generated point", i)
    return Case(name, n, pts, sc, dot.value(order), np.concatenate(Ks) if keep_k else None)


def more_scalars(case, seed, kind):
    """Another scalar vector for the points of `case` (made with keep_k): (buffer, expected tuple)."""
    P = R.CURVES[case.name]
    S = draw_below(np.random.default_rng(seed), case.n, P.Fn.ORDER)
    set_row(S, 0, P.Fn.ORDER - 1)
    buf = Buf(kind, case.n * 32)
    buf.write(0, S)
    if kind == "device":
        torch.cuda.synchronize()
    dot = LimbDot()
    dot.add(case.K, S)
    return buf, H.expected_tuple(case.name, H.expected_from_total(P, dot.value(P.Fn.ORDER)))


def plan(nmsm):
    """The plan of the last collected MSM, for assertion messages."""
    _, info = nmsm.last_timing()
    return "plan c=%d windows=%d L=%d K=%d groups=%d" % (info.c, info.windows, info.entries_per_thread,
                                                         info.reduce_chunk, info.window_groups)


def result(name, out, inf):
    return (*H.unpack_point(name, out), inf)


def submit(case, slot, scalars=None):
    sc = scalars if scalars is not None else case.sc
    assert sc.on_device == case.pts.on_device
    check(lib().nmsm_msm_submit(case.cid, case.pts.ptr, sc.ptr, case.n, case.pts.on_device, slot))


def collect(slot, name):
    out = ctypes.create_string_buffer(192)
    inf = ctypes.c_int(0)
    check(lib().nmsm_msm_collect(slot, ctypes.cast(out, ctypes.c_void_p), ctypes.byref(inf)))
    return result(name, out.raw, inf.value)


def msm_sync(nmsm, case):
    if case.pts.on_device:
        out, inf = nmsm.msm_device(case.cid, case.pts.ptr, case.sc.ptr, case.n)
    else:
        out, inf = nmsm.msm_host_ptr(case.cid, case.pts.ptr, case.sc.ptr, case.n)
    return result(case.name, out, inf)


def device_memory_needed(name, n, extra=0):
    """Rough device footprint of an n-term MSM: inputs, the prepared points (SPLIT entries per term), the sorted bucket
    entries, 1/8 slack of the workspace buffers, plus 2 GiB for everything else."""
    pb = point_bytes_of(name)
    aff = pb * 3 // 2 if name == "ed25519" else pb
    return int(n * (pb + 32 + SPLIT[name] * (aff + 80)) * 1.125) + (2 << 30) + extra


def require_free(nbytes, what):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("%s needs about %.1f GiB of device memory, %.1f GiB are free (the GPU is shared)"
                    % (what, nbytes / 2**30, free / 2**30))


# ------------------------------------------------------------------------------------------------
# fixtures
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    yield m
    for t in _G_TABLES.values():
        t.close()
    _G_TABLES.clear()
    # the four slots' workspaces grew to this module's sizes: give them back to the tests that follow
    lib().nmsm_shutdown()
    check(lib().nmsm_init(0))


@pytest.fixture
def slots(nmsm):
    """Leaves no MSM pending when a test fails half-way (later tests need free slots)."""
    yield
    out = ctypes.create_string_buffer(192)
    inf = ctypes.c_int(0)
    for s in range(4):
        lib().nmsm_msm_collect(s, ctypes.cast(out, ctypes.c_void_p), ctypes.byref(inf))
    nmsm.set_window_groups(0)
    nmsm.set_profiling(False)


@pytest.fixture
def release_workspace(nmsm, slots):
    """After a large MSM: give its slot workspace (tens of GB) and torch's cached blocks back to the device."""
    yield
    lib().nmsm_shutdown()
    check(lib().nmsm_init(0))
    torch.cuda.empty_cache()


# four curves, sizes and input kinds, one per slot in the first round
FOUR = (("bls12_381_G1", 1 << 20, "pageable"),  # 96 MiB of points: the staged H2D path, k_prepare on prep_stream
        ("bn254_G1", 1 << 18, "pinned"),
        ("bls12_381_G2", 1 << 16, "device"),
        ("secp256k1", 1 << 15, "device"))


@pytest.fixture(scope="module")
def four_cases(nmsm):
    cases = [make_case(name, n, 100 + i, kind) for i, (name, n, kind) in enumerate(FOUR)]
    yield cases
    for c in cases:
        c.free()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------
# several MSMs in flight
# ------------------------------------------------------------------------------------------------
def run_four_slots(nmsm, cases, check_plan=None):
    """Case i on slot i, collected out of submission order; then case i on slot i + 1 (mod 4), every submit while the
    other three slots are busy, so each slot's workspace is resized beside running MSMs."""
    for rot, order in ((0, (2, 0, 3, 1)), (1, (1, 3, 0, 2))):
        for i, c in enumerate(cases):
            submit(c, (i + rot) % 4)
        for i in order:
            slot = (i + rot) % 4
            got = collect(slot, cases[i].name)
            assert got == cases[i].exp, (cases[i].label, "slot %d" % slot, plan(nmsm))
            if check_plan:
                check_plan(cases[i])


@gpu
@pytest.mark.parametrize("mode", ["default", "window_groups_4", "profiling"])
def test_four_slots_distinct_curves(nmsm, slots, four_cases, mode):
    """Four slots busy at once with different curves, sizes and input memory (pageable, pinned, device).  The forced
    window groups run the multi-stream group pipeline on every slot; profiling forces the linear pipeline (k_prepare on
    the main stream)."""

    def check_plan(case):
        _, info = nmsm.last_timing()
        if mode == "profiling":
            assert info.window_groups == 1, (case.label, plan(nmsm))
        elif mode == "window_groups_4":  # engine.cuh submit_msm: groups of ceil(W / 4) windows
            per = -(-info.windows // min(4, info.windows))
            assert info.window_groups == -(-info.windows // per), (case.label, plan(nmsm))

    nmsm.set_window_groups(4 if mode == "window_groups_4" else 0)
    nmsm.set_profiling(mode == "profiling")
    run_four_slots(nmsm, four_cases, check_plan)


@gpu
def test_four_slots_same_shape_distinct_inputs(nmsm, slots):
    """bench.py's in-flight shape (four BLS12-381 G1 MSMs of 2^20 device-resident terms) with different points and
    scalars per slot: a slot that read another slot's prepared points, sorted entries or buckets gives a wrong point."""
    cases = [make_case("bls12_381_G1", 1 << 20, 200 + i, "device") for i in range(4)]
    try:
        run_four_slots(nmsm, cases)
    finally:
        for c in cases:
            c.free()


@gpu
def test_points_submit_in_flight(nmsm, slots):
    """nmsm_msm_points_submit on two prepared sets (bn254 G1 without a table, BLS12-381 G1 with the fixed-base table),
    host and device scalars, one set on two slots at once with different scalars, mixed with plain submits."""
    a = make_case("bn254_G1", 1 << 16, 300, "pageable", keep_k=True)
    b = make_case("bls12_381_G1", 1 << 16, 301, "pageable", keep_k=True)
    plain = make_case("secp256k1", 1 << 15, 302, "device")
    a2, a2_exp = more_scalars(a, 303, "device")
    b2, b2_exp = more_scalars(b, 304, "device")
    set_a = nmsm.PointSet(a.cid, a.pts.tobytes(), a.n)
    set_b = nmsm.PointSet(b.cid, b.pts.tobytes(), b.n)
    c, levels = set_b.precompute(0)
    try:
        def psubmit(ps, case, scalars, slot):
            check(lib().nmsm_msm_points_submit(ps.handle, scalars.ptr, case.n, scalars.on_device, slot))

        rounds = [
            # (slot, what to submit, expected, collect order)
            [(0, lambda s: psubmit(set_a, a, a.sc, s), a),
             (1, lambda s: psubmit(set_b, b, b2, s), (b, b2_exp)),
             (2, lambda s: submit(plain, s), plain),
             (3, lambda s: psubmit(set_a, a, a2, s), (a, a2_exp))],
            [(0, lambda s: psubmit(set_b, b, b.sc, s), b),
             (1, lambda s: submit(plain, s), plain),
             (2, lambda s: psubmit(set_a, a, a2, s), (a, a2_exp)),
             (3, lambda s: psubmit(set_b, b, b2, s), (b, b2_exp))],
        ]
        for k, entries in enumerate(rounds):
            for slot, fn, _ in entries:
                fn(slot)
            for slot in ((3, 1, 2, 0), (1, 3, 0, 2))[k]:
                want = entries[slot][2]
                case, exp = want if isinstance(want, tuple) else (want, want.exp)
                got = collect(slot, case.name)
                assert got == exp, (case.label, "round %d slot %d" % (k, slot), "table c=%d levels=%d" % (c, levels),
                                    plan(nmsm))
    finally:
        set_a.close()
        set_b.close()
        for x in (a, b, plain):
            x.free()
        a2.free()
        b2.free()


@gpu
def test_partial_shards_held_on_all_slots(nmsm, slots):
    """nmsm_msm_submit_partial: four shards of uneven sizes of one MSM held on all four slots before any collect, the
    raw accumulators folded by nmsm_fold_partials_device."""
    case = make_case("bls12_381_G1", 1 << 18, 400, "device")
    try:
        pb, acc_b = point_bytes_of(case.name), lib().nmsm_acc_bytes(case.cid)
        accs = torch.zeros(4 * acc_b, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        bounds = [0, 70001, 131072, 200003, case.n]
        for j in range(4):
            lo, hi = bounds[j], bounds[j + 1]
            check(lib().nmsm_msm_submit_partial(case.cid, case.pts.ptr + lo * pb, case.sc.ptr + lo * 32, hi - lo,
                                                accs.data_ptr() + j * acc_b, j))
        for j in (2, 0, 3, 1):
            check(lib().nmsm_msm_collect(j, None, None))
        out = ctypes.create_string_buffer(pb)
        inf = ctypes.c_int(0)
        check(lib().nmsm_fold_partials_device(case.cid, accs.data_ptr(), 4, ctypes.cast(out, ctypes.c_void_p),
                                              ctypes.byref(inf)))
        assert result(case.name, out.raw, inf.value) == case.exp, (case.label, plan(nmsm))
    finally:
        case.free()


def sync_calls(nmsm):
    """One small call of every synchronous entry point family, inputs and oracle verdicts prepared up front:
    [(label, call, expected)]."""
    import random

    import bls_cases as BC
    import bn254_pairing_cases as BN
    import ecdsa_cases as E
    import schnorr_cases as S
    from nmsm import fft as GF
    from oracle import ecdsa_ref as ER
    from oracle import noble_fft as OF
    from oracle import schnorr_ref as SR

    rnd = random.Random(600)
    out = []
    # nmsm_msm: a small one, and one whose 24 MiB of pageable points go through the shared staging buffers
    P, pts, scalars, _ = H.soak_inputs("bls12_381_G1", 300, seed_offset=6)
    pb, sb = H.pack_points("bls12_381_G1", pts), H.pack_scalars(scalars)
    out.append(("msm", lambda: result("bls12_381_G1", *nmsm.msm_packed(4, pb, sb, 300)),
                H.expected_tuple("bls12_381_G1", R.pippenger(P, pts, scalars))))
    staged = make_case("bls12_381_G1", 1 << 18, 601, "pageable")
    out.append(("msm staged", lambda: msm_sync(nmsm, staged), staged.exp))
    # nmsm_mul_batch
    Q = R.CURVES["secp256k1"]
    qs = R.normalizeZ(Q, [Q.BASE.multiply(rnd.randrange(1, Q.Fn.ORDER)) for _ in range(8)])
    ks = [rnd.randrange(1, Q.Fn.ORDER) for _ in qs]
    qb, kb = H.pack_points("secp256k1", qs), H.pack_scalars(ks)
    out.append(("mul_batch", lambda: nmsm.mul_batch_packed(0, qb, kb, 8, False)[0],
                b"".join(H.point_bytes("secp256k1", q.multiply(k)) for q, k in zip(qs, ks))))

    # point-table create + multiply
    B = R.CURVES["bn254_G1"]
    base = R.normalizeZ(B, [B.BASE.multiply(rnd.randrange(1, B.Fn.ORDER))])[0]
    tks = [1, B.Fn.ORDER - 1] + [rnd.randrange(1, B.Fn.ORDER) for _ in range(6)]

    def table_mul():
        t = nmsm.PointTable(2, H.point_bytes("bn254_G1", base))
        try:
            return t.mul_batch(H.pack_scalars(tks), len(tks), False)[0]
        finally:
            t.close()

    out.append(("point_table", table_mul, b"".join(H.point_bytes("bn254_G1", base.multiply(k)) for k in tks)))
    # decode
    encs = [bytes.fromhex(c) for c in load_golden("bls12_381.json")["G1_Compressed"][:16]]

    def decode():
        xy, st = nmsm.points_decode(4, b"".join(encs), 16)
        return list(st), [H.unpack_point("bls12_381_G1", xy[i * 96:(i + 1) * 96]) for i in range(1, 16)]

    out.append(("decode", decode, ([2] + [1] * 15, [R.bls12_381_g1_decode(e) for e in encs[1:]])))
    # torsion
    tp = pts[:2] + H.bls_g1_non_subgroup_points(2, seed=61)
    tb = H.pack_points("bls12_381_G1", tp)
    out.append(("torsion", lambda: nmsm.torsion_free_packed(6, tb, 4), b"\x01\x01\x00\x00"))
    # NTT
    p = OF.FR["bn254"]
    coeffs = [rnd.randrange(p) for _ in range(1 << 10)]
    out.append(("ntt", lambda: GF.FFT(GF.rootsOfUnity("bn254", 7)).direct(coeffs),
                OF.FFT(OF.RootsOfUnity(p, 7)).direct(coeffs)))
    # ECDSA and Schnorr (the first of them after nmsm_init builds the shared table of G)
    ecases = E.edge_cases(61)
    out.append(("ecdsa", lambda: nmsm.ecdsa_verify_batch([c[1] for c in ecases], [c[2] for c in ecases],
                                                         [c[3] for c in ecases]),
                [ER.secp256k1_ecdsa_verify(c[1], c[2], c[3]) for c in ecases]))
    scases = S.edge_cases(62)
    out.append(("schnorr", lambda: nmsm.schnorr_verify_batch([c[1] for c in scases], [c[2] for c in scases],
                                                             [c[3] for c in scases]),
                [SR.secp256k1_schnorr_verify(c[1], c[2], c[3]) for c in scases]))
    # ed25519 batch verify: the RFC 8032 vectors, then one of them corrupted (s >= l)
    vec = load_golden("ed25519.json")["vectors"][:16]
    sigs = [bytes.fromhex(v["sig"]) for v in vec]
    msgs = [bytes.fromhex(v["msg"]) for v in vec]
    pks = [bytes.fromhex(v["pk"]) for v in vec]
    bad = list(sigs)
    bad[5] = bad[5][:63] + bytes([bad[5][63] | 0xF0])
    assert all(R.ed25519_verify(s, m, k) for s, m, k in zip(sigs, msgs, pks))
    out.append(("ed25519", lambda: (nmsm.ed25519_verify_batch(sigs, msgs, pks), nmsm.ed25519_verify_batch(bad, msgs, pks)),
                ((True, -1), (False, 5))))
    # pairing checks: verdicts known by bilinearity
    bls_args = BC.pack_checks([BC.true_check(rnd, 2), BC.false_check(rnd, 3), BC.true_check(rnd, 1)])
    out.append(("bls12_381 pairing", lambda: nmsm.pairing_check_batch_packed(*bls_args, 3), b"\x01\x00\x01"))
    bn_args = BN.pack_checks([BN.false_check(rnd, 2), BN.groth16_check(rnd), BN.true_check(rnd, 3)])
    out.append(("bn254 pairing", lambda: nmsm.bn254_pairing_check_batch_packed(*bn_args, 3), b"\x00\x01\x01"))
    return out


@gpu
def test_synchronous_calls_beside_busy_slots(nmsm, slots, four_cases):
    """With slots 1 to 3 busy, every synchronous entry point family runs once on slot 0 (the staging buffers, the table of
    G, the signature scratch and the NTT buffers are global) and agrees with its oracle; then slots 1 to 3 collect their
    MSMs unharmed."""
    calls = sync_calls(nmsm)
    busy = {1: four_cases[0], 2: four_cases[2], 3: four_cases[1]}
    for slot, case in busy.items():
        submit(case, slot)
    try:
        for label, call, exp in calls:
            assert call() == exp, label
    finally:
        for slot in (3, 1, 2):
            assert collect(slot, busy[slot].name) == busy[slot].exp, (busy[slot].label, "slot %d" % slot, plan(nmsm))


@gpu
def test_slot0_pending_refuses_synchronous_calls(nmsm, slots):
    """While an MSM submitted on slot 0 is pending, every synchronous entry point returns NMSM_ERR_ARG with its message
    (arguments are valid, so a missing guard would run the call and overwrite slot 0), the asynchronous ones refuse
    slot 0 as busy, and the pending MSM still collects the right point."""
    from nmsm import _lib

    L = lib()
    pending = make_case("bls12_381_G1", 1 << 18, 500, "device")
    g1 = R.CURVES["bls12_381_G1"]
    gb = H.point_bytes("bls12_381_G1", g1.BASE)
    pt, sc = ctypes.create_string_buffer(gb, 96), ctypes.create_string_buffer(H.pack_scalars([5]), 32)
    d_pt = torch.frombuffer(bytearray(gb), dtype=torch.uint8).cuda()
    d_sc = torch.frombuffer(bytearray(H.pack_scalars([5])), dtype=torch.uint8).cuda()
    d_acc = torch.zeros(L.nmsm_acc_bytes(4), dtype=torch.uint8, device="cuda")
    d_ntt = torch.zeros(32, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ps = nmsm.PointSet(4, gb, 1)
    tbl = nmsm.PointTable(4, gb)
    out, inf, outs = ctypes.create_string_buffer(192), ctypes.c_int(0), ctypes.create_string_buffer(16)
    ok, bad = ctypes.c_int(0), ctypes.c_longlong(0)
    ntt_vals = ctypes.create_string_buffer(32)
    handle = ctypes.c_uint64(0)
    c_, lv = ctypes.c_int(0), ctypes.c_int(0)
    off0 = ctypes.create_string_buffer(8)
    v = lambda b: ctypes.cast(b, ctypes.c_void_p)  # noqa: E731
    sync = {
        "nmsm_msm": lambda: L.nmsm_msm(4, v(pt), v(sc), 1, v(out), ctypes.byref(inf)),
        "nmsm_msm_device": lambda: L.nmsm_msm_device(4, d_pt.data_ptr(), d_sc.data_ptr(), 1, v(out), ctypes.byref(inf)),
        "nmsm_msm_partial_device": lambda: L.nmsm_msm_partial_device(4, d_pt.data_ptr(), d_sc.data_ptr(), 1,
                                                                     d_acc.data_ptr()),
        "nmsm_fold_partials_device": lambda: L.nmsm_fold_partials_device(4, d_acc.data_ptr(), 0, v(out), ctypes.byref(inf)),
        "nmsm_accs_normalize": lambda: L.nmsm_accs_normalize(4, None, 0, 0, None, None),
        "nmsm_mul_batch": lambda: L.nmsm_mul_batch(4, v(pt), v(sc), 1, 0, v(out), v(outs)),
        "nmsm_points_torsion_free": lambda: L.nmsm_points_torsion_free(4, v(pt), 1, v(outs)),
        "nmsm_points_upload": lambda: L.nmsm_points_upload(4, v(pt), 1, ctypes.byref(handle)),
        "nmsm_msm_points": lambda: L.nmsm_msm_points(ps.handle, v(sc), 1, v(out), ctypes.byref(inf)),
        "nmsm_points_precompute": lambda: L.nmsm_points_precompute(ps.handle, 8, ctypes.byref(c_), ctypes.byref(lv)),
        "nmsm_point_table_create": lambda: L.nmsm_point_table_create(4, v(pt), ctypes.byref(handle)),
        "nmsm_point_table_mul_batch": lambda: L.nmsm_point_table_mul_batch(tbl.handle, v(sc), 1, 0, v(out), v(outs)),
        "nmsm_ed25519_verify_batch": lambda: L.nmsm_ed25519_verify_batch(None, None, None, v(off0), 0, None,
                                                                         ctypes.byref(ok), ctypes.byref(bad)),
        "nmsm_secp256k1_verify_batch": lambda: L.nmsm_secp256k1_verify_batch(None, None, None, None, None, 0, 3, None),
        "nmsm_secp256k1_schnorr_verify_batch": lambda: L.nmsm_secp256k1_schnorr_verify_batch(None, None, None, None, 0,
                                                                                             None),
        "nmsm_bls12_381_pairing_check_batch": lambda: L.nmsm_bls12_381_pairing_check_batch(None, None, v(off0), 0, None),
        "nmsm_bn254_pairing_check_batch": lambda: L.nmsm_bn254_pairing_check_batch(None, None, v(off0), 0, None),
        "nmsm_bls12_381_verify_batch": lambda: L.nmsm_bls12_381_verify_batch(None, None, None, 0, None),
        "nmsm_points_decode": lambda: L.nmsm_points_decode(4, None, 0, None, None),
        "nmsm_points_decode_ex": lambda: L.nmsm_points_decode_ex(1, None, 0, 1, None, None),
        "nmsm_points_on_curve": lambda: L.nmsm_points_on_curve(4, v(pt), 1, v(outs)),
        "nmsm_ntt": lambda: L.nmsm_ntt(2, v(ntt_vals), 0, 7, 0, 0, 0),
        "nmsm_ntt_device": lambda: L.nmsm_ntt_device(2, d_ntt.data_ptr(), 0, 7, 0, 0, 0),
    }
    busy = {
        "nmsm_msm_submit": lambda: L.nmsm_msm_submit(4, d_pt.data_ptr(), d_sc.data_ptr(), 1, 1, 0),
        "nmsm_msm_submit_partial": lambda: L.nmsm_msm_submit_partial(4, d_pt.data_ptr(), d_sc.data_ptr(), 1,
                                                                     d_acc.data_ptr(), 0),
        "nmsm_msm_points_submit": lambda: L.nmsm_msm_points_submit(ps.handle, v(sc), 1, 0, 0),
    }
    try:
        submit(pending, 0)
        for fn, call in list(sync.items()) + list(busy.items()):
            rc = call()
            msg = L.nmsm_last_error().decode()
            assert (rc, msg) == (_lib.ERR_ARG, SLOT0_MSG if fn in sync else BUSY_MSG), fn
        assert collect(0, pending.name) == pending.exp, (pending.label, plan(nmsm))
        # slot 0 is free again: the refused calls run
        assert L.nmsm_msm(4, v(pt), v(sc), 1, v(out), ctypes.byref(inf)) == 0
        assert result("bls12_381_G1", out.raw[:96], inf.value) == H.expected_tuple("bls12_381_G1", g1.BASE.multiply(5))
        assert L.nmsm_ntt(2, v(ntt_vals), 0, 7, 0, 0, 0) == 0
    finally:
        ps.close()
        tbl.close()
        pending.free()


@gpu
def test_n_of_2p31_is_refused_before_allocating(nmsm, slots):
    """n = 2^31 on every MSM entry point, host and device inputs, every curve id: NMSM_ERR_ARG "n must be < 2^31" from
    16-byte buffers, i.e. before anything n-sized is allocated or copied; no slot is left pending and the library keeps
    working."""
    from nmsm import _lib

    L = lib()
    n = 1 << 31
    h = ctypes.create_string_buffer(16)
    d = torch.zeros(16, dtype=torch.uint8, device="cuda")
    d_acc = torch.zeros(256, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    out, inf = ctypes.create_string_buffer(192), ctypes.c_int(0)
    hp, dp, ap = ctypes.addressof(h), d.data_ptr(), d_acc.data_ptr()
    for cid in range(8):
        calls = {
            "nmsm_msm (host)": lambda: L.nmsm_msm(cid, hp, hp, n, ctypes.cast(out, ctypes.c_void_p), ctypes.byref(inf)),
            "nmsm_msm_submit (host)": lambda: L.nmsm_msm_submit(cid, hp, hp, n, 0, 1),
            "nmsm_msm_device": lambda: L.nmsm_msm_device(cid, dp, dp, n, ctypes.cast(out, ctypes.c_void_p),
                                                         ctypes.byref(inf)),
            "nmsm_msm_submit (device)": lambda: L.nmsm_msm_submit(cid, dp, dp, n, 1, 2),
            "nmsm_msm_partial_device": lambda: L.nmsm_msm_partial_device(cid, dp, dp, n, ap),
            "nmsm_msm_submit_partial": lambda: L.nmsm_msm_submit_partial(cid, dp, dp, n, ap, 3),
        }
        for fn, call in calls.items():
            rc = call()
            assert (rc, L.nmsm_last_error().decode()) == (_lib.ERR_ARG, "n must be < 2^31"), (fn, cid)
    for s in range(4):
        assert L.nmsm_msm_collect(s, ctypes.cast(out, ctypes.c_void_p), ctypes.byref(inf)) == _lib.ERR_ARG
        assert L.nmsm_last_error().decode() == "nothing submitted on this slot"
    # afterwards: a synchronous MSM and one in flight on every slot
    P, pts, scalars, total = H.soak_inputs("bn254_G1", 500, seed_offset=31)
    exp = H.expected_tuple("bn254_G1", H.expected_from_total(P, total))
    pb, sb = H.pack_points("bn254_G1", pts), H.pack_scalars(scalars)
    assert result("bn254_G1", *nmsm.msm_packed(2, pb, sb, 500)) == exp
    keep = [(ctypes.create_string_buffer(pb, len(pb)), ctypes.create_string_buffer(sb, len(sb))) for _ in range(4)]
    for s in range(4):
        check(L.nmsm_msm_submit(2, ctypes.addressof(keep[s][0]), ctypes.addressof(keep[s][1]), 500, 0, s))
    for s in (3, 2, 1, 0):
        assert collect(s, "bn254_G1") == exp, s


# ------------------------------------------------------------------------------------------------
# sizes above 2^20: host inputs up to 2^24, device-resident above (bounds host memory)
# ------------------------------------------------------------------------------------------------
LARGE = [
    pytest.param("bls12_381_G1", 22, id="bls12_381_G1-2^22"),
    pytest.param("bls12_381_G2", 22, id="bls12_381_G2-2^22"),
    pytest.param("bn254_G1", 24, id="bn254_G1-2^24"),
    pytest.param("secp256k1", 22, id="secp256k1-2^22"),
    pytest.param("ed25519", 22, id="ed25519-2^22"),
    # 2^25 G2 terms: word offsets into the prepared array (4n entries of 48 words) pass 2^32
    pytest.param("bls12_381_G2", 25, id="bls12_381_G2-2^25", marks=pytest.mark.slow),
    # 2^25 G1 terms: byte offsets into the prepared array (2n x 96 B) pass 2^32; 2^26: DESIGN §3's capacity
    pytest.param("bls12_381_G1", 25, id="bls12_381_G1-2^25", marks=pytest.mark.slow),
    pytest.param("bls12_381_G1", 26, id="bls12_381_G1-2^26", marks=pytest.mark.slow),
]


@gpu
@pytest.mark.parametrize("name,log_n", LARGE)
def test_msm_above_2p20(nmsm, release_workspace, name, log_n):
    n = 1 << log_n
    kind = "pageable" if log_n <= 24 else "device"
    require_free(device_memory_needed(name, n), "%s MSM of 2^%d terms" % (name, log_n))
    case = make_case(name, n, 1000 + 10 * log_n + SPLIT[name], kind)
    try:
        got = msm_sync(nmsm, case)
        assert got == case.exp, (case.label, plan(nmsm))
    finally:
        case.free()


@gpu
def test_fixed_base_table_2p22_auto_window(nmsm, release_workspace):
    """nmsm_points_precompute with the automatic window at 2^22 BLS12-381 G1 points, two scalar vectors."""
    name, n = "bls12_381_G1", 1 << 22
    # the table: up to ~13 levels of 2n prepared points
    require_free(device_memory_needed(name, n, extra=13 * 2 * n * 96), "fixed-base table of 2^22 points")
    case = make_case(name, n, 2200, "pageable", keep_k=True)
    ps = nmsm.PointSet(case.cid, case.pts.tobytes(), n)
    s2, exp2 = more_scalars(case, 2201, "pageable")
    try:
        c, levels = ps.precompute(0)
        assert 8 <= c <= 22 and levels >= 1, (c, levels)
        for scalars, exp in ((case.sc, case.exp), (s2, exp2)):
            out, inf = ps.msm(scalars.tobytes(), n)
            assert result(name, out, inf) == exp, (case.label, "table c=%d levels=%d" % (c, levels), plan(nmsm))
            _, info = nmsm.last_timing()
            assert info.windows == 1 and info.c == c, plan(nmsm)
    finally:
        ps.close()
        case.free()
        s2.free()
