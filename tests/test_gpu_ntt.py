"""nmsm_ntt / nmsm_ntt_device (csrc/ntt.cu) checked exactly at every size it supports, 2^0 .. 2^27, in every boundary
layout and direction, on both fields, through both entry points.

The transform runs as ceil(log_n / 10) passes over memory, each up to 10 stages on a 2048-element shared-memory tile;
log_n 1..10 is one pass, 11..20 two, 21..27 three (the middle pass's tile mixes low and high index bits).  The
references (tests/ntt_cases.py) never touch the library:
  * the closed form of a geometric input's transform, checked on every output up to 2^24 and on 2^16 random outputs
    plus a byte-exact round trip above (those sizes are also marked slow);
  * the vectorised restatement of the oracle's fft_core on dense random inputs, up to 2^22;
  * the oracle itself for the residue generators, whose omega is not a primitive root.
Every assertion names the field, log_n, G, direction, layout and entry point, and the first mismatching index.
"""
import ctypes

import numpy as np
import pytest
import torch

import ntt_cases as C

pytestmark = pytest.mark.gpu

CURVE = {"bn254": 2, "bls12_381": 4}  # NMSM_BN254_G1 / NMSM_BLS12_381_G1: their scalar field Fr
ERR_SCALAR = -2
FULL_CHECK_MAX = 24       # every output checked up to 2^24; sampled above
SAMPLES = 1 << 16
BOUNDARIES = (10, 11, 20, 21, 27)  # every layout and direction at the pass-count boundaries and at the largest size


def lib():
    from nmsm import _lib

    return _lib.load()


def check(rc):
    from nmsm import _lib

    _lib.check(rc)


def release():
    """Give back the NTT buffers (four of 32 * 2^log_n bytes, plus slack) and torch's cached blocks."""
    lib().nmsm_shutdown()
    check(lib().nmsm_init(0))
    torch.cuda.empty_cache()


def require_free(log_n, what):
    nbytes = int(5 * 32 * 1.125 * (1 << log_n)) + (1 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("%s needs about %.1f GiB of device memory, %.1f GiB are free (the GPU is shared)"
                    % (what, nbytes / 2**30, free / 2**30))


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    yield m
    release()


@pytest.fixture(scope="module")
def pool():
    """workers for the closed-form checks and geometric inputs"""
    with C.Pool() as p:
        yield p


@pytest.fixture(scope="module")
def ref_pool():
    """workers for the dense references (a minute each at 2^22): kept apart so that the checks never queue behind them"""
    with C.Pool(8) as p:
        yield p


def describe(field, log_n, gen, inv, bi, bo, via):
    return "%s log_n=%d G=%d %s brp_input=%d brp_output=%d via %s" % (
        field, log_n, gen, "inverse" if inv else "direct", bi, bo, via)


def transform(field, log_n, raw, gen, inv, bi, bo, via):
    """one call of nmsm_ntt ("host") or nmsm_ntt_device ("device", a torch buffer); returns the buffer's bytes"""
    args = (log_n, gen, int(inv), int(bi), int(bo))
    if via == "host":
        buf = ctypes.create_string_buffer(raw, len(raw))
        check(lib().nmsm_ntt(CURVE[field], ctypes.cast(buf, ctypes.c_void_p), *args))
        return buf.raw
    t = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
    torch.cuda.synchronize()  # the library runs on its own stream
    check(lib().nmsm_ntt_device(CURVE[field], ctypes.c_void_p(t.data_ptr()), *args))
    out = t.cpu().numpy().tobytes()
    del t
    return out


def first_diff(got, exp):
    g, e = C.rows(got), C.rows(exp)
    bad = np.nonzero((g != e).any(axis=1))[0]
    return int(bad[0]) if len(bad) else -1


def ref_gen(gen):
    return 5 if gen == 0 else gen  # 0 asks the library for its default generator, which is 5 (findGenerator)


# ------------------------------------------------------------------------------------------------
# 1. every size, both fields: geometric inputs against the closed form
# ------------------------------------------------------------------------------------------------
def sweep_cases():
    out = []
    for fi, field in enumerate(C.FIELDS):
        for log_n in range(28):
            marks = [pytest.mark.slow] if log_n > FULL_CHECK_MAX else []
            out.append(pytest.param(field, log_n, marks=marks, id="%s-%d" % (field, log_n)))
    return out


def sweep_combos(field, log_n):
    """all eight at the boundaries; elsewhere one, rotating with log_n, so that each combination meets one, two and
    three passes (log_n 1..10 and 11..20 run all eight in turn; 21..27 are all-eight at 21 and 27)"""
    if log_n in BOUNDARIES:
        return list(C.COMBOS)
    return [C.COMBOS[(log_n + 3 * C.FIELDS.index(field)) % 8]]


@pytest.mark.parametrize("field,log_n", sweep_cases())
def test_every_size_closed_form(nmsm, pool, dense_refs, field, log_n):
    # (dense_refs only starts the dense cases' references here, so that they run beside this sweep)
    require_free(log_n, "a 2^%d NTT" % log_n)
    n = 1 << log_n
    gen = 0 if log_n % 3 == 0 else 7
    c = C.geometric_c(field, log_n, 1000 + log_n)
    natural = C.geometric(field, log_n, c, pool)
    permuted = C.permute_rows(natural, log_n) if log_n else natural
    brp = C.brp_index(log_n)
    try:
        for j, (inv, bi, bo) in enumerate(sweep_combos(field, log_n)):
            via = "device" if (log_n + j) % 2 else "host"
            what = describe(field, log_n, gen, inv, bi, bo, via)
            stored_in = permuted if bi else natural
            out = transform(field, log_n, stored_in, gen, inv, bi, bo, via)
            if log_n <= FULL_CHECK_MAX:
                logical = C.rows(out)[brp].tobytes() if bo else out
                bad = C.closed_form_mismatch(field, ref_gen(gen), log_n, c, inv, logical, pool)
                assert bad == -1, "%s: closed form fails at output %d" % (what, bad)
            else:
                ks = np.sort(np.random.default_rng(log_n * 8 + j).choice(n, SAMPLES, replace=False))
                ks[0], ks[-1] = 0, n - 1
                pos = brp[ks] if bo else ks
                vals = C.unpack(C.rows(out)[pos].tobytes())
                bad = C.closed_form_sample_mismatch(field, ref_gen(gen), log_n, c, inv, ks, vals)
                assert bad == -1, "%s: closed form fails at output %d" % (what, bad)
                # the opposite direction with the layouts swapped gives the stored input back
                back = transform(field, log_n, out, gen, not inv, bo, bi, "host" if via == "device" else "device")
                d = first_diff(back, stored_in)
                assert d == -1, "%s: round trip differs first at element %d" % (what, d)
                del back
            del out
    finally:
        if log_n > FULL_CHECK_MAX:
            del natural, permuted
            release()


# ------------------------------------------------------------------------------------------------
# 2. dense random inputs against the vectorised oracle restatement, every output
# ------------------------------------------------------------------------------------------------
def dense_cases():
    out = []
    for fi, field in enumerate(C.FIELDS):
        for j, combo in enumerate(C.COMBOS):
            out.append((field, 14, 7 if j % 2 else 0, combo))
        for k, log_n in enumerate((17, 20, 21, 22)):
            out.append((field, log_n, (7, 0, 7, 5)[k], C.COMBOS[(3 * k + 5 * fi + 1) % 8]))
    return out


DENSE = dense_cases()


@pytest.fixture(scope="module")
def dense_refs(ref_pool):
    """the references of every dense case, submitted at once (they run beside the GPU tests)"""
    futs = {}
    for case in DENSE:
        field, log_n, gen, (inv, bi, bo) = case
        raw = C.dense_random(field, log_n, 50 + log_n)
        futs[case] = (raw, C.reference_bytes(ref_pool, field, ref_gen(gen), raw, inv, bi, bo))
    return futs


@pytest.mark.parametrize("case", DENSE, ids=["%s-%d-G%d-%d%d%d" % (f, n, g, *c) for f, n, g, c in DENSE])
def test_dense_random_matches_reference(nmsm, dense_refs, case):
    field, log_n, gen, (inv, bi, bo) = case
    raw, fut = dense_refs[case]
    exp = fut.result()
    for via in (("host", "device") if log_n <= 17 else ("device" if log_n % 2 else "host",)):
        got = transform(field, log_n, raw, gen, inv, bi, bo, via)
        d = first_diff(got, exp)
        assert d == -1, "%s: dense random input, first mismatch at element %d" % (describe(field, log_n, gen, inv, bi, bo, via), d)


def test_all_top_elements(nmsm):
    """every element r - 1: the largest sums and differences in every butterfly"""
    for field in C.FIELDS:
        for log_n, (inv, bi, bo) in ((12, C.COMBOS[0]), (13, C.COMBOS[7]), (16, C.COMBOS[5])):
            raw = C.all_top(field, log_n)
            exp = C.pack(C.fft(C.FR[field], 7, C.unpack(raw), inv, bi, bo))
            got = transform(field, log_n, raw, 7, inv, bi, bo, "host")
            d = first_diff(got, exp)
            assert d == -1, "%s: all r - 1, first mismatch at %d" % (describe(field, log_n, 7, inv, bi, bo, "host"), d)


# ------------------------------------------------------------------------------------------------
# 3. generators
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("field", C.FIELDS)
def test_generators(nmsm, pool, field):
    """7, the default (0, which must equal 5), 5, 2^64 - 1 (the top word of k_ntt_setup's G) and the residues 1, 2, 4,
    against the oracle restatement, in one and two passes; 0 and 5 give identical bytes"""
    p = C.FR[field]
    for gi, gen in enumerate((7, 0, 5, 2**64 - 1, 1, 2, 4)):
        for log_n in (3, 10, 11, 12, 13):
            raw = C.dense_random(field, log_n, 7 * gi + log_n)
            for j in range(2):
                inv, bi, bo = C.COMBOS[(gi + log_n + 4 * j) % 8]
                via = ("host", "device")[j]
                exp = C.pack(C.fft(p, ref_gen(gen), C.unpack(raw), inv, bi, bo))
                got = transform(field, log_n, raw, gen, inv, bi, bo, via)
                d = first_diff(got, exp)
                assert d == -1, "%s: first mismatch at %d" % (describe(field, log_n, gen, inv, bi, bo, via), d)
    raw = C.dense_random(field, 16, 3)
    assert transform(field, 16, raw, 0, False, False, False, "host") == transform(field, 16, raw, 5, False, False, False, "device")
    if C.is_non_residue(p, 2**64 - 1):  # bn254: the closed form holds for this G too, at three passes
        c = C.geometric_c(field, 21, 4)
        out = transform(field, 21, C.geometric(field, 21, c, pool), 2**64 - 1, False, False, False, "device")
        bad = C.closed_form_mismatch(field, 2**64 - 1, 21, c, False, out, pool)
        assert bad == -1, "%s: closed form fails at %d" % (describe(field, 21, 2**64 - 1, 0, 0, 0, "device"), bad)


# ------------------------------------------------------------------------------------------------
# 4. the root-table cache (ntt_key_field / ntt_key_gen / ntt_key_bits)
# ------------------------------------------------------------------------------------------------
CACHE_SEQUENCE = (
    ("bn254", 7, 12, False),
    ("bls12_381", 7, 12, False),   # same size and G, other field
    ("bls12_381", 5, 12, False),
    ("bls12_381", 0, 12, False),   # the default after an explicit 5
    ("bls12_381", 5, 13, False),
    ("bn254", 7, 12, False),       # back to the first key
    ("bn254", 7, 12, True),        # inverse on the cached table
    ("bls12_381", 7, 20, False),
    ("bls12_381", 7, 11, True),    # shrink: the table is rebuilt inside the larger buffer
    ("bls12_381", 7, 20, True),    # regrow into the same buffer
)


def test_root_table_cache(nmsm, pool):
    for rnd in range(2):
        for i, (field, gen, log_n, inv) in enumerate(CACHE_SEQUENCE):
            bi, bo = bool(i % 2), bool(i % 3 == 0)
            via = ("host", "device")[(i + rnd) % 2]
            what = "round %d step %d: %s" % (rnd, i, describe(field, log_n, gen, inv, bi, bo, via))
            if log_n <= 13:
                raw = C.dense_random(field, log_n, 300 + i)
                exp = C.pack(C.fft(C.FR[field], ref_gen(gen), C.unpack(raw), inv, bi, bo))
                d = first_diff(transform(field, log_n, raw, gen, inv, bi, bo, via), exp)
                assert d == -1, "%s: first mismatch at %d" % (what, d)
            else:
                c = C.geometric_c(field, log_n, 300 + i)
                nat = C.geometric(field, log_n, c, pool)
                out = transform(field, log_n, C.permute_rows(nat, log_n) if bi else nat, gen, inv, bi, bo, via)
                logical = C.permute_rows(out, log_n) if bo else out
                bad = C.closed_form_mismatch(field, ref_gen(gen), log_n, c, inv, logical, pool)
                assert bad == -1, "%s: closed form fails at %d" % (what, bad)
        release()  # the same sequence again on a fresh context


# ------------------------------------------------------------------------------------------------
# 5. invalid elements at scale, and the ABI's size limits
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("field", C.FIELDS)
def test_invalid_elements_at_scale(nmsm, pool, field):
    log_n = 22
    require_free(log_n, "a 2^22 NTT")
    n, p = 1 << log_n, C.FR[field]
    c = C.geometric_c(field, log_n, 77)
    good = C.geometric(field, log_n, c, pool)
    transform(field, 10, C.dense_random(field, 10, 1), 3, False, False, False, "host")  # another key in the cache
    bad_at = sorted({n - 1, (1 << 21) + 12345, 3 << 20, (1 << 21) + 12347, n - 2})
    rows = C.rows(good).copy()
    for j, i in enumerate(bad_at):
        rows[i] = np.frombuffer(C.INVALID(p)[j % 4].to_bytes(32, "little"), dtype=np.uint8)
    planted = rows.tobytes()
    for via in ("host", "device"):
        for inv, bi, bo in (C.COMBOS[0], C.COMBOS[6]):
            what = describe(field, log_n, 7, inv, bi, bo, via)
            args = (CURVE[field], None, log_n, 7, int(inv), int(bi), int(bo))
            if via == "host":
                buf = ctypes.create_string_buffer(planted, len(planted))
                rc = lib().nmsm_ntt(args[0], ctypes.cast(buf, ctypes.c_void_p), *args[2:])
                after = buf.raw
            else:
                t = torch.frombuffer(bytearray(planted), dtype=torch.uint8).cuda()
                torch.cuda.synchronize()
                rc = lib().nmsm_ntt_device(args[0], ctypes.c_void_p(t.data_ptr()), *args[2:])
                after = t.cpu().numpy().tobytes()
                del t
            assert rc == ERR_SCALAR, "%s: rc %d" % (what, rc)
            assert lib().nmsm_last_error_index() == bad_at[0], what
            assert ("invalid field element at index %d" % bad_at[0]).encode() in lib().nmsm_last_error(), what
            d = first_diff(after, planted)
            assert d == -1, "%s: the caller's buffer changed at element %d" % (what, d)
            # the next valid call on the same key is exact: the failed call left a usable table
            out = transform(field, log_n, C.permute_rows(good, log_n) if bi else good, 7, inv, bi, bo, via)
            logical = C.permute_rows(out, log_n) if bo else out
            m = C.closed_form_mismatch(field, 7, log_n, c, inv, logical, pool)
            assert m == -1, "%s: after the rejected call, closed form fails at %d" % (what, m)


def test_abi_size_limits(nmsm):
    dummy = ctypes.create_string_buffer(b"\x01" * 64, 64)
    ptr = ctypes.cast(dummy, ctypes.c_void_p)
    for log_n in range(28, 32):
        assert lib().nmsm_ntt(4, ptr, log_n, 7, 0, 0, 0) != 0, log_n
        assert b"above 2^27" in lib().nmsm_last_error(), log_n
    for log_n in (32, 33):  # the reference's own limit (bits > 31), then BLS12-381's 2-adicity
        assert lib().nmsm_ntt(4, ptr, log_n, 7, 0, 0, 0) != 0, log_n
        assert b"wrong bits %d" % log_n in lib().nmsm_last_error(), log_n
    assert lib().nmsm_ntt(2, ptr, 28, 7, 0, 0, 0) != 0 and b"above 2^27" in lib().nmsm_last_error()
    assert lib().nmsm_ntt(2, ptr, 29, 7, 0, 0, 0) != 0 and b"wrong bits 29 powerOfTwo=28" in lib().nmsm_last_error()
    for curve in (2, 4):
        assert lib().nmsm_ntt(curve, ptr, -1, 7, 0, 0, 0) != 0 and b"wrong bits -1" in lib().nmsm_last_error()
    assert dummy.raw == b"\x01" * 64
    # the library still works afterwards
    raw = C.dense_random("bn254", 1, 0)
    assert transform("bn254", 1, raw, 7, False, False, False, "host") == C.pack(C.fft(C.FR["bn254"], 7, C.unpack(raw), False, False, False))


# ------------------------------------------------------------------------------------------------
# 6. a context re-bound to another device
# ------------------------------------------------------------------------------------------------
def test_reinit_on_another_device(nmsm):
    """The 64 KB shared-memory opt-in of the pass kernels belongs to a device's context: after nmsm_shutdown /
    nmsm_init(1), a two-pass transform still launches and is exact."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible CUDA devices")
    field, log_n = "bls12_381", 12
    raw = C.dense_random(field, log_n, 8)
    exp = C.pack(C.fft(C.FR[field], 7, C.unpack(raw), False, False, False))
    assert transform(field, log_n, raw, 7, False, False, False, "host") == exp  # the opt-in is set on device 0 first
    lib().nmsm_shutdown()
    try:
        check(lib().nmsm_init(1))
        got = transform(field, log_n, raw, 7, False, False, False, "host")
        d = first_diff(got, exp)
        assert d == -1, "device 1: %s: first mismatch at %d" % (describe(field, log_n, 7, 0, 0, 0, "host"), d)
    finally:
        lib().nmsm_shutdown()
        check(lib().nmsm_init(0))
