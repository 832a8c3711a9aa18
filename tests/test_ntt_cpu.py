"""The NTT's CPU side: the references of tests/ntt_cases.py pinned to oracle/noble_fft, and the Python mirror's
handling of the generator (nmsm/fft.py), which must be settled before any call reaches the library.  No device."""
import random

import numpy as np
import pytest

import ntt_cases as C
from nmsm import fft as GF
from oracle import noble_fft as OF


@pytest.mark.parametrize("field", C.FIELDS)
def test_vectorised_reference_matches_oracle(field):
    """ntt_cases.fft == noble_fft.FFT for log_n 0..12, every layout, both directions, generators 5, 7, 2, 4."""
    p = C.FR[field]
    rnd = random.Random(5)
    for gen in (5, 7, 2, 4):
        oracle = OF.FFT(OF.RootsOfUnity(p, gen))
        for bits in range(13):
            n = 1 << bits
            a = [rnd.randrange(p) for _ in range(n)]
            a[0], a[-1] = p - 1, 0
            for inv, bi, bo in C.COMBOS:
                if bits > 9 and (bits + gen + 2 * bi + bo) % 4:  # every layout at every size up to 2^9, a quarter above
                    continue
                exp = (oracle.inverse if inv else oracle.direct)(a, bi, bo)
                got = C.fft(p, gen, a, inv, bi, bo)
                assert list(got) == exp, (field, gen, bits, "inverse" if inv else "direct", bi, bo)


def test_vectorised_reference_fft_core_both_flavours():
    """fft_core itself (DIT with and without the input permutation, DIF with and without the output one)."""
    p = C.FR["bn254"]
    rnd = random.Random(6)
    for bits in (0, 1, 3, 8, 11):
        n = 1 << bits
        a = [rnd.randrange(p) for _ in range(n)]
        roots = OF.RootsOfUnity(p, 7).roots(bits)
        for dit in (False, True):
            for brp in (False, True):
                assert list(C.fft_core(p, np.array(a, dtype=object), np.array(roots, dtype=object), dit, brp)) == \
                    OF.fft_core(p, a, roots, dit, brp), (bits, dit, brp)


def test_helpers():
    p = C.FR["bls12_381"]
    for n, start in ((1, 0), (5, 3), (64, 0), (1000, 77)):
        assert list(C.powers(3, n, p, start)) == [pow(3, start + i, p) for i in range(n)]
    for bits in range(9):
        assert list(C.brp_index(bits)) == [OF.reverse_bits(i, bits) for i in range(1 << bits)]
    vals = [random.Random(1).randrange(p) for _ in range(16)]
    raw = C.pack(vals)
    assert list(C.unpack(raw)) == vals
    assert list(C.unpack(C.permute_rows(raw, 4))) == OF.bit_reversal_permutation(vals)
    for field in C.FIELDS:
        p = C.FR[field]
        d = C.unpack(C.dense_random(field, 12, 3))
        assert max(d) < p and min(d) == 0 and p - 1 in set(d) and len(set(d)) > 4000
        assert set(C.unpack(C.all_top(field, 3))) == {p - 1}
        assert all(v >= p for v in C.INVALID(p)) and all(v < 1 << 256 for v in C.INVALID(p))
        for g in C.NON_RESIDUES:
            assert C.is_non_residue(p, g)
        for g in C.RESIDUES:
            assert not C.is_non_residue(p, g)
    assert C.is_non_residue(C.FR["bn254"], 2**64 - 1) and not C.is_non_residue(C.FR["bls12_381"], 2**64 - 1)
    assert [C.npass(n) for n in (0, 1, 10, 11, 20, 21, 27)] == [0, 1, 1, 2, 2, 3, 3]


@pytest.mark.parametrize("field", C.FIELDS)
def test_closed_form_matches_oracle(field):
    """The closed form holds exactly on the oracle's own outputs, every layout, log_n 0..10, G in {5, 7}; it fails on
    an output that is off in one element."""
    p = C.FR[field]
    for gen in C.NON_RESIDUES:
        oracle = OF.FFT(OF.RootsOfUnity(p, gen))
        for bits in range(11):
            c = C.geometric_c(field, bits, 100 + bits)
            logical = list(C.unpack(C.geometric(field, bits, c)))
            assert logical == [pow(c, i, p) for i in range(1 << bits)]
            for inv, bi, bo in C.COMBOS:
                stored_in = OF.bit_reversal_permutation(logical) if bi else logical
                out = (oracle.inverse if inv else oracle.direct)(stored_in, bi, bo)
                nat = OF.bit_reversal_permutation(out) if bo else out
                raw = C.pack(nat)
                assert C.closed_form_mismatch(field, gen, bits, c, inv, raw) == -1, (field, gen, bits, inv, bi, bo)
                ks = list(range(1 << bits))
                assert C.closed_form_sample_mismatch(field, gen, bits, c, inv, ks, nat) == -1
                if bits >= 2:
                    k = (5 * bits + 1) % (1 << bits)
                    wrong = list(nat)
                    wrong[k] = (wrong[k] + 1) % p
                    assert C.closed_form_mismatch(field, gen, bits, c, inv, C.pack(wrong)) == k
                    # a layout mistake (output left bit-reversed) breaks it too
                    assert C.closed_form_mismatch(field, gen, bits, c, inv, C.pack(OF.bit_reversal_permutation(nat))) >= 0
    with pytest.raises(AssertionError, match="residue"):
        C.omega(field, 4, 8)


def test_closed_form_chunked_in_pool(monkeypatch):
    """The pooled paths (chunked geometric input, chunked check, reference jobs) agree with the single-process ones;
    the first bad index is found in a chunk other than the first."""
    monkeypatch.setattr(C, "CHUNK", 1 << 10)  # the parent splits the work: 4 chunks at 2^12
    field, bits = "bn254", 12
    p = C.FR[field]
    c = C.geometric_c(field, bits, 9)
    with C.Pool(2) as pool:
        raw = C.geometric(field, bits, c, pool)
        assert raw == C.geometric(field, bits, c)
        out = C.pack(C.fft(p, 7, C.unpack(raw), False, False, False))
        assert C.closed_form_mismatch(field, 7, bits, c, False, out, pool) == -1
        bad = bytearray(out)
        k = (1 << bits) - 3
        bad[k * 32] ^= 1
        assert C.closed_form_mismatch(field, 7, bits, c, False, bytes(bad), pool) == k
        fut = C.reference_bytes(pool, field, 7, C.dense_random(field, 10, 1), True, True, False)
        assert fut.result() == C.pack(OF.FFT(OF.RootsOfUnity(p, 7)).inverse(list(C.unpack(C.dense_random(field, 10, 1))),
                                                                             True, False))


# ------------------------------------------------------------------------------------------------
# the mirror's generator: G mod r, 64 bits, 0 is not "the default"
# ------------------------------------------------------------------------------------------------
class FakeLib:
    """Records what would reach nmsm_ntt / nmsm_ntt_device and leaves the buffer as it is."""

    def __init__(self):
        self.calls = []

    def nmsm_ntt(self, curve, buf, log_n, generator, inverse, bi, bo):
        self.calls.append(("host", curve, log_n, generator))
        return 0

    def nmsm_ntt_device(self, curve, ptr, log_n, generator, inverse, bi, bo):
        self.calls.append(("device", curve, log_n, generator))
        return 0


@pytest.fixture
def fake_lib(monkeypatch):
    fake = FakeLib()
    monkeypatch.setattr(GF._lib, "ensure_init", lambda: None)
    monkeypatch.setattr(GF._lib, "load", lambda: fake)
    return fake


@pytest.fixture
def no_lib(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("reached the library")

    monkeypatch.setattr(GF._lib, "ensure_init", refuse)
    monkeypatch.setattr(GF._lib, "load", refuse)


@pytest.mark.parametrize("field", C.FIELDS)
def test_generator_reduced_mod_r(field, fake_lib):
    """G and G + r name the same roots (the oracle's pow(G, odd, r)); the ABI gets G mod r."""
    r = C.FR[field]
    assert OF.RootsOfUnity(r, r + 7).omega(10) == OF.RootsOfUnity(r, 7).omega(10)
    GF.FFT(GF.rootsOfUnity(field, r + 7)).direct([1, 2, 3, 4])
    GF.FFT(GF.rootsOfUnity(field, 5 * r + 2**64 - 1)).inverse([1, 2])
    GF.FFT(GF.rootsOfUnity(field)).direct([1])
    GF.ntt_packed(field, bytes(64), 1, generator=3 * r + 11)
    GF.ntt_packed(field, bytes(64), 1)
    GF.ntt_device(field, 0x1000, 4, generator=r + 5)
    curve = GF.FIELD_CURVE[field]
    assert fake_lib.calls == [("host", curve, 2, 7), ("host", curve, 1, 2**64 - 1), ("host", curve, 0, 0),
                              ("host", curve, 1, 11), ("host", curve, 1, 0), ("device", curve, 4, 5)]
    assert GF.rootsOfUnity(field, r + 7).generator == 7 and GF.rootsOfUnity(field, r + 7).info["G"] == r + 7


@pytest.mark.parametrize("field", C.FIELDS)
def test_generator_out_of_abi_range_raises_before_the_library(field, no_lib):
    """2^64 + 7 used to reach the library as 7 (ctypes wraps c_uint64), -1 as 2^64 - 1, and 0 or r meant the
    default 5.  Each is now a ValueError raised on the host."""
    r = C.FR[field]
    for g in (2**64 + 7, 2**64, -1, -5, r - 1, 2**200):
        with pytest.raises(ValueError, match="does not fit in the 64-bit generator"):
            GF.rootsOfUnity(field, g)
        with pytest.raises(ValueError, match="does not fit in the 64-bit generator"):
            GF.ntt_packed(field, bytes(32), 0, generator=g)
        with pytest.raises(ValueError, match="does not fit in the 64-bit generator"):
            GF.ntt_device(field, 0x1000, 0, generator=g)
    for g in (0, r, 7 * r, -r):
        with pytest.raises(ValueError, match="is 0 mod r"):
            GF.rootsOfUnity(field, g)
    for g in (r, -r):
        with pytest.raises(ValueError, match="is 0 mod r"):
            GF.ntt_packed(field, bytes(32), 0, generator=g)
