"""Host-side mirror of the reference's NTT interface over the C ABI (nmsm_ntt, include/nmsm.h).

    roots = rootsOfUnity("bls12_381", 7)      # /root/reference/src/abstract/fft.ts:230  rootsOfUnity(Fr, generator)
    fft = FFT(roots)                           # fft.ts:518  FFT(roots, Fr)
    evals = fft.direct(coeffs)                 # fft.ts:552  direct(values, brpInput=False, brpOutput=False)
    coeffs = fft.inverse(evals)                # fft.ts:559

Values are Python ints in [0, r); the transform runs on the GPU (no CPU fallback: NmsmError without a device).
`ntt_packed` is the typed-array fast path (n * 32 bytes, little-endian), `ntt_device` the zero-copy one.

The generator G is an element of Fr, so it is taken mod r, as the reference's pow(G, oddFactor, r) does: G and G + r
give the same transform.  The C ABI carries G in 64 bits and reads 0 as "the default generator (5)".  A G whose
residue mod r is 0 or does not fit in 64 bits therefore raises ValueError before anything reaches the library; it is
never truncated.  `ntt_packed` / `ntt_device` keep the ABI's convention that generator=0 asks for the default.
"""
import ctypes

from . import _lib
from ._lib import NmsmError

# curve ids whose scalar field Fr the transform runs over (include/nmsm.h)
FIELD_CURVE = {"bn254": 2, "bls12_381": 4}
FR_ORDER = {
    "bn254": 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001,
    "bls12_381": 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001,
}
TWO_ADICITY = {"bn254": 28, "bls12_381": 32}


def _is_pow2(n: int) -> bool:
    return n != 0 and (n & (n - 1)) == 0


def abi_generator(field: str, generator: int) -> int:
    """G mod r as the 64-bit value nmsm_ntt takes (0 stays 0: the default generator)."""
    if generator == 0:
        return 0
    g = generator % FR_ORDER[field]
    if g == 0:
        raise ValueError("rootsOfUnity: generator %d is 0 mod r" % generator)
    if g >= 1 << 64:
        raise ValueError("rootsOfUnity: generator %d is %d mod r, which does not fit in the 64-bit generator argument"
                         % (generator, g))
    return g


def ntt_packed(field: str, values: bytes, log_n: int, inverse=False, brp_input=False, brp_output=False, generator=0) -> bytes:
    """2^log_n canonical little-endian 32-byte elements in, transformed elements out."""
    n = 1 << log_n
    if len(values) != n * 32:
        raise ValueError("FFT: wrong Polynomial length")
    generator = abi_generator(field, generator)
    _lib.ensure_init()
    lib = _lib.load()
    buf = ctypes.create_string_buffer(bytes(values), n * 32)
    rc = lib.nmsm_ntt(FIELD_CURVE[field], ctypes.cast(buf, ctypes.c_void_p), log_n, generator, 1 if inverse else 0,
                      1 if brp_input else 0, 1 if brp_output else 0)
    try:
        _lib.check(rc)
    except NmsmError as e:
        raise ValueError(str(e)) from e
    return buf.raw[: n * 32]


def ntt_device(field: str, d_values: int, log_n: int, inverse=False, brp_input=False, brp_output=False, generator=0) -> None:
    """In place on a device buffer (raw device pointer, 16-byte aligned)."""
    generator = abi_generator(field, generator)
    _lib.ensure_init()
    rc = _lib.load().nmsm_ntt_device(FIELD_CURVE[field], ctypes.c_void_p(d_values), log_n, generator,
                                      1 if inverse else 0, 1 if brp_input else 0, 1 if brp_output else 0)
    try:
        _lib.check(rc)
    except NmsmError as e:
        raise ValueError(str(e)) from e


class RootsOfUnity:
    """The part of fft.ts:182-312 a caller of FFT() needs: field, generator, 2-adicity (tables live on the GPU)."""

    def __init__(self, field: str, generator=None):
        if field not in FIELD_CURVE:
            raise ValueError("rootsOfUnity: scalar fields of bn254 and bls12_381 only")
        if generator is not None and not isinstance(generator, int):
            raise TypeError('"generator" expected bigint, got type=' + type(generator).__name__)
        if generator is not None and generator % FR_ORDER[field] == 0:
            raise ValueError("rootsOfUnity: generator %d is 0 mod r" % generator)
        # the value passed to the library: G mod r, or 0 for the default
        self.field, self.generator = field, (0 if generator is None else abi_generator(field, generator))
        self.info = {"G": generator if generator is not None else 5, "powerOfTwo": TWO_ADICITY[field],
                     "oddFactor": (FR_ORDER[field] - 1) >> TWO_ADICITY[field]}


def rootsOfUnity(field: str, generator=None) -> RootsOfUnity:
    return RootsOfUnity(field, generator)


class FFT:
    """fft.ts:518-575 for Fr of bn254 / BLS12-381."""

    def __init__(self, roots: RootsOfUnity):
        self.roots = roots

    def _run(self, values, inverse, brp_input, brp_output):
        n = len(values)
        if not _is_pow2(n):
            raise ValueError("FFT: Polynomial size should be power of two")
        bits = n.bit_length() - 1
        if bits > 31 or bits > TWO_ADICITY[self.roots.field]:
            raise ValueError("rootsOfUnity: wrong bits %d powerOfTwo=%d" % (bits, TWO_ADICITY[self.roots.field]))
        r = FR_ORDER[self.roots.field]
        packed = b"".join((v % r if v < 0 else v).to_bytes(32, "little") for v in values)
        out = ntt_packed(self.roots.field, packed, bits, inverse, brp_input, brp_output, self.roots.generator)
        return [int.from_bytes(out[i * 32:(i + 1) * 32], "little") for i in range(n)]

    def direct(self, values, brpInput=False, brpOutput=False):
        return self._run(values, False, brpInput, brpOutput)

    def inverse(self, values, brpInput=False, brpOutput=False):
        return self._run(values, True, brpInput, brpOutput)
