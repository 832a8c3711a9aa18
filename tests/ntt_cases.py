"""Exact references and inputs for the NTT over Fr of bn254 and BLS12-381 (nmsm_ntt, csrc/ntt.cu).  CPU only.

Two references, both independent of the library:

* `fft` restates oracle/noble_fft.fft_core / FFT (DIT and DIF stage loops, the brp boundary, inverse with 1/N) on
  numpy object arrays of Python ints, one whole stage per array operation.  Same arithmetic, same twiddle indices,
  roughly 1.5x faster than the list-based oracle; still about a minute per transform at 2^22.
* `closed_form_mismatch` checks a transform of a geometric input a_i = c^i without running one.  With omega a
  primitive N-th root of unity and c^N != 1,
      direct(a)[k]  = sum_i (c omega^k)^i    = (c^N - 1) / (c omega^k - 1)
      inverse(a)[i] = N^-1 sum_k (c omega^-i)^k = N^-1 (c^N - 1) / (c omega^-i - 1)
  so out[k] * (c omega^(+-k) - 1) == (c^N - 1) (times N^-1 for the inverse), with no inversion per output.  The input
  is dense, so every twiddle of every stage reaches the outputs.  omega comes from oracle/noble_fft.RootsOfUnity,
  which is primitive only for a non-residue G (5, 7; 2^64 - 1 on bn254): residues are compared with the oracle.

Layouts: with brp_input the stored input x is the logical input in bit-reversed order, x[j] = a[brp(j)]; with
brp_output the stored output y holds out[brp(j)] at j.  Elements travel as 32-byte little-endian rows.

The heavy loops run in worker processes (`Pool`, spawned: the workers import numpy and this module only, never torch
or CUDA), so that the references keep up with the GPU at 2^20 .. 2^27.
"""
import concurrent.futures
import multiprocessing
import os

import numpy as np

from oracle import noble_fft as OF

FIELDS = ("bn254", "bls12_381")
FR = OF.FR
TWO_ADICITY = {"bn254": 28, "bls12_381": 32}
NON_RESIDUES = (5, 7)          # both fields; the default generator is 5
RESIDUES = (1, 2, 3, 4)        # both fields: omega is not a primitive root, the closed form does not hold
CHUNK = 1 << 18                # elements per worker job
# (inverse, brp_input, brp_output), the order sizes rotate through
COMBOS = tuple((inv, bi, bo) for inv in (False, True) for bi in (False, True) for bo in (False, True))
INVALID = lambda p: (p, p + 1, 1 << 255, (1 << 256) - 1)  # noqa: E731  elements >= r


def is_non_residue(p: int, g: int) -> bool:
    return pow(g, p >> 1, p) == p - 1


def npass(log_n: int) -> int:
    """passes csrc/ntt.cu splits a transform of 2^log_n into (10 stages at most per pass)"""
    return (log_n + 9) // 10 if log_n else 0


# ------------------------------------------------------------------------------------------------
# element packing and permutations
# ------------------------------------------------------------------------------------------------
def pack(values) -> bytes:
    return b"".join(int(v).to_bytes(32, "little") for v in values)


def unpack(raw) -> np.ndarray:
    mv = memoryview(raw)
    return np.array([int.from_bytes(mv[i:i + 32], "little") for i in range(0, len(mv), 32)], dtype=object)


def rows(raw) -> np.ndarray:
    """bytes -> (n, 32) uint8 view"""
    return np.frombuffer(raw, dtype=np.uint8).reshape(-1, 32)


def brp_index(bits: int) -> np.ndarray:
    """brp(j) for j < 2^bits, as an index array"""
    i = np.arange(1 << bits, dtype=np.int64)
    r = np.zeros_like(i)
    for b in range(bits):
        r |= ((i >> b) & 1) << (bits - 1 - b)
    return r


def permute_rows(raw, bits: int) -> bytes:
    """bit-reversal permutation of 2^bits 32-byte rows (an involution)"""
    return rows(raw)[brp_index(bits)].tobytes()


# ------------------------------------------------------------------------------------------------
# powers and the vectorised restatement of fft_core
# ------------------------------------------------------------------------------------------------
def powers(x: int, n: int, p: int, start: int = 0) -> np.ndarray:
    """[x^start, x^(start+1), ..., x^(start+n-1)] mod p as an outer product of two ~sqrt(n)-sized power tables"""
    if n == 0:
        return np.zeros(0, dtype=object)
    lo_n = 1 << ((max(n, 1) - 1).bit_length() + 1) // 2
    lo, cur = [], 1
    for _ in range(lo_n):
        lo.append(cur)
        cur = cur * x % p
    step = cur  # x^lo_n
    hi_n = -(-n // lo_n)
    hi, cur = [], pow(x, start, p)
    for _ in range(hi_n):
        hi.append(cur)
        cur = cur * step % p
    out = (np.array(hi, dtype=object)[:, None] * np.array(lo, dtype=object)[None, :]) % p
    return out.ravel()[:n]


def fft_core(p: int, values: np.ndarray, roots: np.ndarray, dit: bool, brp: bool = True) -> np.ndarray:
    """oracle/noble_fft.fft_core, one stage per array operation; returns a new array"""
    n = len(values)
    assert n and n & (n - 1) == 0 and len(roots) == n
    bits = n.bit_length() - 1
    v = np.array(values, dtype=object)
    if dit and brp:
        v = v[brp_index(bits)]
    for i in range(bits):
        s = i + 1 if dit else bits - i
        m = 1 << s
        m2 = m >> 1
        stride = n >> s
        w = roots[0:m2 * stride:stride]  # roots[j * stride], j < m2
        blk = v.reshape(n // m, 2, m2)
        a, b = blk[:, 0, :], blk[:, 1, :]
        if dit:
            t = b * w % p
            a2, b2 = (a + t) % p, (a - t) % p
        else:
            a2, b2 = (a + b) % p, (a - b) * w % p
        blk[:, 0, :] = a2
        blk[:, 1, :] = b2
    if not dit and brp:
        v = v[brp_index(bits)]
    return v


def fft(p: int, generator, values, inverse: bool, brp_input: bool, brp_output: bool) -> np.ndarray:
    """oracle/noble_fft.FFT(RootsOfUnity(p, generator)).direct / .inverse on a stored (layout-ordered) input"""
    values = np.asarray(values, dtype=object)
    n = len(values)
    bits = n.bit_length() - 1
    w = OF.RootsOfUnity(p, generator).omega(bits)
    roots = powers(w, n, p)
    if inverse:
        roots = roots[(-np.arange(n)) % n]  # [r0] + r[1:][::-1]
    if brp_input and brp_output:
        res = fft_core(p, values[brp_index(bits)], roots, dit=False, brp=False)
    elif brp_input:
        res = fft_core(p, values, roots, dit=True, brp=False)
    elif brp_output:
        res = fft_core(p, values, roots, dit=False, brp=False)
    else:
        res = fft_core(p, values, roots, dit=True, brp=True)
    if inverse:
        res = res * pow(n, -1, p) % p
    return res


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
def dense_random(field: str, log_n: int, seed: int) -> bytes:
    """fixed-seed elements below r, with 0 and r - 1 planted at the ends and in the middle"""
    p = FR[field]
    n = 1 << log_n
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    a[:, 31] = rng.integers(0, p >> 248, size=n, dtype=np.uint8)  # < (p >> 248) * 2^248 <= p
    top = np.frombuffer((p - 1).to_bytes(32, "little"), dtype=np.uint8)
    for i, v in ((0, top), (n - 1, 0), (n // 2, 0), (n // 3, top)):
        a[i] = v
    return a.tobytes()


def all_top(field: str, log_n: int) -> bytes:
    """every element r - 1"""
    return (FR[field] - 1).to_bytes(32, "little") * (1 << log_n)


def geometric_c(field: str, log_n: int, seed: int) -> int:
    """a random c with c^N != 1 (so that every c omega^k != 1 when omega is primitive)"""
    p = FR[field]
    rng = np.random.default_rng(seed)
    while True:
        c = int.from_bytes(rng.bytes(32), "little") % p
        if c > 1 and pow(c, 1 << log_n, p) != 1:
            return c


def _geometric_chunk(p, c, start, count):
    return pack(powers(c, count, p, start))


def geometric(field: str, log_n: int, c: int, pool=None) -> bytes:
    """a_i = c^i, i < 2^log_n (natural order)"""
    p, n = FR[field], 1 << log_n
    if pool is None or n <= CHUNK:
        return _geometric_chunk(p, c, 0, n)
    return b"".join(pool.map(_geometric_chunk, [p] * (n // CHUNK), [c] * (n // CHUNK), range(0, n, CHUNK),
                             [CHUNK] * (n // CHUNK)))


# ------------------------------------------------------------------------------------------------
# the closed-form check
# ------------------------------------------------------------------------------------------------
def omega(field: str, generator: int, log_n: int) -> int:
    """omega of the oracle (never the library's), asserted primitive"""
    p = FR[field]
    w = OF.RootsOfUnity(p, generator).omega(log_n)
    assert log_n == 0 or pow(w, 1 << (log_n - 1), p) == p - 1, "omega is not primitive: G=%d is a residue" % generator
    return w


def closed_form_rhs(field: str, log_n: int, c: int, inverse: bool) -> int:
    p = FR[field]
    rhs = (pow(c, 1 << log_n, p) - 1) % p
    return rhs * pow(1 << log_n, -1, p) % p if inverse else rhs


def _closed_form_chunk(p, c, w, rhs, logical_raw, k0):
    """first k (absolute) in [k0, k0 + len) with out[k] * (c w^k - 1) != rhs, or -1"""
    out = unpack(logical_raw)
    d = (c * powers(w, len(out), p, k0) - 1) % p
    bad = np.nonzero((out * d) % p != rhs)[0]
    return int(bad[0]) + k0 if len(bad) else -1


def closed_form_mismatch(field: str, generator: int, log_n: int, c: int, inverse: bool, logical_raw, pool=None) -> int:
    """first output index whose value breaks the closed form, or -1; `logical_raw` is the output in natural order"""
    p, n = FR[field], 1 << log_n
    w = omega(field, generator, log_n)
    if inverse:
        w = pow(w, -1, p)
    rhs = closed_form_rhs(field, log_n, c, inverse)
    if pool is None or n <= CHUNK:
        return _closed_form_chunk(p, c, w, rhs, logical_raw, 0)
    mv = memoryview(logical_raw)
    jobs = [pool.submit(_closed_form_chunk, p, c, w, rhs, bytes(mv[k * 32:(k + CHUNK) * 32]), k) for k in range(0, n, CHUNK)]
    bad = [j.result() for j in jobs]
    bad = [b for b in bad if b >= 0]
    return min(bad) if bad else -1


def closed_form_sample_mismatch(field: str, generator: int, log_n: int, c: int, inverse: bool, ks, values) -> int:
    """the closed form at the output indices ks only (values[t] = out[ks[t]]); first failing k or -1"""
    p = FR[field]
    w = omega(field, generator, log_n)
    if inverse:
        w = pow(w, -1, p)
    rhs = closed_form_rhs(field, log_n, c, inverse)
    for k, v in zip(ks, values):
        if v * (c * pow(w, int(k), p) - 1) % p != rhs:
            return int(k)
    return -1


# ------------------------------------------------------------------------------------------------
# worker pool
# ------------------------------------------------------------------------------------------------
def _reference_job(field, generator, raw, inverse, brp_input, brp_output):
    return pack(fft(FR[field], generator, unpack(raw), inverse, brp_input, brp_output))


def reference_bytes(pool, field, generator, raw, inverse, brp_input, brp_output):
    """future of the vectorised reference's output (stored layout) as bytes"""
    return pool.submit(_reference_job, field, generator, raw, inverse, brp_input, brp_output)


def Pool(max_workers=None):
    """process pool of spawned workers (not forked: the parent may hold a CUDA context and torch's threads)"""
    try:
        cpus = len(os.sched_getaffinity(0))
    except AttributeError:
        cpus = os.cpu_count() or 1
    return concurrent.futures.ProcessPoolExecutor(max_workers=max_workers or max(2, min(cpus, 16)),
                                                  mp_context=multiprocessing.get_context("spawn"))
