"""Keccak-f[1600] and the Keccak sponge (FIPS 202 §3-5), written from the definitions: the round constants come from
the rc(t) LFSR and the rho offsets from the (x, y) -> (y, 2x + 3y) walk, not from tables.  The padding byte is a
parameter: 0x06 gives SHA3-256 (checked against hashlib), 0x01 the original Keccak-256 Ethereum uses.  Test
infrastructure only.
"""
from __future__ import annotations

_MASK = (1 << 64) - 1


def _rc_bit(t: int) -> int:
    """FIPS 202 Algorithm 5: rc(t)"""
    if t % 255 == 0:
        return 1
    r = [1, 0, 0, 0, 0, 0, 0, 0]
    for _ in range(t % 255):
        r = [0] + r
        r[0] ^= r[8]
        r[4] ^= r[8]
        r[5] ^= r[8]
        r[6] ^= r[8]
        r = r[:8]
    return r[0]


ROUND_CONSTANTS = [sum(_rc_bit(j + 7 * ir) << ((1 << j) - 1) for j in range(7)) for ir in range(24)]


def _rho_offsets():
    off = [[0] * 5 for _ in range(5)]
    x, y = 1, 0
    for t in range(24):
        off[x][y] = ((t + 1) * (t + 2) // 2) % 64
        x, y = y, (2 * x + 3 * y) % 5
    return off


RHO = _rho_offsets()


def _rot(v: int, n: int) -> int:
    n %= 64
    return ((v << n) | (v >> (64 - n))) & _MASK


def keccak_f1600(lanes):
    """The permutation on 25 lanes, lanes[x + 5 y]; returns a new list."""
    A = [[lanes[x + 5 * y] for y in range(5)] for x in range(5)]
    for ir in range(24):
        C = [A[x][0] ^ A[x][1] ^ A[x][2] ^ A[x][3] ^ A[x][4] for x in range(5)]
        D = [C[(x - 1) % 5] ^ _rot(C[(x + 1) % 5], 1) for x in range(5)]
        A = [[A[x][y] ^ D[x] for y in range(5)] for x in range(5)]
        B = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                B[y][(2 * x + 3 * y) % 5] = _rot(A[x][y], RHO[x][y])
        A = [[B[x][y] ^ ((~B[(x + 1) % 5][y]) & B[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
        A[0][0] ^= ROUND_CONSTANTS[ir]
    return [A[i % 5][i // 5] for i in range(25)]


def sponge(data: bytes, pad: int, rate: int = 136, out_len: int = 32) -> bytes:
    """Keccak[c = 1600 - 8 rate] over data with the multi-rate padding pad || 0* || 0x80 (one byte pad | 0x80 when
    they meet)."""
    msg = bytearray(data)
    msg.append(pad)
    while len(msg) % rate:
        msg.append(0)
    msg[-1] |= 0x80
    lanes = [0] * 25
    for off in range(0, len(msg), rate):
        block = msg[off:off + rate]
        for k in range(rate // 8):
            lanes[k] ^= int.from_bytes(block[8 * k:8 * k + 8], "little")
        lanes = keccak_f1600(lanes)
    out = b""
    while True:
        out += b"".join(lanes[k].to_bytes(8, "little") for k in range(rate // 8))
        if len(out) >= out_len:
            return out[:out_len]
        lanes = keccak_f1600(lanes)


def keccak256(data: bytes) -> bytes:
    return sponge(bytes(data), 0x01)


def sha3_256(data: bytes) -> bytes:
    return sponge(bytes(data), 0x06)
