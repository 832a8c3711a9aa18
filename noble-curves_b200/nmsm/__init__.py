"""nmsm — host-side mirror of noble-curves' scalar-multiplication / MSM surface over libnmsm.so.

The reference's host language is TypeScript (no Node / N-API headers exist in this image, see
INTEGRATION.md for the addon a maintainer would add); this Python layer mirrors the same names,
argument meaning and error behaviour so the parity tests read like the reference's own tests:

    pippenger(c, points, scalars)          /root/reference/src/abstract/curve.ts:863-905
    mulAddUnsafe(c, points, scalars)       src/abstract/curve.ts:820-836 (same value, computed as an MSM)
    Point.multiply / Point.multiplyUnsafe  src/abstract/weierstrass.ts:900-928, src/abstract/edwards.ts:555-577
    Point.BASE / ZERO / fromAffine / toAffine / add / double / negate / equals / is0
    secp256k1.Point, ed25519.Point, bn254.G1/G2.Point, bls12_381.G1/G2.Point

plus the packed fast paths the reference lacks (SURVEY §8b): msm_packed, msm_device, multiply_many.
Every curve operation runs on the GPU through the C ABI; the host only marshals bytes and validates
argument shapes.  Nothing here imports `oracle/`.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence, Tuple

from . import _lib
from ._lib import NmsmError, PlanInfo, TIMING_NAMES, init  # noqa: F401

SECP256K1, ED25519, BN254_G1, BN254_G2, BLS12_381_G1, BLS12_381_G2 = range(6)


class _Field:
    """Shape-compatible stand-in for the IField members the MSM surface reads (modular.ts:429-607)."""

    def __init__(self, order: int, is_le: bool = False):
        self.ORDER = order
        self.BITS = order.bit_length()
        self.BYTES = (self.BITS + 7) // 8
        self.isLE = is_le

    def isValid(self, num) -> bool:
        return isinstance(num, int) and not isinstance(num, bool) and 0 <= num < self.ORDER

    def isValidNot0(self, num) -> bool:
        return self.isValid(num) and num != 0


class _Field2:
    def __init__(self, fp: _Field):
        self.Fp = fp
        self.ORDER = fp.ORDER * fp.ORDER
        self.BITS = self.ORDER.bit_length()
        self.BYTES = 2 * fp.BYTES

    def isValid(self, num) -> bool:
        return isinstance(num, tuple) and len(num) == 2 and self.Fp.isValid(num[0]) and self.Fp.isValid(num[1])


def _coord_to_bytes(v, nbytes: int, parts: int) -> bytes:
    if parts == 1:
        return v.to_bytes(nbytes, "little")
    return v[0].to_bytes(nbytes, "little") + v[1].to_bytes(nbytes, "little")


def _coord_from_bytes(b: bytes, nbytes: int, parts: int):
    if parts == 1:
        return int.from_bytes(b[:nbytes], "little")
    return (int.from_bytes(b[:nbytes], "little"), int.from_bytes(b[nbytes:2 * nbytes], "little"))


def _make_point_class(name: str, curve_id: int, p: int, n: int, h: int, Gx, Gy, parts: int, edwards: bool):
    base_fp = _Field(p, is_le=edwards)
    Fp = base_fp if parts == 1 else _Field2(base_fp)
    Fn = _Field(n, is_le=edwards)
    fp_bytes = 48 if p.bit_length() > 256 else 32
    zero_coord = 0 if parts == 1 else (0, 0)
    one_coord = 1 if parts == 1 else (1, 0)

    class Point:
        """Affine host handle of a curve point; every group operation runs on the GPU."""

        __slots__ = ("x", "y", "_inf", "_valid")
        CURVE_ID = curve_id
        NAME = name

        def __init__(self, x, y, _inf: bool = False, _valid: bool = False):
            """Like the reference's constructor (weierstrass.ts:695-704, edwards.ts:377-385) this does NOT validate
            curve or subgroup membership.  `_valid` is the host mirror of the reference's validityCache
            (weierstrass.ts:760-771): set by assertValidity / fromBytes / BASE / ZERO and inherited by the results
            of group operations on valid inputs.  pippenger only takes the endomorphism schedule on BLS12-381 G1
            when every input carries it (phi(P) = lambda*P needs the prime-order subgroup)."""
            if not Fp.isValid(x):
                raise ValueError("bad point coordinate x")
            # weierstrass.ts:698-701: a finite point with y = 0 is 2-torsion and is rejected by the constructor
            if not Fp.isValid(y) or (not edwards and not _inf and y == zero_coord):
                raise ValueError("bad point coordinate y")
            self.x, self.y, self._inf, self._valid = x, y, bool(_inf), bool(_valid)

        # -- noble's projective accessors (weierstrass.ts:687-704 / edwards.ts:370-385), Z = 1 ----
        @property
        def X(self):
            return self.x

        @property
        def Y(self):
            return one_coord if (self._inf and not edwards) else self.y

        @property
        def Z(self):
            return zero_coord if (self._inf and not edwards) else one_coord

        @staticmethod
        def fromAffine(p):
            """weierstrass.ts:711-718 / edwards.ts:396-402."""
            if not isinstance(p, dict) or not Fp.isValid(p.get("x")) or not Fp.isValid(p.get("y")):
                raise ValueError("invalid affine point")
            x, y = p["x"], p["y"]
            if not edwards and x == zero_coord and y == zero_coord:
                return Point.ZERO
            if edwards and x == 0 and y == 1:
                return Point.ZERO
            return Point(x, y)

        def toAffine(self):
            """weierstrass.ts:951-969 (ZERO -> (0,0)) / edwards.ts:595-609 (ZERO -> (0,1))."""
            return {"x": self.x, "y": self.y}

        def is0(self) -> bool:
            return self._inf

        def equals(self, other) -> bool:
            if not isinstance(other, Point):
                raise TypeError("Weierstrass Point expected" if not edwards else "EdwardsPoint expected")
            return self._inf == other._inf and self.x == other.x and self.y == other.y

        def negate(self):
            if self._inf:
                return self
            if edwards:  # -(x, y) = (-x, y)   edwards.ts:497-500
                return Point((-self.x) % p, self.y, False, self._valid)
            if parts == 1:  # weierstrass.ts:785-787
                return Point(self.x, (-self.y) % p, False, self._valid)
            return Point(self.x, ((-self.y[0]) % p, (-self.y[1]) % p), False, self._valid)

        def add(self, other):
            if not isinstance(other, Point):
                raise TypeError("Weierstrass Point expected" if not edwards else "EdwardsPoint expected")
            return _msm_points(Point, [self, other], [1, 1])

        def subtract(self, other):
            return self.add(other.negate())

        def double(self):
            return _msm_points(Point, [self], [2])

        def hasEvenY(self) -> bool:
            """weierstrass.ts:768-772 (prime base fields only: Fp2 has no isOdd)"""
            if edwards or parts != 1:
                raise ValueError("Field doesn't support isOdd")
            return (self.toAffine()["y"] & 1) == 0

        def assertValidity(self) -> None:
            """weierstrass.ts:752-771 / edwards.ts:461-480: on-curve + prime-order-subgroup check (both on the GPU:
            the curve equation through nmsm_points_on_curve, n*P == O through nmsm_points_torsion_free)."""
            if self._inf:
                if name.startswith("bls12_381") or edwards:  # allowInfinityPoint (bls12-381.ts) / Edwards identity
                    return
                raise ValueError("bad point: ZERO")
            if self._valid:
                return
            if points_on_curve(curve_id, self.to_packed(), 1)[0] != 1:
                raise ValueError("bad point: equation left != right")
            if h != 1 and torsion_free_packed(_ANY_POINT_ID.get(curve_id, curve_id), self.to_packed(), 1)[0] != 1:
                raise ValueError("bad point: not in prime-order subgroup")
            self._valid = True

        def multiply(self, scalar):
            """weierstrass.ts:900-907 / edwards.ts:555-564: 1 <= scalar < n."""
            if not Fn.isValidNot0(scalar):
                raise ValueError(
                    "invalid scalar: expected 1 <= sc < curve.n" if edwards else "invalid scalar: out of range"
                )
            return multiply_many(Point, [self], [scalar], unsafe=False)[0]

        def multiplyUnsafe(self, scalar):
            """weierstrass.ts:915-928 / edwards.ts:571-577: 0 <= scalar < n."""
            if not Fn.isValid(scalar):
                raise ValueError(
                    "invalid scalar: expected 0 <= sc < curve.n" if edwards else "invalid scalar: out of range"
                )
            return multiply_many(Point, [self], [scalar], unsafe=True)[0]

        def precompute(self, windowSize: int = 8, isLazy: bool = True):
            """weierstrass.ts:740-745 / edwards.ts:449-453: a cache hint in the reference; results never depend on
            it.  Here it marks the point for a device-resident multiplication table (nmsm_point_table_create; the
            GPU picks its own 16-bit windows, `windowSize` is only validated).  Like the reference's WeakMap cache
            (curve.ts:412,532) the table is built at the first multiply (isLazy) or now, and multiply_many /
            multiply / multiplyUnsafe of this point then take the table route."""
            _validate_w(windowSize, Fn.BITS)
            # curve.ts:776-781 setWindowSize sizes against the blinded path: ceil((bits + BLIND_BITS) / W) + 1 windows
            _validate_table_bytes((-(-(Fn.BITS + 128) // windowSize) + 1) * 2 ** (windowSize - 1), Fp.BYTES)
            _TABLE_MARKS.add((Point.CURVE_ID, self.x, self.y))
            if not isLazy:
                _table_for(Point, self)
            return self

        def clearCofactor(self):
            """weierstrass.ts:977-982 / edwards.ts:611-618 ([h]P; identity map for cofactor-1 curves)."""
            if h == 1:
                return self
            if h >= n:
                raise NotImplementedError("cofactor >= group order: outside the accelerated scalar range")
            return self.multiplyUnsafe(h)

        def isSmallOrder(self) -> bool:
            return self.is0() if h == 1 else self.clearCofactor().is0()

        def isTorsionFree(self) -> bool:
            """weierstrass.ts:971-975 / edwards.ts:584-586: n*P == O, evaluated as (n-1)*P + P on the GPU."""
            if self._inf:
                return True
            return self.multiplyUnsafe(n - 1).add(self).is0()

        def toBytes(self, isCompressed: bool = True) -> bytes:
            """Wire encodings of the reference: SEC1 (weierstrass.ts:541-563), Zcash flags for BLS12-381
            (bls12-381.ts:377-402), RFC 8032 for ed25519 (edwards.ts:620-628).  Pure byte packing on the host."""
            if edwards:
                b = bytearray(self.y.to_bytes(32, "little"))
                if self.x & 1:
                    b[31] |= 0x80
                return bytes(b)
            if name.startswith("bls12_381"):
                if parts != 1:
                    raise NotImplementedError("G2 wire format is not part of the accelerated path")
                if self._inf:
                    return bytes([0xC0 if isCompressed else 0x40]) + bytes(47 if isCompressed else 95)
                xb = bytearray(self.x.to_bytes(48, "big"))
                if isCompressed:
                    xb[0] |= 0x80 | (0x20 if (self.y * 2) // p else 0)
                    return bytes(xb)
                return bytes(xb) + self.y.to_bytes(48, "big")
            if parts != 1:
                raise NotImplementedError("Fp2 curves: wire format is not part of the accelerated path")
            if self._inf:
                raise ValueError("bad point: ZERO")
            xb = self.x.to_bytes(fp_bytes, "big")
            if isCompressed:
                return bytes([3 if self.y & 1 else 2]) + xb
            return b"\x04" + xb + self.y.to_bytes(fp_bytes, "big")

        @staticmethod
        def fromBytes(b: bytes, zip215: bool = False):
            """Point.fromBytes (weierstrass.ts:720-724; edwards.ts:405-436 `fromBytes(bytes, zip215 = false)`): decode on
            the GPU (nmsm_points_decode_ex), then the reference's validity check (subgroup membership where the
            cofactor is not 1).  Edwards: the default is the strict RFC 8032 decoding (y < p, no x = 0 with the sign
            bit set) exactly like the reference; zip215=True accepts the non-canonical encodings ZIP-215 allows.
            Like the reference, Edwards fromBytes does not run a subgroup check (edwards.ts:436)."""
            enc_len = {"secp256k1": 33, "bls12_381_G1": 48, "bls12_381_G2": 96, "ed25519": 32}.get(name)
            if enc_len is None or len(b) != enc_len:
                raise ValueError("bad point: got length %d, expected compressed=%s" % (len(b), enc_len))
            if not isinstance(zip215, bool):
                raise TypeError('"zip215" expected boolean')
            out, st = points_decode(curve_id, bytes(b), 1, zip215=bool(zip215) and edwards)
            if st[0] == 0:
                raise ValueError("bad point: is not on curve" if not edwards else "bad point: invalid y coordinate")
            P_ = Point.from_packed(out, 1 if st[0] == 2 else 0)
            if name in ("bls12_381_G1", "bls12_381_G2") and not P_.isTorsionFree():
                raise ValueError("bad point: not in prime-order subgroup")
            if not edwards:
                P_._valid = True  # decodePoint checks the equation, assertValidity the subgroup (weierstrass.ts:720-724)
            return P_

        @staticmethod
        def fromHex(hex_: str, zip215: bool = False):
            """weierstrass.ts:726-728 / edwards.ts:438-440: fromBytes(hexToBytes(hex))"""
            if not isinstance(hex_, str):
                raise TypeError("hex string expected, got " + type(hex_).__name__)
            try:
                raw = bytes.fromhex(hex_)
            except ValueError as e:
                raise ValueError("hex string expected, got non-hex character") from e
            return Point.fromBytes(raw, zip215) if edwards else Point.fromBytes(raw)

        def toHex(self, *args) -> str:
            return self.toBytes(*args).hex()

        def to_packed(self) -> bytes:
            return _coord_to_bytes(self.x, fp_bytes, parts) + _coord_to_bytes(self.y, fp_bytes, parts)

        @staticmethod
        def from_packed(b: bytes, is_inf: int, valid: bool = False):
            cb = fp_bytes * parts
            if is_inf:
                return Point.ZERO
            return Point(_coord_from_bytes(b[:cb], fp_bytes, parts), _coord_from_bytes(b[cb:2 * cb], fp_bytes, parts),
                         False, valid)

        def __repr__(self):
            return f"<{name}.Point {'ZERO' if self._inf else self.toAffine()}>"

    Point.__name__ = Point.__qualname__ = f"{name}_Point"
    Point.Fp = Fp
    Point.Fn = Fn
    Point.FP_BYTES = fp_bytes
    Point.PARTS = parts
    Point.POINT_BYTES = 2 * fp_bytes * parts
    Point.IS_EDWARDS = edwards
    Point.cofactor = h
    Point.BASE = Point(Gx, Gy, False, True)
    Point.ZERO = Point(0, 1, True, True) if edwards else Point(zero_coord, zero_coord, True, True)
    return Point


# Parameter blocks: SURVEY §8 a17 (src/secp256k1.ts:48-56, src/ed25519.ts:49-63, src/bn254.ts:80-90,207-223,
# src/bls12-381.ts:134-148,321-345).  tests/test_abi.py cross-checks them against the oracle's copies.
_BLS_P = 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB
_BLS_N = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
_BN_P = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
_BN_N = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001


class _NS:
    def __init__(self, **kw):
        self.__dict__.update(kw)


secp256k1 = _NS(
    Point=_make_point_class(
        "secp256k1", SECP256K1,
        2**256 - 2**32 - 977,
        0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141, 1,
        0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798,
        0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8, 1, False,
    )
)
ed25519 = _NS(
    Point=_make_point_class(
        "ed25519", ED25519,
        2**255 - 19,
        2**252 + 27742317777372353535851937790883648493, 8,
        0x216936D3CD6E53FEC0A4E231FDD6DC5C692CC7609525A7B2C9562D608F25D51A,
        0x6666666666666666666666666666666666666666666666666666666666666658, 1, True,
    )
)
bn254 = _NS(
    G1=_NS(Point=_make_point_class("bn254_G1", BN254_G1, _BN_P, _BN_N, 1, 1, 2, 1, False)),
    G2=_NS(
        Point=_make_point_class(
            "bn254_G2", BN254_G2, _BN_P, _BN_N,
            0x30644E72E131A029B85045B68181585E06CEECDA572A2489345F2299C0F9FA8D,
            (10857046999023057135944570762232829481370756359578518086990519993285655852781,
             11559732032986387107991004021392285783925812861821192530917403151452391805634),
            (8495653923123431417604973247489272438418190587263600148770280649306958101930,
             4082367875863433681332203403145435568316851327593401208105741076214120093531),
            2, False,
        )
    ),
)
bls12_381 = _NS(
    G1=_NS(
        Point=_make_point_class(
            "bls12_381_G1", BLS12_381_G1, _BLS_P, _BLS_N, 0x396C8C005555E1568C00AAAB0000AAAB,
            0x17F1D3A73197D7942695638C4FA9AC0FC3688C4F9774B905A14E3A3F171BAC586C55E83FF97A1AEFFB3AF00ADB22C6BB,
            0x08B3F481E3AAA0F1A09E30ED741D8AE4FCF5E095D5D00AF600DB18CB2C04B3EDD03CC744A2888AE40CAA232946C5E7E1,
            1, False,
        )
    ),
    G2=_NS(
        Point=_make_point_class(
            "bls12_381_G2", BLS12_381_G2, _BLS_P, _BLS_N,
            0x5D543A95414E7F1091D50792876A202CD91DE4547085ABAA68A205B2E5A7DDFA628F1CB4D9E82EF21537E293A6691AE1616EC6E786F0C70CF1C38E31C7238E5,
            (0x024AA2B2F08F0A91260805272DC51051C6E47AD4FA403B02B4510B647AE3D1770BAC0326A805BBEFD48056C8C121BDB8,
             0x13E02B6052719F607DACD3A088274F65596BD0D09920B61AB5DA61BBDC7F5049334CF11213945D57E5AC7D055D042B7E),
            (0x0CE5D527727D6E118CC9CDC6DA2E351AADFD9BAA8CBDD3A76D429A695160D12C923AC9CC3BACA289E193548608B82801,
             0x0606C4A02EA734CC32ACD2B02BC28B99CB3E287E85A763AF267492AB572E99AB3F370D275CEC1DA1AAA9075FF05F79BE),
            2, False,
        )
    ),
)

CURVES = {
    "secp256k1": secp256k1.Point,
    "ed25519": ed25519.Point,
    "bn254_G1": bn254.G1.Point,
    "bn254_G2": bn254.G2.Point,
    "bls12_381_G1": bls12_381.G1.Point,
    "bls12_381_G2": bls12_381.G2.Point,
}


# ----------------------------------------------------------------------------------------------
# validation (exact messages of curve.ts:390-404, :875)
# ----------------------------------------------------------------------------------------------
TABLE_BYTES_MAX = 2 ** 31  # curve.ts:37


def validatePointCons(c) -> None:
    """curve.ts:259-272: the generic helpers dereference fromAffine / fromBytes / fromHex / BASE / ZERO / Fp / Fn of the
    point constructor; fail with a typed error up front instead of an attribute error later."""
    if not isinstance(c, type):
        raise TypeError('"Point" expected constructor, got type=' + type(c).__name__)
    for fn_name in ("fromAffine", "fromBytes", "fromHex"):
        if not callable(getattr(c, fn_name, None)):
            raise TypeError('"Point.%s" expected function' % fn_name)
    for obj_name in ("BASE", "ZERO"):
        if getattr(c, obj_name, None) is None:
            raise TypeError('"Point.%s" expected object' % obj_name)
    for f_name in ("Fp", "Fn"):
        f = getattr(c, f_name, None)
        if f is None or not isinstance(getattr(f, "ORDER", None), int) or not isinstance(getattr(f, "BITS", None), int):
            raise TypeError('"Point.%s" expected a field' % f_name)


def _validate_w(W, bits: int, lo: int = 1) -> None:
    """curve.ts:328-331 validateW"""
    if not (isinstance(W, int) and not isinstance(W, bool) and lo <= W <= bits):
        raise ValueError("invalid window size, expected [%d..%d], got W=%s" % (lo, bits, W))


def _validate_table_bytes(num_points: int, fp_bytes: int) -> None:
    """curve.ts:336-346 validateTableBytes: the reference refuses window sizes whose tables would need more than ~2 GiB
    of heap (4 coordinates of Fp.BYTES + 128 bytes of object overhead per point); same rule, same message."""
    nbytes = num_points * (4 * fp_bytes + 128)
    if nbytes > TABLE_BYTES_MAX:
        raise ValueError("invalid window size: table would need ~%d MiB, max %d MiB"
                         % (-(-nbytes // 2 ** 20), TABLE_BYTES_MAX // 2 ** 20))


def _validate_msm_points(points, c) -> None:
    if not isinstance(points, (list, tuple)):
        raise TypeError('"points" expected Array, got type=' + type(points).__name__)
    for i, p in enumerate(points):
        if not isinstance(p, c):
            raise ValueError("invalid point at index " + str(i))


def _validate_msm_scalars(scalars, fn) -> None:
    if not isinstance(scalars, (list, tuple)):
        raise ValueError("array of scalars expected")
    for i, s in enumerate(scalars):
        if not fn.isValid(s):
            raise ValueError("invalid scalar at index " + str(i))


def _pack_points(points: Sequence) -> bytes:
    return b"".join(p.to_packed() for p in points)


def _pack_scalars(scalars: Sequence[int]) -> bytes:
    return b"".join(s.to_bytes(32, "little") for s in scalars)


def _raise_mapped(e: NmsmError):
    # the C ABI already carries the reference's message text for point/scalar errors
    raise ValueError(str(e)) from e


# include/nmsm.h: NMSM_BLS12_381_G1 (4) assumes torsion-free points (GLV); NMSM_BLS12_381_G1_ANY (6) does not
# likewise NMSM_BLS12_381_G2 (5, psi split) / NMSM_BLS12_381_G2_ANY (7)
_ANY_POINT_ID = {4: 6, 5: 7}


def _all_valid(points) -> bool:
    return all(p._valid for p in points)


def _curve_id_for(c, points, assume_torsion_free=None) -> int:
    """Curve id of the C ABI for an MSM over `points`.  BLS12-381 G1 has a cofactor, and the endomorphism schedule of
    id 4 is only the group law on the prime-order subgroup; the reference's pippenger is the plain group law on ANY
    Point instance (its constructor / fromAffine do not validate, weierstrass.ts:695-718).  So id 4 is taken only
    when every input is known valid (assertValidity / fromBytes / BASE / results of arithmetic on such points), or
    when the caller vouches for it; otherwise the plain-window id 6."""
    if c.CURVE_ID not in _ANY_POINT_ID:
        return c.CURVE_ID
    ok = _all_valid(points) if assume_torsion_free is None else bool(assume_torsion_free)
    return c.CURVE_ID if ok else _ANY_POINT_ID[c.CURVE_ID]


def _msm_points(c, points, scalars, assume_torsion_free=None):
    cid = _curve_id_for(c, points, assume_torsion_free)
    out_xy, inf = msm_packed(cid, _pack_points(points), _pack_scalars(scalars), len(points))
    # the group generated by valid points consists of valid points
    return c.from_packed(out_xy, inf, _all_valid(points))


# ----------------------------------------------------------------------------------------------
# public surface
# ----------------------------------------------------------------------------------------------
def msm_packed(curve_id: int, pts: bytes, scalars: bytes, n: int):
    """Packed fast path: canonical little-endian affine points + 32-byte LE scalars -> (xy bytes, is_inf)."""
    _lib.ensure_init()
    lib = _lib.load()
    pb = lib.nmsm_point_bytes(curve_id)
    if pb <= 0:
        raise ValueError("unknown curve id")
    if len(pts) != n * pb or len(scalars) != n * 32:
        raise ValueError("arrays of points and scalars must have equal length")
    out = ctypes.create_string_buffer(pb)
    inf = ctypes.c_int(0)
    pbuf = ctypes.c_char_p(bytes(pts)) if n else None
    sbuf = ctypes.c_char_p(bytes(scalars)) if n else None
    rc = lib.nmsm_msm(curve_id, ctypes.cast(pbuf, ctypes.c_void_p), ctypes.cast(sbuf, ctypes.c_void_p), n,
                      ctypes.cast(out, ctypes.c_void_p), ctypes.byref(inf))
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw, inf.value


def msm_device(curve_id: int, d_pts: int, d_scalars: int, n: int):
    """Inputs already resident in device memory (raw device pointers, e.g. torch `tensor.data_ptr()`)."""
    _lib.ensure_init()
    lib = _lib.load()
    pb = lib.nmsm_point_bytes(curve_id)
    out = ctypes.create_string_buffer(pb)
    inf = ctypes.c_int(0)
    rc = lib.nmsm_msm_device(curve_id, ctypes.c_void_p(d_pts), ctypes.c_void_p(d_scalars), n,
                             ctypes.cast(out, ctypes.c_void_p), ctypes.byref(inf))
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw, inf.value


def msm_host_ptr(curve_id: int, h_pts: int, h_scalars: int, n: int):
    """End-to-end path on raw HOST pointers (e.g. pinned buffers): H2D + MSM + D2H inside the call."""
    _lib.ensure_init()
    lib = _lib.load()
    pb = lib.nmsm_point_bytes(curve_id)
    out = ctypes.create_string_buffer(pb)
    inf = ctypes.c_int(0)
    rc = lib.nmsm_msm(curve_id, ctypes.c_void_p(h_pts), ctypes.c_void_p(h_scalars), n,
                      ctypes.cast(out, ctypes.c_void_p), ctypes.byref(inf))
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw, inf.value


def pippenger(c, points, scalars, assume_torsion_free=None):
    """Drop-in for noble's pippenger (curve.ts:863-905): validates like the reference, runs on the GPU.
    With default arguments the result equals the reference's for EVERY Point instance: on BLS12-381 G1 the
    endomorphism schedule (id 4) is used only when all inputs are known members of the prime-order subgroup (the
    `_valid` bit: assertValidity / fromBytes / BASE / arithmetic on valid points), otherwise plain windows (id 6).
    `assume_torsion_free=True` lets a caller who knows its fromAffine-built points are subgroup members (e.g. an
    SRS) opt into the fast schedule; False forces the plain one."""
    validatePointCons(c)
    _validate_msm_points(points, c)
    _validate_msm_scalars(scalars, c.Fn)
    if len(points) != len(scalars):
        raise ValueError("arrays of points and scalars must have equal length")
    if len(points) == 0:
        return c.ZERO
    return _msm_points(c, points, scalars, assume_torsion_free)


def normalizeZ(c, points):
    """curve.ts:311-326: batch projective -> affine.  Host handles are already canonical affine (every
    GPU result is normalised on the device — k_mul_batch / k_table_mul share ONE inversion per warp, the device form
    of FpInvertBatch modular.ts:734-760), so this validates and returns fresh equal points.  Un-normalised values only
    exist as raw accumulators on the device side of the C ABI; their batch normalisation is normalize_accs
    (nmsm_accs_normalize)."""
    validatePointCons(c)
    _validate_msm_points(points, c)
    return [c.from_packed(p.to_packed(), 1 if p.is0() else 0, p._valid) for p in points]


def aggregate_points(c, points):
    """sum_i P_i (BLS aggregatePublicKeys / aggregateSignatures are exactly this, abstract/bls.ts:860,870):
    an MSM with unit scalars; every term lands in one bucket, which the balanced-segment accumulate and the
    tile stitching handle in parallel."""
    _validate_msm_points(points, c)
    if not points:
        return c.ZERO
    return _msm_points(c, points, [1] * len(points))


def mulAddUnsafe(c, points, scalars, allowOversized: bool = False):
    """curve.ts:820-836 — same value as the Strauss–Shamir walk, evaluated as a (small) MSM on the GPU.
    allowOversized replaces the `s < Fn.ORDER` check by the `Fn.ORDER^4` cap (curve.ts:829-830).  Oversized scalars
    must NOT be reduced mod ORDER (the reference uses them for torsion checks `ORDER*P == O` on points that may lie
    outside the prime-order subgroup), so s is cut into digits of Fn.BITS-1 bits, s = sum_j d_j 2^(b j), and the term
    becomes sum_j d_j * (2^(b j) * P) with every d_j and 2^b in the accelerated range — exact for any point."""
    validatePointCons(c)
    _validate_msm_points(points, c)
    if not isinstance(allowOversized, bool):
        raise TypeError('"allowOversized" expected boolean')
    if not allowOversized:
        _validate_msm_scalars(scalars, c.Fn)
    else:
        if not isinstance(scalars, (list, tuple)):
            raise ValueError("array of scalars expected")
        cap = c.Fn.ORDER ** 4
        for i, s_ in enumerate(scalars):
            if not (isinstance(s_, int) and not isinstance(s_, bool) and 0 <= s_ < cap):
                raise ValueError("invalid scalar at index " + str(i))
    if len(points) != len(scalars):
        raise ValueError("arrays of points and scalars must have equal length")
    if len(points) == 0:
        return c.ZERO
    if all(s_ < c.Fn.ORDER for s_ in scalars):
        return _msm_points(c, points, scalars)
    b = c.Fn.BITS - 1
    step, mask = 1 << b, (1 << b) - 1
    pts2, sc2 = [], []
    for P_, s_ in zip(points, scalars):
        Q = P_
        while True:
            pts2.append(Q)
            sc2.append(s_ & mask)
            s_ >>= b
            if s_ == 0:
                break
            Q = multiply_many(c, [Q], [step], unsafe=True)[0]  # 2^b * Q, plain double-and-add on any point
    return _msm_points(c, pts2, sc2)


def torsion_free_packed(curve_id: int, pts: bytes, n: int) -> bytes:
    """Batch Point.isTorsionFree (nmsm_points_torsion_free): one byte per point, 1 = n*P == O."""
    _lib.ensure_init()
    lib = _lib.load()
    pb = lib.nmsm_point_bytes(curve_id)
    if len(pts) != n * pb:
        raise ValueError("expected %d bytes per point" % pb)
    out = ctypes.create_string_buffer(max(1, n))
    rc = lib.nmsm_points_torsion_free(curve_id, ctypes.cast(ctypes.c_char_p(bytes(pts)), ctypes.c_void_p), n,
                                      ctypes.cast(out, ctypes.c_void_p))
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw[:n]


class PointTable:
    """Device-resident multiplication table of ONE point (nmsm_point_table_create): d * 2^(16 j) * P."""

    def __init__(self, curve_id: int, point_xy: bytes):
        _lib.ensure_init()
        self._lib = _lib.load()
        self.curve_id = curve_id
        h = ctypes.c_uint64(0)
        try:
            _lib.check(self._lib.nmsm_point_table_create(curve_id, ctypes.cast(ctypes.c_char_p(bytes(point_xy)), ctypes.c_void_p),
                                                         ctypes.byref(h)))
        except NmsmError as e:
            _raise_mapped(e)
        self.handle = h.value

    def mul_batch(self, scalars: bytes, n: int, allow_zero: bool):
        pb = self._lib.nmsm_point_bytes(self.curve_id)
        if len(scalars) != n * 32:
            raise ValueError("expected 32 bytes per scalar")
        out = ctypes.create_string_buffer(max(1, n * pb))
        infs = ctypes.create_string_buffer(max(1, n))
        rc = self._lib.nmsm_point_table_mul_batch(self.handle, ctypes.cast(ctypes.c_char_p(bytes(scalars)), ctypes.c_void_p), n,
                                                  1 if allow_zero else 0, ctypes.cast(out, ctypes.c_void_p),
                                                  ctypes.cast(infs, ctypes.c_void_p))
        try:
            _lib.check(rc)
        except NmsmError as e:
            _raise_mapped(e)
        return out.raw[: n * pb], infs.raw[:n]

    def close(self):
        if self.handle:
            self._lib.nmsm_point_table_free(self.handle)
            self.handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# points marked by Point.precompute(), and the few most recently used device tables (36-107 MB each)
_TABLE_MARKS: set = set()
_TABLES: dict = {}
_TABLES_MAX = 4


def _table_for(c, point) -> PointTable:
    key = (c.CURVE_ID, point.x, point.y)
    t = _TABLES.pop(key, None)
    if t is None:
        t = PointTable(c.CURVE_ID, _pack_points([point]))
        while len(_TABLES) >= _TABLES_MAX:
            _TABLES.pop(next(iter(_TABLES))).close()
    _TABLES[key] = t  # most recently used last
    return t


def multiply_many(c, points, scalars, unsafe: bool = False) -> List:
    """Batch form of Point.multiply (unsafe=False: 1 <= k < n) / multiplyUnsafe (unsafe=True: 0 <= k < n).
    When every entry of `points` is the same precomputed point (Point.precompute) the device table route is used."""
    _validate_msm_points(points, c)
    if len(points) != len(scalars):
        raise ValueError("arrays of points and scalars must have equal length")
    for s in scalars:
        ok = c.Fn.isValid(s) if unsafe else c.Fn.isValidNot0(s)
        if not ok:
            if c.IS_EDWARDS:
                raise ValueError("invalid scalar: expected %d <= sc < curve.n" % (0 if unsafe else 1))
            raise ValueError("invalid scalar: out of range")
    n = len(points)
    if n == 0:
        return []
    p0 = points[0]
    if (c.CURVE_ID, p0.x, p0.y) in _TABLE_MARKS and not p0.is0() and all(q is p0 or q.equals(p0) for q in points):
        out_xy, infs = _table_for(c, p0).mul_batch(_pack_scalars(scalars), n, unsafe)
    else:
        out_xy, infs = mul_batch_packed(c.CURVE_ID, _pack_points(points), _pack_scalars(scalars), n, unsafe)
    pb = c.POINT_BYTES
    return [c.from_packed(out_xy[i * pb:(i + 1) * pb], infs[i], points[i]._valid) for i in range(n)]


def normalize_accs(curve_id: int, accs, n: int, on_device: bool = False):
    """nmsm_accs_normalize — the device form of normalizeZ (curve.ts:311-326): n raw accumulators (bytes, or a device
    pointer with on_device=True; nmsm_acc_bytes each) -> (packed canonical affine points, infinity flags), one field
    inversion per 32 points."""
    _lib.ensure_init()
    lib = _lib.load()
    pb, ab = lib.nmsm_point_bytes(curve_id), lib.nmsm_acc_bytes(curve_id)
    if pb <= 0:
        raise ValueError("unknown curve id")
    if not on_device and len(accs) != n * ab:
        raise ValueError("expected %d bytes per accumulator" % ab)
    out = ctypes.create_string_buffer(max(1, n * pb))
    infs = ctypes.create_string_buffer(max(1, n))
    src = ctypes.c_void_p(accs) if on_device else ctypes.cast(ctypes.c_char_p(bytes(accs)), ctypes.c_void_p)
    _lib.check(lib.nmsm_accs_normalize(curve_id, src, 1 if on_device else 0, n, ctypes.cast(out, ctypes.c_void_p),
                                       ctypes.cast(infs, ctypes.c_void_p)))
    return out.raw[: n * pb], infs.raw[:n]


def mul_batch_packed(curve_id: int, pts: bytes, scalars: bytes, n: int, allow_zero: bool):
    _lib.ensure_init()
    lib = _lib.load()
    pb = lib.nmsm_point_bytes(curve_id)
    if len(pts) != n * pb or len(scalars) != n * 32:
        raise ValueError("arrays of points and scalars must have equal length")
    out = ctypes.create_string_buffer(max(1, n * pb))
    infs = ctypes.create_string_buffer(max(1, n))
    rc = lib.nmsm_mul_batch(curve_id, ctypes.cast(ctypes.c_char_p(bytes(pts)), ctypes.c_void_p),
                            ctypes.cast(ctypes.c_char_p(bytes(scalars)), ctypes.c_void_p), n, 1 if allow_zero else 0,
                            ctypes.cast(out, ctypes.c_void_p), ctypes.cast(infs, ctypes.c_void_p))
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw[: n * pb], infs.raw[:n]


class PointSet:
    """Device-resident, validated and prepared point array (nmsm_points_upload): the fixed-base fast path."""

    def __init__(self, curve_id: int, pts: bytes, n: int):
        _lib.ensure_init()
        self._lib = _lib.load()
        self.curve_id, self.n = curve_id, n
        h = ctypes.c_uint64(0)
        try:
            _lib.check(self._lib.nmsm_points_upload(curve_id, ctypes.cast(ctypes.c_char_p(bytes(pts)), ctypes.c_void_p),
                                                    n, ctypes.byref(h)))
        except NmsmError as e:
            _raise_mapped(e)
        self.handle = h.value
        self.table_bits, self.table_levels = 0, 1

    def precompute(self, window_bits: int = 0):
        """Build the fixed-base table 2^(c*j) * P_i on the device (nmsm_points_precompute; the analogue of
        Point.precompute, curve.ts:532-577, for a whole set).  Returns (window bits, levels)."""
        c, lv = ctypes.c_int(0), ctypes.c_int(0)
        _lib.check(self._lib.nmsm_points_precompute(self.handle, int(window_bits), ctypes.byref(c), ctypes.byref(lv)))
        self.table_bits, self.table_levels = c.value, lv.value
        return c.value, lv.value

    def msm(self, scalars: bytes, n: int):
        pb = self._lib.nmsm_point_bytes(self.curve_id)
        out = ctypes.create_string_buffer(pb)
        inf = ctypes.c_int(0)
        rc = self._lib.nmsm_msm_points(self.handle, ctypes.cast(ctypes.c_char_p(bytes(scalars)), ctypes.c_void_p), n,
                                       ctypes.cast(out, ctypes.c_void_p), ctypes.byref(inf))
        try:
            _lib.check(rc)
        except NmsmError as e:
            _raise_mapped(e)
        return out.raw, inf.value

    def close(self):
        if self.handle:
            self._lib.nmsm_points_free(self.handle)
            self.handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def interleavedMSMUnsafe(c, points, windowSize: int = 4, precompute: bool = True, assume_torsion_free=None):
    """curve.ts:937-959: captures a FIXED point set once and returns `scalars -> sum s_i*P_i`.  Here the
    captured state is the device-resident prepared array plus (precompute=True, like the reference's per-point
    tables built at capture time) the fixed-base table of nmsm_points_precompute; `windowSize` is accepted for
    signature compatibility (the GPU schedule picks its own window).  Fewer scalars than points are zero-padded.
    BLS12-381 G1: the endomorphism id is used only for sets of known-valid points (see pippenger)."""
    validatePointCons(c)
    _validate_w(windowSize, c.Fn.BITS, 2)
    _validate_msm_points(points, c)
    _validate_table_bytes(len(points) * 2 ** (windowSize - 2), c.Fp.BYTES)  # curve.ts:947
    n = len(points)
    valid = _all_valid(points)
    ps = PointSet(_curve_id_for(c, points, assume_torsion_free), _pack_points(points), n) if n else None
    if ps is not None and precompute:
        ps.precompute(0)

    def run(scalars):
        _validate_msm_scalars(scalars, c.Fn)
        if len(scalars) > n:
            raise ValueError("array of scalars must not be larger than array of points")
        if n == 0:
            return c.ZERO
        padded = list(scalars) + [0] * (n - len(scalars))
        out, inf = ps.msm(_pack_scalars(padded), n)
        return c.from_packed(out, inf, valid)

    return run


def ed25519_verify_batch(signatures, messages, public_keys, z: bytes | None = None):
    """Batch form of ed25519.verify (edwards.ts:942-989, ZIP-215 decoding as ed25519's default): returns
    (ok, bad_index).  ok is True iff every signature would be accepted individually (up to 2^-128);
    bad_index is the first signature rejected without the group equation (undecodable point / s >= l), else -1.
    `z`: optional n*16 bytes of caller randomness (default os.urandom)."""
    import os
    import struct

    n = len(signatures)
    if len(messages) != n or len(public_keys) != n:
        raise ValueError("signatures, messages and public keys must have equal length")
    for s, p in zip(signatures, public_keys):
        if len(s) != 64 or len(p) != 32:
            raise ValueError("signature expected 64 bytes, publicKey 32 bytes")
    if z is None:
        z = os.urandom(16 * n)
    if len(z) != 16 * n:
        raise ValueError("z must hold 16 bytes per signature")
    offs = [0]
    for m in messages:
        offs.append(offs[-1] + len(m))
    blob = b"".join(bytes(m) for m in messages)
    return ed25519_verify_batch_packed(b"".join(signatures), b"".join(public_keys), blob,
                                       struct.pack("<%dQ" % (n + 1), *offs), n, bytes(z))


def ed25519_verify_batch_packed(sigs: bytes, pks: bytes, msgs: bytes, msg_off: bytes, n: int, z: bytes):
    """The C-ABI call itself (nmsm_ed25519_verify_batch) on caller-packed arrays: n*64 signature bytes, n*32 key bytes,
    the concatenated messages with n+1 little-endian u64 offsets, n*16 bytes of randomness."""
    if len(sigs) != 64 * n or len(pks) != 32 * n or len(msg_off) != 8 * (n + 1) or len(z) != 16 * n:
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    ok = ctypes.c_int(0)
    bad = ctypes.c_longlong(-1)
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    rc = lib.nmsm_ed25519_verify_batch(cp(sigs), cp(pks), cp(msgs or b"\0"), cp(msg_off), n, cp(z), ctypes.byref(ok),
                                       ctypes.byref(bad))
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return bool(ok.value), int(bad.value)


ED25519_VERIFY_STRICT = 1  # include/nmsm.h NMSM_ED25519_VERIFY_STRICT


def ed25519_verify_each(signatures, messages, public_keys, zip215: bool = True) -> List[bool]:
    """ed25519.verify(sig, msg, publicKey, { zip215 }) (edwards.ts:942-989) for every signature of a batch: one verdict
    per signature, unlike ed25519_verify_batch's single batch equation.  zip215 = True is noble's default for ed25519;
    False is RFC 8032 decoding with small-order keys rejected.  Raises where the reference throws before its `try`
    (non-bytes arguments, a signature that is not 64 bytes, a key that is not 32 bytes) and for lists of different
    lengths; everything else (an undecodable R or key, s >= l, a small-order key in strict mode, a failed equation) is
    a False verdict."""
    n = len(signatures)
    if len(messages) != n or len(public_keys) != n:
        raise ValueError("signatures, messages and public keys must have equal length")
    for what, items in (("signature", signatures), ("message", messages), ("publicKey", public_keys)):
        for x in items:
            if not isinstance(x, (bytes, bytearray, memoryview)):
                raise TypeError('"%s" expected Uint8Array, got type=%s' % (what, type(x).__name__))
    for what, items, size in (("signature", signatures, 64), ("publicKey", public_keys, 32)):
        for x in items:
            if len(x) != size:
                raise ValueError('"%s" expected Uint8Array of length %d, got length=%d' % (what, size, len(x)))
    out = ed25519_verify_each_packed(b"".join(bytes(s) for s in signatures), b"".join(bytes(p) for p in public_keys),
                                     b"".join(bytes(m) for m in messages), _pack_offsets(messages), n, zip215)
    return [b == 1 for b in out]


def ed25519_verify_each_packed(sigs: bytes, pks: bytes, msgs: bytes, msg_off: bytes, n: int,
                               zip215: bool = True) -> bytes:
    """The C-ABI call itself (nmsm_ed25519_verify_each) on caller-packed arrays: n*64 signature bytes, n*32 key bytes,
    the concatenated messages with n+1 little-endian u64 offsets.  Returns n verdict bytes (1 = valid)."""
    if len(sigs) != 64 * n or len(pks) != 32 * n or len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    rc = lib.nmsm_ed25519_verify_each(cp(sigs or b"\0"), cp(pks or b"\0"), cp(msgs or b"\0"), cp(msg_off), n,
                                      0 if zip215 else ED25519_VERIFY_STRICT, out)
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw[:n]


def _ed25519_verify(signature, message, publicKey, zip215: bool = True) -> bool:
    """ed25519.verify for one signature (the per-signature entry point with n = 1)."""
    return ed25519_verify_each([signature], [message], [publicKey], zip215=zip215)[0]


ed25519.verify = _ed25519_verify


ECDSA_PREHASH = 1  # include/nmsm.h NMSM_ECDSA_PREHASH
ECDSA_LOW_S = 2  # include/nmsm.h NMSM_ECDSA_LOW_S


def _pack_offsets(items) -> bytes:
    import struct

    offs = [0]
    for b in items:
        offs.append(offs[-1] + len(b))
    return struct.pack("<%dQ" % len(offs), *offs)


def _check_ecdsa_args(signatures, messages, public_keys, sig_len: int = 64):
    n = len(signatures)
    if len(messages) != n or len(public_keys) != n:
        raise ValueError("signatures, messages and public keys must have equal length")
    for what, items in (("signature", signatures), ("message", messages), ("publicKey", public_keys)):
        for x in items:
            if not isinstance(x, (bytes, bytearray, memoryview)):
                raise TypeError('"%s" expected Uint8Array, got type=%s' % (what, type(x).__name__))
    for s in signatures:
        if len(s) != sig_len:
            raise ValueError('"compact signature" expected Uint8Array of length %d, got length=%d' % (sig_len, len(s)))


def ecdsa_verify_batch(signatures, messages, public_keys, prehash: bool = True, lowS: bool = True) -> List[bool]:
    """Batch form of secp256k1.verify(sig, msg, publicKey, {prehash, lowS}) with format 'compact' (noble-curves
    weierstrass.ts ecdsa().verify): one verdict per signature.  Raises where the reference throws before its `try`
    (non-bytes arguments, a signature that is not 64 bytes) and for lists of different lengths; everything else
    (r, s out of range, high s, an undecodable key, a raw message over 8192 bytes, R = O) is a False verdict."""
    _check_ecdsa_args(signatures, messages, public_keys)
    n = len(signatures)
    flags = (ECDSA_PREHASH if prehash else 0) | (ECDSA_LOW_S if lowS else 0)
    out = ecdsa_verify_batch_packed(b"".join(bytes(s) for s in signatures), b"".join(bytes(p) for p in public_keys),
                                    _pack_offsets(public_keys), b"".join(bytes(m) for m in messages),
                                    _pack_offsets(messages), n, flags)
    return [b == 1 for b in out]


def ecdsa_verify_batch_packed(sigs: bytes, pks: bytes, pk_off: bytes, msgs: bytes, msg_off: bytes, n: int,
                              flags: int = ECDSA_PREHASH | ECDSA_LOW_S) -> bytes:
    """The C-ABI call itself (nmsm_secp256k1_verify_batch) on caller-packed arrays: n*64 signature bytes, the
    concatenated keys and messages with n+1 little-endian u64 offsets each.  Returns n verdict bytes (1 = valid)."""
    if len(sigs) != 64 * n or len(pk_off) != 8 * (n + 1) or len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    rc = lib.nmsm_secp256k1_verify_batch(cp(sigs or b"\0"), cp(pks or b"\0"), cp(pk_off), cp(msgs or b"\0"),
                                         cp(msg_off), n, flags, out)
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw[:n]


def _secp256k1_verify(signature, message, publicKey, prehash: bool = True, lowS: bool = True,
                      format: str = "compact") -> bool:
    """secp256k1.verify for one signature (the batch entry point with n = 1)."""
    if format != "compact":
        raise NotImplementedError("signature format %r is not part of the accelerated path (compact only)" % (format,))
    return ecdsa_verify_batch([signature], [message], [publicKey], prehash=prehash, lowS=lowS)[0]


secp256k1.verify = _secp256k1_verify


def p256_ecdsa_verify_batch(signatures, messages, public_keys, prehash: bool = True, lowS: bool = False) -> List[bool]:
    """Batch form of p256.verify(sig, msg, publicKey, {prehash, lowS}) with format 'compact' (noble-curves nist.ts,
    weierstrass.ts ecdsa().verify): one verdict per signature.  The defaults are noble's for p256 (lowS false, as
    OpenSSL).  Raises as ecdsa_verify_batch; everything else (r, s out of range, high s under lowS, an undecodable key,
    a raw message over 8192 bytes, R = O) is a False verdict."""
    _check_ecdsa_args(signatures, messages, public_keys)
    flags = (ECDSA_PREHASH if prehash else 0) | (ECDSA_LOW_S if lowS else 0)
    out = p256_ecdsa_verify_batch_packed(b"".join(bytes(s) for s in signatures),
                                         b"".join(bytes(p) for p in public_keys), _pack_offsets(public_keys),
                                         b"".join(bytes(m) for m in messages), _pack_offsets(messages),
                                         len(signatures), flags)
    return [b == 1 for b in out]


def p256_ecdsa_verify_batch_packed(sigs: bytes, pks: bytes, pk_off: bytes, msgs: bytes, msg_off: bytes, n: int,
                                   flags: int = ECDSA_PREHASH) -> bytes:
    """The C-ABI call itself (nmsm_p256_verify_batch) on caller-packed arrays, laid out as for
    ecdsa_verify_batch_packed.  Returns n verdict bytes (1 = valid)."""
    if len(sigs) != 64 * n or len(pk_off) != 8 * (n + 1) or len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    rc = lib.nmsm_p256_verify_batch(cp(sigs or b"\0"), cp(pks or b"\0"), cp(pk_off), cp(msgs or b"\0"), cp(msg_off), n,
                                    flags, out)
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw[:n]


def _p256_verify(signature, message, publicKey, prehash: bool = True, lowS: bool = False,
                 format: str = "compact") -> bool:
    """p256.verify for one signature (the batch entry point with n = 1)."""
    if format != "compact":
        raise NotImplementedError("signature format %r is not part of the accelerated path (compact only)" % (format,))
    return p256_ecdsa_verify_batch([signature], [message], [publicKey], prehash=prehash, lowS=lowS)[0]


# noble-curves' `p256` export (nist.ts; also `secp256r1`).  Verification only: P-256 is not an MSM curve and has no
# Point class here, so it is not in CURVES.
p256 = _NS(verify=_p256_verify)
secp256r1 = p256

P256VERIFY_INPUT_BYTES = 160  # EIP-7951 / RIP-7212: hash || r || s || qx || qy, 32 bytes each


def p256verify_precompile_batch(inputs) -> List[bool]:
    """Ethereum's P256VERIFY precompile (EIP-7951 on L1, RIP-7212 on rollups) over a batch: True where the precompile
    returns the 32-byte word 1, False where it returns empty output.  `inputs` is a list of byte strings or one buffer
    of n * 160 bytes.  An input that is not 160 bytes is False.  Each input runs as a P-256 ECDSA verification with
    the 32-byte hash as the raw message (no prehash, no lowS) and the key 04 || qx || qy: that checks r, s in [1, n),
    qx, qy < p, Q on the curve (which rejects (0, 0)), R != O and R.x mod n == r, the precompile's rules."""
    import numpy as np

    if isinstance(inputs, (bytes, bytearray, memoryview)):
        buf = bytes(inputs)
        if len(buf) % P256VERIFY_INPUT_BYTES:
            raise ValueError("a packed P256VERIFY batch must be a multiple of 160 bytes, got %d" % len(buf))
        items = np.frombuffer(buf, np.uint8).reshape(-1, P256VERIFY_INPUT_BYTES)
        good = np.ones(len(items), bool)
    else:
        for x in inputs:
            if not isinstance(x, (bytes, bytearray, memoryview)):
                raise TypeError("P256VERIFY input expected bytes, got type=%s" % type(x).__name__)
        good = np.array([len(x) == P256VERIFY_INPUT_BYTES for x in inputs], bool)
        items = np.zeros((len(inputs), P256VERIFY_INPUT_BYTES), np.uint8)
        for i, x in enumerate(inputs):
            if good[i]:
                items[i] = np.frombuffer(bytes(x), np.uint8)
    idx = np.flatnonzero(good)
    m = len(idx)
    out = np.zeros(len(good), bool)
    if m == 0:
        return out.tolist()
    sel = items[idx]
    sigs = np.ascontiguousarray(sel[:, 32:96]).tobytes()
    msgs = np.ascontiguousarray(sel[:, :32]).tobytes()
    keys = np.empty((m, 65), np.uint8)
    keys[:, 0] = 4
    keys[:, 1:] = sel[:, 96:]
    off = lambda w: (np.arange(m + 1, dtype="<u8") * w).tobytes()  # noqa: E731
    res = p256_ecdsa_verify_batch_packed(sigs, keys.tobytes(), off(65), msgs, off(32), m, 0)
    out[idx] = np.frombuffer(res, np.uint8) == 1
    return out.tolist()


def p384_ecdsa_verify_batch(signatures, messages, public_keys, prehash: bool = True, lowS: bool = False) -> List[bool]:
    """Batch form of p384.verify(sig, msg, publicKey, {prehash, lowS}) with format 'compact' (noble-curves nist.ts,
    weierstrass.ts ecdsa().verify): one verdict per signature.  Signatures are 96 bytes r || s, keys 49-byte compressed
    or 97-byte uncompressed SEC1, and prehash hashes with SHA-384.  The defaults are noble's for p384 (lowS false, as
    OpenSSL).  Raises as p256_ecdsa_verify_batch; everything else (r, s out of range, high s under lowS, an undecodable
    key, a raw message over 8192 bytes, R = O) is a False verdict."""
    _check_ecdsa_args(signatures, messages, public_keys, sig_len=96)
    flags = (ECDSA_PREHASH if prehash else 0) | (ECDSA_LOW_S if lowS else 0)
    out = p384_ecdsa_verify_batch_packed(b"".join(bytes(s) for s in signatures),
                                         b"".join(bytes(p) for p in public_keys), _pack_offsets(public_keys),
                                         b"".join(bytes(m) for m in messages), _pack_offsets(messages),
                                         len(signatures), flags)
    return [b == 1 for b in out]


def p384_ecdsa_verify_batch_packed(sigs: bytes, pks: bytes, pk_off: bytes, msgs: bytes, msg_off: bytes, n: int,
                                   flags: int = ECDSA_PREHASH) -> bytes:
    """The C-ABI call itself (nmsm_p384_verify_batch) on caller-packed arrays: n*96 signature bytes, the concatenated
    keys and messages with n+1 little-endian u64 offsets each.  Returns n verdict bytes (1 = valid)."""
    if len(sigs) != 96 * n or len(pk_off) != 8 * (n + 1) or len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    rc = lib.nmsm_p384_verify_batch(cp(sigs or b"\0"), cp(pks or b"\0"), cp(pk_off), cp(msgs or b"\0"), cp(msg_off), n,
                                    flags, out)
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw[:n]


def _p384_verify(signature, message, publicKey, prehash: bool = True, lowS: bool = False,
                 format: str = "compact") -> bool:
    """p384.verify for one signature (the batch entry point with n = 1)."""
    if format != "compact":
        raise NotImplementedError("signature format %r is not part of the accelerated path (compact only)" % (format,))
    return p384_ecdsa_verify_batch([signature], [message], [publicKey], prehash=prehash, lowS=lowS)[0]


# noble-curves' `p384` export (nist.ts; also `secp384r1`).  Verification only, as p256: not in CURVES.
p384 = _NS(verify=_p384_verify)
secp384r1 = p384


def schnorr_verify_batch(signatures, messages, public_keys) -> List[bool]:
    """Batch form of schnorr.verify(signature, message, publicKey) (noble-curves secp256k1.ts, BIP340): one verdict
    per signature.  Raises where the reference throws before its `try` (non-bytes arguments, a signature that is not 64
    bytes, a key that is not 32 bytes) and for lists of different lengths; everything else (a key that is not an x
    coordinate on the curve, r >= p, s >= n, R = O, an odd y(R), x(R) != r) is a False verdict."""
    n = len(signatures)
    if len(messages) != n or len(public_keys) != n:
        raise ValueError("signatures, messages and public keys must have equal length")
    for what, items in (("signature", signatures), ("message", messages), ("publicKey", public_keys)):
        for x in items:
            if not isinstance(x, (bytes, bytearray, memoryview)):
                raise TypeError('"%s" expected Uint8Array, got type=%s' % (what, type(x).__name__))
    for what, items, size in (("signature", signatures, 64), ("publicKey", public_keys, 32)):
        for x in items:
            if len(x) != size:
                raise ValueError('"%s" expected Uint8Array of length %d, got length=%d' % (what, size, len(x)))
    out = schnorr_verify_batch_packed(b"".join(bytes(s) for s in signatures), b"".join(bytes(p) for p in public_keys),
                                      b"".join(bytes(m) for m in messages), _pack_offsets(messages), n)
    return [b == 1 for b in out]


def schnorr_verify_batch_packed(sigs: bytes, pks: bytes, msgs: bytes, msg_off: bytes, n: int) -> bytes:
    """The C-ABI call itself (nmsm_secp256k1_schnorr_verify_batch) on caller-packed arrays: n*64 signature bytes, n*32
    x-only key bytes, the concatenated messages with n+1 little-endian u64 offsets.  Returns n verdict bytes (1 = valid)."""
    if len(sigs) != 64 * n or len(pks) != 32 * n or len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    rc = lib.nmsm_secp256k1_schnorr_verify_batch(cp(sigs or b"\0"), cp(pks or b"\0"), cp(msgs or b"\0"), cp(msg_off), n,
                                                 out)
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw[:n]


def _schnorr_verify(signature, message, publicKey) -> bool:
    """schnorr.verify for one signature (the batch entry point with n = 1)."""
    return schnorr_verify_batch([signature], [message], [publicKey])[0]


schnorr = _NS(verify=_schnorr_verify)  # the reference's `schnorr` export (secp256k1.ts)


# ---- secp256k1 ECDSA public-key recovery and Ethereum ecrecover (include/nmsm.h nmsm_secp256k1_*recover_batch) -----
def ecdsa_recover_batch(signatures, messages, prehash: bool = True) -> List[Optional[bytes]]:
    """Batch form of secp256k1.recoverPublicKey(signature, message, {prehash}) with the 65-byte 'recovered' format
    rec || r || s (noble-curves weierstrass.ts Signature.recoverPublicKey): per signature the recovered key as 33-byte
    SEC1 compressed bytes, or None where the reference throws (a recovery id outside 0..3, r or s outside [1, n), an x
    coordinate >= p or off the curve, a raw message over 8192 bytes, Q = O).  Raises for non-bytes arguments, a
    signature that is not 65 bytes and lists of different lengths."""
    n = len(signatures)
    if len(messages) != n:
        raise ValueError("signatures and messages must have equal length")
    for what, items in (("signature", signatures), ("message", messages)):
        for x in items:
            if not isinstance(x, (bytes, bytearray, memoryview)):
                raise TypeError('"%s" expected Uint8Array, got type=%s' % (what, type(x).__name__))
    for s in signatures:
        if len(s) != 65:
            raise ValueError('"recovered signature" expected Uint8Array of length 65, got length=%d' % len(s))
    xy, ok = ecdsa_recover_batch_packed(b"".join(bytes(s) for s in signatures), b"".join(bytes(m) for m in messages),
                                        _pack_offsets(messages), n, ECDSA_PREHASH if prehash else 0)
    out = []
    for k in range(n):
        if not ok[k]:
            out.append(None)
            continue
        x, y = xy[64 * k:64 * k + 32], xy[64 * k + 32:64 * k + 64]
        out.append(bytes([2 + (y[0] & 1)]) + x[::-1])
    return out


def ecdsa_recover_batch_packed(sigs65: bytes, msgs: bytes, msg_off: bytes, n: int, flags: int = ECDSA_PREHASH):
    """The C-ABI call itself (nmsm_secp256k1_recover_batch) on caller-packed arrays: n*65 signature bytes (rec || r ||
    s), the concatenated messages with n+1 little-endian u64 offsets.  Returns (n*64 bytes of keys in the affine
    packing, little-endian x || y, zero for a failed item; n verdict bytes, 1 = recovered)."""
    if len(sigs65) != 65 * n or len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    xy = ctypes.create_string_buffer(max(64 * n, 1))
    ok = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    rc = lib.nmsm_secp256k1_recover_batch(cp(sigs65 or b"\0"), cp(msgs or b"\0"), cp(msg_off), n, flags, xy, ok)
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return xy.raw[:64 * n], ok.raw[:n]


def _secp256k1_recover_public_key(signature, message, prehash: bool = True) -> bytes:
    """secp256k1.recoverPublicKey for one signature (the batch entry point with n = 1): the 33-byte compressed key
    (the reference's default toBytes()).  Raises ValueError where the reference throws."""
    key = ecdsa_recover_batch([signature], [message], prehash=prehash)[0]
    if key is None:
        raise ValueError("public key recovery failed: invalid recovery id, r, s or message, or the key is the point "
                         "at infinity")
    return key


secp256k1.recoverPublicKey = _secp256k1_recover_public_key


def eth_ecrecover_batch(inputs) -> List[bytes]:
    """Ethereum's ecrecover precompile (0x01) over a batch: per input the precompile's output, the 32-byte word 12
    zero bytes || address, or b"" where the precompile returns empty output.  An input is right-padded with zeros to
    128 bytes or truncated to its first 128, as the precompile reads its call data."""
    inputs = list(inputs)
    buf = []
    for j, data in enumerate(inputs):
        if not isinstance(data, (bytes, bytearray, memoryview)):
            raise TypeError("input %d: bytes expected, got type=%s" % (j, type(data).__name__))
        buf.append(bytes(data[:128]).ljust(128, b"\0"))
    if not buf:
        return []
    words, ok = eth_ecrecover_batch_packed(b"".join(buf), len(buf))
    return [words[32 * k:32 * k + 32] if ok[k] else b"" for k in range(len(buf))]


def eth_ecrecover_batch_packed(inputs128: bytes, n: int):
    """The C-ABI call itself (nmsm_secp256k1_ecrecover_batch): n*128 input bytes h || v || r || s.  Returns (n*32
    bytes of address words, zero for a failed item; n verdict bytes, 1 = recovered)."""
    if len(inputs128) != 128 * n:
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    words = ctypes.create_string_buffer(max(32 * n, 1))
    ok = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    rc = lib.nmsm_secp256k1_ecrecover_batch(cp(inputs128 or b"\0"), n, words, ok)
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return words.raw[:32 * n], ok.raw[:n]


# ---- BLS12-381 pairing checks and BLS signatures (include/nmsm.h nmsm_bls12_381_*) -----------------------------------
def _bls_g2_compress(pt) -> bytes:
    """Zcash-flag compressed G2 encoding (bls12-381.ts:377-402,488-491): x.c1 || x.c0 big-endian, sort bit over
    [y.c1, y.c0]."""
    if pt.is0():
        return bytes([0xC0]) + bytes(95)
    (x0, x1), (y0, y1) = pt.x, pt.y
    b = bytearray(x1.to_bytes(48, "big") + x0.to_bytes(48, "big"))
    part = y1 if y1 else y0
    b[0] |= 0x80 | (0x20 if (part * 2) // _BLS_P else 0)
    return bytes(b)


def _pack_pairing_checks(checks, G1, G2, label: str):
    """lists of (G1 Point, G2 Point) pairs -> the packed arguments of a pairing-check entry point"""
    import struct

    g1, g2, offs = [], [], [0]
    for j, check in enumerate(checks):
        for pair in check:
            if len(pair) != 2 or not isinstance(pair[0], G1) or not isinstance(pair[1], G2):
                raise TypeError("check %d: (%s.G1.Point, %s.G2.Point) pairs expected" % (j, label, label))
            g1.append(pair[0])
            g2.append(pair[1])
        offs.append(len(g1))
    return _pack_points(g1), _pack_points(g2), struct.pack("<%dQ" % len(offs), *offs), len(checks)


def _pairing_check_call(fn: str, g1_bytes: int, g1_xy: bytes, g2_xy: bytes, pair_off: bytes, n_checks: int) -> bytes:
    """the C call of a pairing-check entry point fn with G1 points of g1_bytes bytes (G2 points are twice that)"""
    if len(pair_off) != 8 * (n_checks + 1):
        raise ValueError("packed arrays do not match n_checks")
    total = int.from_bytes(pair_off[-8:], "little") if n_checks else 0
    if len(g1_xy) != g1_bytes * total or len(g2_xy) != 2 * g1_bytes * total:
        raise ValueError("packed arrays do not match the pair count")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n_checks, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    _lib.check(getattr(lib, fn)(cp(g1_xy or b"\0"), cp(g2_xy or b"\0"), cp(pair_off), n_checks, out))
    return out.raw[:n_checks]


def pairing_check_batch(checks) -> List[bool]:
    """One verdict per check: checks[j] is a list of (G1 Point, G2 Point) pairs, True iff the product of their pairings
    is 1 (noble's pairingBatch compared with Fp12.ONE).  A pair with an identity point contributes 1 (the reference
    throws on the zero point); points are not subgroup-checked (assertValidity / isTorsionFree does that).  Raises
    ValueError for a point off its curve."""
    args = _pack_pairing_checks(checks, bls12_381.G1.Point, bls12_381.G2.Point, "bls12_381")
    try:
        out = pairing_check_batch_packed(*args)
    except NmsmError as e:
        _raise_mapped(e)
    return [b == 1 for b in out]


def pairing_check_batch_packed(g1_xy: bytes, g2_xy: bytes, pair_off: bytes, n_checks: int) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_pairing_check_batch): packed affine G1 (96 B) and G2 (192 B) points and
    n_checks + 1 little-endian u64 pair offsets.  Returns n_checks verdict bytes; raises NmsmError (with .code and
    .index) on an error."""
    return _pairing_check_call("nmsm_bls12_381_pairing_check_batch", 96, g1_xy, g2_xy, pair_off, n_checks)


def bls_verify_batch(signatures, message_points, public_keys) -> List[bool]:
    """Batch form of bls12_381.verify(signature, message, publicKey) for long signatures (public key in G1, signature in
    G2): one verdict per signature.  Signatures are 96-byte and keys 48-byte Zcash-flag compressed encodings, or Points
    (encoded first).  Messages must already be hashed to G2 (bls12_381.G2.Point): hash-to-curve is not implemented, so
    bytes messages raise.  A signature or key that does not decode, is the identity or lies outside its subgroup is a
    False verdict; a message point off the curve raises ValueError."""
    n = len(signatures)
    if len(message_points) != n or len(public_keys) != n:
        raise ValueError("signatures, messages and public keys must have equal length")
    G2 = bls12_381.G2.Point
    sigs, pks = _bls_sigs_and_keys(signatures, public_keys)
    for m in message_points:
        if isinstance(m, (bytes, bytearray, memoryview, str)):
            raise NotImplementedError("hash-to-curve is not implemented: pass the message hashed to G2 as a "
                                      "bls12_381.G2.Point")
        if not isinstance(m, G2):
            raise TypeError('"message" expected bls12_381.G2.Point, got type=%s' % type(m).__name__)
    try:
        out = bls_verify_batch_packed(sigs, pks, _pack_points(message_points), n)
    except NmsmError as e:
        _raise_mapped(e)
    return [b == 1 for b in out]


def _bls_sigs_and_keys(signatures, public_keys):
    """the packed signature and key arguments of the verify entry points: 96-byte and 48-byte Zcash-flag compressed
    encodings, or Points (encoded first)"""
    G1, G2 = bls12_381.G1.Point, bls12_381.G2.Point
    sigs, pks = [], []
    for s in signatures:
        if isinstance(s, G2):
            s = _bls_g2_compress(s)
        if not isinstance(s, (bytes, bytearray, memoryview)):
            raise TypeError('"signature" expected Uint8Array or G2 Point, got type=%s' % type(s).__name__)
        if len(s) != 96:
            raise ValueError('"signature" expected Uint8Array of length 96, got length=%d' % len(s))
        sigs.append(bytes(s))
    for k in public_keys:
        if isinstance(k, G1):
            k = k.toBytes(True)
        if not isinstance(k, (bytes, bytearray, memoryview)):
            raise TypeError('"publicKey" expected Uint8Array or G1 Point, got type=%s' % type(k).__name__)
        if len(k) != 48:
            raise ValueError('"publicKey" expected Uint8Array of length 48, got length=%d' % len(k))
        pks.append(bytes(k))
    return b"".join(sigs), b"".join(pks)


def bls_verify_batch_packed(sigs96: bytes, pks48: bytes, msg_pts: bytes, n: int) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_verify_batch): n*96 signature bytes, n*48 key bytes and n*192 bytes of
    affine G2 message points.  Returns n verdict bytes; raises NmsmError (with .code and .index) on an error."""
    if len(sigs96) != 96 * n or len(pks48) != 48 * n or len(msg_pts) != 192 * n:
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    _lib.check(lib.nmsm_bls12_381_verify_batch(cp(sigs96 or b"\0"), cp(pks48 or b"\0"), cp(msg_pts or b"\0"), n, out))
    return out.raw[:n]


def _bls_verify(signature, message, publicKey) -> bool:
    """bls12_381.verify for one signature (the batch entry point with n = 1)."""
    return bls_verify_batch([signature], [message], [publicKey])[0]


bls12_381.verify = _bls_verify


# ---- BLS12-381 hash to G2 (include/nmsm.h nmsm_bls12_381_hash_to_g2_batch, nmsm_bls12_381_verify_msg_batch) ------
DST_G2_NUL = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_"  # noble's default tag for long signatures
DST_G2_POP = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_"  # proof-of-possession scheme (Ethereum consensus)


def _h2c_args(messages, dst):
    """(message bytes list, tag bytes) after the checks noble's hashToCurve makes: bytes messages, a non-empty tag
    (a str tag is UTF-8, as noble accepts strings)"""
    if isinstance(dst, str):
        dst = dst.encode()
    if not isinstance(dst, (bytes, bytearray, memoryview)):
        raise TypeError('"DST" expected Uint8Array or string, got type=%s' % type(dst).__name__)
    if len(dst) == 0:
        raise ValueError("DST must be non-empty (RFC 9380 §3.1)")
    msgs = []
    for m in messages:
        if not isinstance(m, (bytes, bytearray, memoryview)):
            raise TypeError('"message" expected Uint8Array, got type=%s' % type(m).__name__)
        msgs.append(bytes(m))
    return msgs, bytes(dst)


def bls_hash_to_g2_batch(messages, dst=DST_G2_NUL) -> List:
    """Batch form of bls12_381.G2.hashToCurve(msg, { DST }) (RFC 9380 suite BLS12381G2_XMD:SHA-256_SSWU_RO_): one
    bls12_381.G2.Point per message, each in G2.  Messages are bytes of any length; the tag is non-empty bytes (or str),
    one tag for the whole batch."""
    msgs, dst = _h2c_args(messages, dst)
    if not msgs:
        return []
    xy = bls_hash_to_g2_batch_packed(b"".join(msgs), _pack_offsets(msgs), len(msgs), dst)
    G2 = bls12_381.G2.Point
    out = []
    for k in range(len(msgs)):
        b = xy[192 * k:192 * k + 192]
        out.append(G2.from_packed(b, not any(b), valid=True))
    return out


def bls_hash_to_g2_batch_packed(msgs: bytes, msg_off: bytes, n: int, dst: bytes) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_hash_to_g2_batch): the concatenated messages with n+1 little-endian u64
    offsets and the tag.  Returns n*192 bytes of affine G2 points; raises NmsmError (with .code) on an error."""
    if len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(192 * n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    _lib.check(lib.nmsm_bls12_381_hash_to_g2_batch(cp(msgs or b"\0"), cp(msg_off), n, cp(dst or b"\0"), len(dst), out))
    return out.raw[:192 * n]


def _g2_hash_to_curve(msg, options=None):
    """bls12_381.G2.hashToCurve(msg, { DST }) for one message (the batch entry point with n = 1); the default tag is
    noble's BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_."""
    dst = DST_G2_NUL
    if options is not None:
        if not isinstance(options, dict):
            raise TypeError("options expected dict, got type=%s" % type(options).__name__)
        dst = options.get("DST", DST_G2_NUL)
    return bls_hash_to_g2_batch([msg], dst)[0]


bls12_381.G2.hashToCurve = _g2_hash_to_curve


def bls_verify_messages_batch(signatures, messages, public_keys, dst=DST_G2_NUL) -> List[bool]:
    """bls_verify_batch with message bytes, hashed to G2 on the GPU under dst in the same call: verdict i is
    bls12_381.verify(signature_i, G2.hashToCurve(message_i, { DST }), publicKey_i).  Signatures and keys as for
    bls_verify_batch; a signature or key that does not decode, is the identity or lies outside its subgroup is a False
    verdict."""
    n = len(signatures)
    if len(messages) != n or len(public_keys) != n:
        raise ValueError("signatures, messages and public keys must have equal length")
    msgs, dst = _h2c_args(messages, dst)
    sigs, pks = _bls_sigs_and_keys(signatures, public_keys)
    if n == 0:
        return []
    try:
        out = bls_verify_messages_batch_packed(sigs, pks, b"".join(msgs), _pack_offsets(msgs), n, dst)
    except NmsmError as e:
        _raise_mapped(e)
    return [b == 1 for b in out]


def bls_verify_messages_batch_packed(sigs96: bytes, pks48: bytes, msgs: bytes, msg_off: bytes, n: int,
                                     dst: bytes) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_verify_msg_batch): n*96 signature bytes, n*48 key bytes, the concatenated
    messages with n+1 little-endian u64 offsets and the tag.  Returns n verdict bytes; raises NmsmError on an error."""
    if len(sigs96) != 96 * n or len(pks48) != 48 * n or len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    _lib.check(lib.nmsm_bls12_381_verify_msg_batch(cp(sigs96 or b"\0"), cp(pks48 or b"\0"), cp(msgs or b"\0"),
                                                   cp(msg_off), n, cp(dst or b"\0"), len(dst), out))
    return out.raw[:n]


# ---- BLS12-381 aggregate verification (include/nmsm.h nmsm_bls12_381_aggregate_verify_batch) ------------------------
def _bls_agg_layout(checks):
    """checks[j] = (signature, [(message bytes, [public keys]), ...]) -> (signature bytes, group offsets, messages, key
    offsets, keys as given).  Type and length checks only; no device."""
    G2 = bls12_381.G2.Point
    sigs, group_off, msgs, key_off, keys = [], [0], [], [0], []
    for j, check in enumerate(checks):
        if not isinstance(check, (tuple, list)) or len(check) != 2:
            raise TypeError("check %d: (signature, [(message, [public keys]), ...]) expected" % j)
        s, groups = check
        sigs.append(s)
        for group in groups:
            if not isinstance(group, (tuple, list)) or len(group) != 2:
                raise TypeError("check %d: (message, [public keys]) groups expected" % j)
            m, ks = group
            if isinstance(m, G2):
                raise TypeError("check %d: messages are hashed here: pass the message bytes, not a G2 Point" % j)
            msgs.append(m)
            keys.extend(ks)
            key_off.append(len(keys))
        group_off.append(len(msgs))
    return sigs, group_off, msgs, key_off, keys


def _bls_agg_keys(keys) -> bytes:
    """the 96-byte affine packing of public keys (48-byte encodings or G1 Points), every one decoded and subgroup-checked
    on the GPU unless it is a Point known valid; a key that fails is packed as the identity, which fails its check"""
    G1 = bls12_381.G1.Point
    for k in keys:
        if isinstance(k, G1):
            continue
        if not isinstance(k, (bytes, bytearray, memoryview)):
            raise TypeError('"publicKey" expected Uint8Array or G1 Point, got type=%s' % type(k).__name__)
        if len(k) != 48:
            raise ValueError('"publicKey" expected Uint8Array of length 48, got length=%d' % len(k))
    ident = bytes(96)
    packed = {}  # unique encodings and Points to check -> packed key
    encs = sorted({bytes(k) for k in keys if not isinstance(k, G1)})
    if encs:
        xy, st = points_decode(BLS12_381_G1, b"".join(encs), len(encs))
        ok = torsion_free_packed(BLS12_381_G1, xy, len(encs))
        for i, e in enumerate(encs):
            packed[e] = xy[96 * i:96 * i + 96] if st[i] == 1 and ok[i] == 1 else ident
    pts = [k for k in keys if isinstance(k, G1) and not k._valid and not k.is0()]
    if pts:
        raw = _pack_points(pts)
        on = points_on_curve(BLS12_381_G1, raw, len(pts))
        ok = torsion_free_packed(BLS12_381_G1, raw, len(pts))
        for i, p in enumerate(pts):
            packed[id(p)] = raw[96 * i:96 * i + 96] if on[i] == 1 and ok[i] == 1 else ident
    out = []
    for k in keys:
        if not isinstance(k, G1):
            out.append(packed[bytes(k)])
        elif k.is0():
            out.append(ident)
        else:
            out.append(packed.get(id(k)) or k.to_packed())
    return b"".join(out)


def bls_aggregate_verify_batch(checks, dst=DST_G2_NUL) -> List[bool]:
    """Aggregate verification over a batch: checks[j] = (signature, [(message bytes, [public keys]), ...]), verdict j is
    e(-G1, sig) prod_g e(sum of group g's keys, hashToCurve(m_g, { DST })) == 1 (noble's verifyBatch with the keys of
    each message summed; one group is FastAggregateVerify).  Signatures are 96-byte encodings or G2 Points, keys 48-byte
    encodings or G1 Points.  A signature or key that does not decode, is the identity or lies outside its subgroup, an
    empty check or group, and a group whose keys sum to the identity are a False verdict.  Byte keys are decoded and
    subgroup-checked once per distinct encoding on the GPU; Points not known valid are checked likewise."""
    checks = list(checks)
    sigs, group_off, msgs, key_off, keys = _bls_agg_layout(checks)
    msgs, dst = _h2c_args(msgs, dst)
    sigs96, _ = _bls_sigs_and_keys(sigs, [])
    if not checks:
        return []
    import struct

    pack = lambda v: struct.pack("<%dQ" % len(v), *v)  # noqa: E731
    try:
        out = bls_aggregate_verify_batch_packed(sigs96, pack(group_off), b"".join(msgs), _pack_offsets(msgs),
                                                _bls_agg_keys(keys), pack(key_off), len(checks), dst)
    except NmsmError as e:
        _raise_mapped(e)
    return [b == 1 for b in out]


def bls_aggregate_verify_batch_packed(sigs96: bytes, group_off: bytes, msgs: bytes, msg_off: bytes, keys_xy: bytes,
                                      key_off: bytes, n_checks: int, dst: bytes) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_aggregate_verify_batch): n_checks*96 signature bytes, n_checks+1 group
    offsets, the concatenated messages with n_groups+1 offsets, 96-byte affine keys with n_groups+1 key offsets (all
    offsets little-endian u64) and the tag.  Returns n_checks verdict bytes; raises NmsmError on an error."""
    if len(sigs96) != 96 * n_checks or len(group_off) != 8 * (n_checks + 1):
        raise ValueError("packed arrays do not match n_checks")
    n_groups = int.from_bytes(group_off[-8:], "little")
    if len(msg_off) != 8 * (n_groups + 1) or len(key_off) != 8 * (n_groups + 1):
        raise ValueError("packed arrays do not match the group count")
    if len(keys_xy) != 96 * int.from_bytes(key_off[-8:], "little"):
        raise ValueError("packed arrays do not match the key count")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n_checks, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    _lib.check(lib.nmsm_bls12_381_aggregate_verify_batch(cp(sigs96 or b"\0"), cp(group_off), n_checks,
                                                         cp(msgs or b"\0"), cp(msg_off), cp(keys_xy or b"\0"),
                                                         cp(key_off), cp(dst or b"\0"), len(dst), out))
    return out.raw[:n_checks]


def bls_fast_aggregate_verify_batch(signatures, messages, public_keys, dst=DST_G2_POP) -> List[bool]:
    """Ethereum's FastAggregateVerify over a batch: verdict j checks signatures[j] over messages[j] against the sum of
    public_keys[j] (a list of keys), under the proof-of-possession tag by default.  Rules as bls_aggregate_verify_batch;
    an empty key list is False."""
    n = len(signatures)
    if len(messages) != n or len(public_keys) != n:
        raise ValueError("signatures, messages and public keys must have equal length")
    return bls_aggregate_verify_batch([(s, [(m, list(ks))]) for s, m, ks in zip(signatures, messages, public_keys)],
                                      dst)


def _bls_verify_batch_groups(messages, publicKeys):
    """noble's verifyBatch pairing of keys with messages: one group per distinct message, in first-seen order"""
    if len(messages) != len(publicKeys):
        raise ValueError("messages and publicKeys must have equal length")
    groups = {}
    for m, k in zip(messages, publicKeys):
        if isinstance(m, bls12_381.G2.Point):
            raise TypeError("verifyBatch hashes the messages: pass the message bytes, not a G2 Point")
        if not isinstance(m, (bytes, bytearray, memoryview)):
            raise TypeError('"message" expected Uint8Array, got type=%s' % type(m).__name__)
        groups.setdefault(bytes(m), []).append(k)
    return list(groups.items())


def _bls_verify_batch(signature, messages, publicKeys) -> bool:
    """bls12_381.verifyBatch(signature, messages, publicKeys) (abstract/bls.ts): one aggregate signature over (message,
    key) pairs, messages as bytes hashed under DST_G2_NUL.  Pairs with equal message bytes form one group whose keys are
    summed.  noble groups by message object identity instead; the verdicts differ in one place: a key and its negation
    under the same message bytes sum to the identity here, which is False (IETF KeyValidate of the aggregate key)."""
    return bls_aggregate_verify_batch([(signature, _bls_verify_batch_groups(messages, publicKeys))])[0]


bls12_381.verifyBatch = _bls_verify_batch


# ---- BLS12-381 hash to G1 and short signatures (include/nmsm.h nmsm_bls12_381_hash_to_g1_batch,
# nmsm_bls12_381_short_verify_batch, nmsm_bls12_381_short_verify_msg_batch) ------------------------------------------
DST_G1_NUL = b"BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_"  # noble's default tag for short signatures
DST_G1_POP = b"BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_POP_"  # proof-of-possession scheme, minimal-signature-size


def bls_hash_to_g1_batch(messages, dst=DST_G1_NUL) -> List:
    """Batch form of bls12_381.G1.hashToCurve(msg, { DST }) (RFC 9380 suite BLS12381G1_XMD:SHA-256_SSWU_RO_): one
    bls12_381.G1.Point per message, each in G1.  Messages are bytes of any length; the tag is non-empty bytes (or str),
    one tag for the whole batch."""
    msgs, dst = _h2c_args(messages, dst)
    if not msgs:
        return []
    xy = bls_hash_to_g1_batch_packed(b"".join(msgs), _pack_offsets(msgs), len(msgs), dst)
    G1 = bls12_381.G1.Point
    out = []
    for k in range(len(msgs)):
        b = xy[96 * k:96 * k + 96]
        out.append(G1.from_packed(b, not any(b), valid=True))
    return out


def bls_hash_to_g1_batch_packed(msgs: bytes, msg_off: bytes, n: int, dst: bytes) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_hash_to_g1_batch): the concatenated messages with n+1 little-endian u64
    offsets and the tag.  Returns n*96 bytes of affine G1 points; raises NmsmError (with .code) on an error."""
    if len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(96 * n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    _lib.check(lib.nmsm_bls12_381_hash_to_g1_batch(cp(msgs or b"\0"), cp(msg_off), n, cp(dst or b"\0"), len(dst), out))
    return out.raw[:96 * n]


def _g1_hash_to_curve(msg, options=None):
    """bls12_381.G1.hashToCurve(msg, { DST }) for one message (the batch entry point with n = 1); the default tag is
    noble's BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_."""
    dst = DST_G1_NUL
    if options is not None:
        if not isinstance(options, dict):
            raise TypeError("options expected dict, got type=%s" % type(options).__name__)
        dst = options.get("DST", DST_G1_NUL)
    return bls_hash_to_g1_batch([msg], dst)[0]


bls12_381.G1.hashToCurve = _g1_hash_to_curve


def _bls_short_sigs_and_keys(signatures, public_keys):
    """the packed signature and key arguments of the short-signature entry points: 48-byte and 96-byte Zcash-flag
    compressed encodings, or Points (encoded first)"""
    G1, G2 = bls12_381.G1.Point, bls12_381.G2.Point
    sigs, pks = [], []
    for s in signatures:
        if isinstance(s, G1):
            s = s.toBytes(True)
        if not isinstance(s, (bytes, bytearray, memoryview)):
            raise TypeError('"signature" expected Uint8Array or G1 Point, got type=%s' % type(s).__name__)
        if len(s) != 48:
            raise ValueError('"signature" expected Uint8Array of length 48, got length=%d' % len(s))
        sigs.append(bytes(s))
    for k in public_keys:
        if isinstance(k, G2):
            k = _bls_g2_compress(k)
        if not isinstance(k, (bytes, bytearray, memoryview)):
            raise TypeError('"publicKey" expected Uint8Array or G2 Point, got type=%s' % type(k).__name__)
        if len(k) != 96:
            raise ValueError('"publicKey" expected Uint8Array of length 96, got length=%d' % len(k))
        pks.append(bytes(k))
    return b"".join(sigs), b"".join(pks)


def bls_short_verify_batch(signatures, message_points, public_keys) -> List[bool]:
    """Batch form of bls12_381.verifyShortSignature(signature, message, publicKey) (public key in G2, signature in G1):
    one verdict per signature.  Signatures are 48-byte and keys 96-byte Zcash-flag compressed encodings, or Points
    (encoded first).  Messages are already hashed to G1 (bls12_381.G1.Point; bls_short_verify_messages_batch takes
    bytes).  A signature or key that does not decode, is the identity or lies outside its subgroup is a False verdict;
    a message point off the curve raises ValueError."""
    n = len(signatures)
    if len(message_points) != n or len(public_keys) != n:
        raise ValueError("signatures, messages and public keys must have equal length")
    sigs, pks = _bls_short_sigs_and_keys(signatures, public_keys)
    G1 = bls12_381.G1.Point
    for m in message_points:
        if not isinstance(m, G1):
            raise TypeError('"message" expected bls12_381.G1.Point (bls_short_verify_messages_batch takes bytes), got '
                            'type=%s' % type(m).__name__)
    if n == 0:
        return []
    try:
        out = bls_short_verify_batch_packed(sigs, pks, _pack_points(message_points), n)
    except NmsmError as e:
        _raise_mapped(e)
    return [b == 1 for b in out]


def bls_short_verify_batch_packed(sigs48: bytes, pks96: bytes, msg_pts: bytes, n: int) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_short_verify_batch): n*48 signature bytes, n*96 key bytes and n*96 bytes
    of affine G1 message points.  Returns n verdict bytes; raises NmsmError (with .code and .index) on an error."""
    if len(sigs48) != 48 * n or len(pks96) != 96 * n or len(msg_pts) != 96 * n:
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    _lib.check(lib.nmsm_bls12_381_short_verify_batch(cp(sigs48 or b"\0"), cp(pks96 or b"\0"), cp(msg_pts or b"\0"), n,
                                                     out))
    return out.raw[:n]


def bls_short_verify_messages_batch(signatures, messages, public_keys, dst=DST_G1_NUL) -> List[bool]:
    """bls_short_verify_batch with message bytes, hashed to G1 on the GPU under dst in the same call: verdict i is
    bls12_381.verifyShortSignature(signature_i, G1.hashToCurve(message_i, { DST }), publicKey_i)."""
    n = len(signatures)
    if len(messages) != n or len(public_keys) != n:
        raise ValueError("signatures, messages and public keys must have equal length")
    msgs, dst = _h2c_args(messages, dst)
    sigs, pks = _bls_short_sigs_and_keys(signatures, public_keys)
    if n == 0:
        return []
    try:
        out = bls_short_verify_messages_batch_packed(sigs, pks, b"".join(msgs), _pack_offsets(msgs), n, dst)
    except NmsmError as e:
        _raise_mapped(e)
    return [b == 1 for b in out]


def bls_short_verify_messages_batch_packed(sigs48: bytes, pks96: bytes, msgs: bytes, msg_off: bytes, n: int,
                                           dst: bytes) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_short_verify_msg_batch): n*48 signature bytes, n*96 key bytes, the
    concatenated messages with n+1 little-endian u64 offsets and the tag.  Returns n verdict bytes; raises NmsmError on
    an error."""
    if len(sigs48) != 48 * n or len(pks96) != 96 * n or len(msg_off) != 8 * (n + 1):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    _lib.check(lib.nmsm_bls12_381_short_verify_msg_batch(cp(sigs48 or b"\0"), cp(pks96 or b"\0"), cp(msgs or b"\0"),
                                                         cp(msg_off), n, cp(dst or b"\0"), len(dst), out))
    return out.raw[:n]


def _bls_verify_short_signature(signature, message, publicKey) -> bool:
    """bls12_381.verifyShortSignature for one signature: a bytes message is hashed to G1 under DST_G1_NUL, as noble
    does; a bls12_381.G1.Point is taken as already hashed."""
    if isinstance(message, (bytes, bytearray, memoryview)):
        return bls_short_verify_messages_batch([signature], [message], [publicKey], DST_G1_NUL)[0]
    return bls_short_verify_batch([signature], [message], [publicKey])[0]


bls12_381.verifyShortSignature = _bls_verify_short_signature


# ---- EIP-4844 KZG proofs (include/nmsm.h nmsm_bls12_381_kzg_verify_proof_batch, nmsm_bls12_381_kzg_verify_blob_batch)
# The consensus specs' verify_kzg_proof / verify_blob_kzg_proof RAISE on malformed input (a length, a point that does
# not decode or lies outside G1, a field element >= r); these batch forms return False for that item instead, as the
# point-evaluation precompile fails the call.  Only the arguments' shapes and the setup point raise.
KZG_FIELD_ELEMENTS_PER_BLOB = 4096
KZG_BYTES_PER_BLOB = 32 * KZG_FIELD_ELEMENTS_PER_BLOB
KZG_BLS_MODULUS = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
POINT_EVALUATION_INPUT_BYTES = 192  # versioned_hash || z || y || commitment || proof
# what the precompile returns on success: FIELD_ELEMENTS_PER_BLOB and BLS_MODULUS as 32-byte big-endian words
POINT_EVALUATION_OUTPUT = KZG_FIELD_ELEMENTS_PER_BLOB.to_bytes(32, "big") + KZG_BLS_MODULUS.to_bytes(32, "big")


def _kzg_bytes(items, width: int, name: str) -> bytes:
    out = []
    for x in items:
        if not isinstance(x, (bytes, bytearray, memoryview)):
            raise TypeError('"%s" expected bytes, got type=%s' % (name, type(x).__name__))
        if len(x) != width:
            raise ValueError('"%s" expected %d bytes, got length=%d' % (name, width, len(x)))
        out.append(bytes(x))
    return b"".join(out)


def _kzg_scalars(items, name: str) -> bytes:
    """z or y values as 32-byte big-endian words: ints in [0, 2^256) or 32-byte values (a value >= r is a False verdict)"""
    out = []
    for x in items:
        if isinstance(x, int) and not isinstance(x, bool):
            if not 0 <= x < 1 << 256:
                raise ValueError('"%s" expected an integer in [0, 2^256), got %d' % (name, x))
            x = x.to_bytes(32, "big")
        out.append(x)
    return _kzg_bytes(out, 32, name)


def _kzg_setup(setup_g2) -> bytes:
    if isinstance(setup_g2, bls12_381.G2.Point):
        setup_g2 = _bls_g2_compress(setup_g2)
    return _kzg_bytes([setup_g2], 96, "setup_g2")


def kzg_verify_proof_batch(commitments, zs, ys, proofs, setup_g2) -> List[bool]:
    """Batch form of the consensus specs' verify_kzg_proof(commitment, z, y, proof) (EIP-4844): one verdict per item.
    Commitments and proofs are 48-byte compressed G1 encodings; z and y are ints or 32-byte big-endian values;
    setup_g2 is [tau] G2 (KZG_SETUP_G2_MONOMIAL[1]) as 96 compressed bytes or a bls12_381.G2.Point.  Malformed items
    are False (the spec raises); a setup point that does not decode or lies outside G2 raises NmsmError (ERR_ARG)."""
    n = len(commitments)
    if len(zs) != n or len(ys) != n or len(proofs) != n:
        raise ValueError("commitments, zs, ys and proofs must have equal length")
    args = (_kzg_bytes(commitments, 48, "commitment"), _kzg_scalars(zs, "z"), _kzg_scalars(ys, "y"),
            _kzg_bytes(proofs, 48, "proof"))
    setup = _kzg_setup(setup_g2)
    if n == 0:
        return []
    return [b == 1 for b in kzg_verify_proof_batch_packed(*args, None, n, setup)]


def kzg_verify_proof_batch_packed(commitments48: bytes, zs32: bytes, ys32: bytes, proofs48: bytes,
                                  versioned_hashes32: Optional[bytes], n: int, setup_g2_96: bytes) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_kzg_verify_proof_batch): n*48 commitment bytes, n*32 z and y bytes
    (big-endian), n*48 proof bytes, n*32 versioned-hash bytes or None, and the 96-byte setup point.  Returns n verdict
    bytes; raises NmsmError (with .code) on an error."""
    if (len(commitments48) != 48 * n or len(zs32) != 32 * n or len(ys32) != 32 * n or len(proofs48) != 48 * n
            or (versioned_hashes32 is not None and len(versioned_hashes32) != 32 * n) or len(setup_g2_96) != 96):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    vh = cp(versioned_hashes32) if versioned_hashes32 is not None else None
    _lib.check(lib.nmsm_bls12_381_kzg_verify_proof_batch(cp(commitments48 or b"\0"), cp(zs32 or b"\0"),
                                                         cp(ys32 or b"\0"), cp(proofs48 or b"\0"), vh, n,
                                                         cp(setup_g2_96), out))
    return out.raw[:n]


def kzg_verify_blob_proof_batch(blobs, commitments, proofs, setup_g2) -> List[bool]:
    """Batch form of the consensus specs' verify_blob_kzg_proof(blob, commitment, proof) (EIP-4844): one verdict per
    blob.  Blobs are KZG_BYTES_PER_BLOB bytes each (4096 big-endian field elements); commitments, proofs and setup_g2
    as for kzg_verify_proof_batch.  A blob with an element >= r, or a malformed point, is False (the spec raises)."""
    n = len(blobs)
    if len(commitments) != n or len(proofs) != n:
        raise ValueError("blobs, commitments and proofs must have equal length")
    args = (_kzg_bytes(blobs, KZG_BYTES_PER_BLOB, "blob"), _kzg_bytes(commitments, 48, "commitment"),
            _kzg_bytes(proofs, 48, "proof"))
    setup = _kzg_setup(setup_g2)
    if n == 0:
        return []
    return [b == 1 for b in kzg_verify_blob_proof_batch_packed(*args, n, setup)]


def kzg_verify_blob_proof_batch_packed(blobs: bytes, commitments48: bytes, proofs48: bytes, n: int,
                                       setup_g2_96: bytes) -> bytes:
    """The C-ABI call itself (nmsm_bls12_381_kzg_verify_blob_batch): n*131072 blob bytes, n*48 commitment and proof
    bytes, the 96-byte setup point.  Returns n verdict bytes; raises NmsmError (with .code) on an error."""
    if (len(blobs) != KZG_BYTES_PER_BLOB * n or len(commitments48) != 48 * n or len(proofs48) != 48 * n
            or len(setup_g2_96) != 96):
        raise ValueError("packed arrays do not match n")
    _lib.ensure_init()
    lib = _lib.load()
    out = ctypes.create_string_buffer(max(n, 1))
    cp = lambda b: ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)  # noqa: E731
    _lib.check(lib.nmsm_bls12_381_kzg_verify_blob_batch(cp(blobs or b"\0"), cp(commitments48 or b"\0"),
                                                        cp(proofs48 or b"\0"), n, cp(setup_g2_96), out))
    return out.raw[:n]


def eth_point_evaluation_batch(inputs, setup_g2) -> List[bool]:
    """Ethereum's point-evaluation precompile (0x0A, EIP-4844) over a batch: True where the precompile succeeds (and
    returns POINT_EVALUATION_OUTPUT), False where it fails.  `inputs` is a list of byte strings or one buffer of
    n * 192 bytes, each versioned_hash || z || y || commitment || proof.  An input that is not 192 bytes is False.  The
    checks: versioned_hash == 0x01 || sha256(commitment)[1:], z and y < r, and verify_kzg_proof."""
    import numpy as np

    W = POINT_EVALUATION_INPUT_BYTES
    if isinstance(inputs, (bytes, bytearray, memoryview)):
        buf = bytes(inputs)
        if len(buf) % W:
            raise ValueError("a packed point-evaluation batch must be a multiple of 192 bytes, got %d" % len(buf))
        items = np.frombuffer(buf, np.uint8).reshape(-1, W)
        good = np.ones(len(items), bool)
    else:
        for x in inputs:
            if not isinstance(x, (bytes, bytearray, memoryview)):
                raise TypeError("point-evaluation input expected bytes, got type=%s" % type(x).__name__)
        good = np.array([len(x) == W for x in inputs], bool)
        items = np.zeros((len(inputs), W), np.uint8)
        for i, x in enumerate(inputs):
            if good[i]:
                items[i] = np.frombuffer(bytes(x), np.uint8)
    setup = _kzg_setup(setup_g2)
    idx = np.flatnonzero(good)
    out = np.zeros(len(good), bool)
    if len(idx) == 0:
        return out.tolist()
    sel = items[idx]
    col = lambda a, b: np.ascontiguousarray(sel[:, a:b]).tobytes()  # noqa: E731
    res = kzg_verify_proof_batch_packed(col(96, 144), col(32, 64), col(64, 96), col(144, 192), col(0, 32), len(idx),
                                        setup)
    out[idx] = np.frombuffer(res, np.uint8) == 1
    return out.tolist()


class KzgSetup:
    """Device-resident EIP-4844 trusted setup for the prover (nmsm_bls12_381_kzg_setup_create): KZG_SETUP_G1_LAGRANGE
    as 4096 x 48 compressed bytes (one buffer or a list), in natural order as the ceremony file lists g1_lagrange.  The
    points are checked to lie in G1 (a bad one raises ValueError; its NmsmError cause carries ERR_POINT and the index)
    and a 1.61 GB table of them is built on the device, freed by close().

    The batch methods are the consensus specs' blob_to_kzg_commitment, compute_kzg_proof and compute_blob_kzg_proof.
    Where the spec raises (a blob element >= r, z >= r, a commitment that fails validate_kzg_g1) the item is None."""

    def __init__(self, g1_lagrange):
        self.handle = 0
        if isinstance(g1_lagrange, (bytes, bytearray, memoryview)):
            buf = bytes(g1_lagrange)
        else:
            buf = _kzg_bytes(g1_lagrange, 48, "g1_lagrange")
        if len(buf) != 48 * KZG_FIELD_ELEMENTS_PER_BLOB:
            raise ValueError("g1_lagrange expected %d points of 48 bytes, got %d bytes"
                             % (KZG_FIELD_ELEMENTS_PER_BLOB, len(buf)))
        _lib.ensure_init()
        self._lib = _lib.load()
        h = ctypes.c_uint64(0)
        try:
            _lib.check(self._lib.nmsm_bls12_381_kzg_setup_create(_kzg_cp(buf), ctypes.byref(h)))
        except NmsmError as e:
            _raise_mapped(e)
        self.handle = h.value

    def blob_to_kzg_commitment_batch_packed(self, blobs: bytes, n: int):
        """The C-ABI call (nmsm_bls12_381_kzg_commit_batch): n*131072 blob bytes -> (n*48 commitment bytes, n ok
        bytes); raises NmsmError on an error."""
        _kzg_check_packed(blobs, n)
        out, ok = ctypes.create_string_buffer(max(48 * n, 1)), ctypes.create_string_buffer(max(n, 1))
        _lib.check(self._lib.nmsm_bls12_381_kzg_commit_batch(self.handle, _kzg_cp(blobs), n, out, ok))
        return out.raw[:48 * n], ok.raw[:n]

    def compute_kzg_proof_batch_packed(self, blobs: bytes, zs32: bytes, n: int):
        """The C-ABI call (nmsm_bls12_381_kzg_compute_proof_batch): n*131072 blob bytes and n*32 big-endian z bytes ->
        (n*48 proof bytes, n*32 y bytes, n ok bytes); raises NmsmError on an error."""
        _kzg_check_packed(blobs, n, zs32, 32)
        out, ys = ctypes.create_string_buffer(max(48 * n, 1)), ctypes.create_string_buffer(max(32 * n, 1))
        ok = ctypes.create_string_buffer(max(n, 1))
        _lib.check(self._lib.nmsm_bls12_381_kzg_compute_proof_batch(self.handle, _kzg_cp(blobs), _kzg_cp(zs32), n, out,
                                                                    ys, ok))
        return out.raw[:48 * n], ys.raw[:32 * n], ok.raw[:n]

    def compute_blob_kzg_proof_batch_packed(self, blobs: bytes, commitments48: bytes, n: int):
        """The C-ABI call (nmsm_bls12_381_kzg_compute_blob_proof_batch): n*131072 blob bytes and n*48 commitment
        bytes -> (n*48 proof bytes, n ok bytes); raises NmsmError on an error."""
        _kzg_check_packed(blobs, n, commitments48, 48)
        out, ok = ctypes.create_string_buffer(max(48 * n, 1)), ctypes.create_string_buffer(max(n, 1))
        _lib.check(self._lib.nmsm_bls12_381_kzg_compute_blob_proof_batch(self.handle, _kzg_cp(blobs),
                                                                         _kzg_cp(commitments48), n, out, ok))
        return out.raw[:48 * n], ok.raw[:n]

    def blob_to_kzg_commitment_batch(self, blobs) -> List[Optional[bytes]]:
        """blob_to_kzg_commitment for each blob: 48 compressed bytes, or None for a blob with an element >= r"""
        n = len(blobs)
        if n == 0:
            return []
        out, ok = self.blob_to_kzg_commitment_batch_packed(_kzg_bytes(blobs, KZG_BYTES_PER_BLOB, "blob"), n)
        return [out[48 * i:48 * i + 48] if ok[i] == 1 else None for i in range(n)]

    def compute_kzg_proof_batch(self, blobs, zs) -> List[Optional[Tuple[bytes, bytes]]]:
        """compute_kzg_proof(blob, z) for each pair: (48-byte proof, 32-byte big-endian y), or None where the spec
        raises.  z is an int in [0, 2^256) or 32 big-endian bytes."""
        n = len(blobs)
        if len(zs) != n:
            raise ValueError("blobs and zs must have equal length")
        args = (_kzg_bytes(blobs, KZG_BYTES_PER_BLOB, "blob"), _kzg_scalars(zs, "z"))
        if n == 0:
            return []
        out, ys, ok = self.compute_kzg_proof_batch_packed(*args, n)
        return [(out[48 * i:48 * i + 48], ys[32 * i:32 * i + 32]) if ok[i] == 1 else None for i in range(n)]

    def compute_blob_kzg_proof_batch(self, blobs, commitments) -> List[Optional[bytes]]:
        """compute_blob_kzg_proof(blob, commitment) for each pair: the 48-byte proof, or None where the spec raises"""
        n = len(blobs)
        if len(commitments) != n:
            raise ValueError("blobs and commitments must have equal length")
        args = (_kzg_bytes(blobs, KZG_BYTES_PER_BLOB, "blob"), _kzg_bytes(commitments, 48, "commitment"))
        if n == 0:
            return []
        out, ok = self.compute_blob_kzg_proof_batch_packed(*args, n)
        return [out[48 * i:48 * i + 48] if ok[i] == 1 else None for i in range(n)]

    def close(self):
        if self.handle:
            self._lib.nmsm_bls12_381_kzg_setup_free(self.handle)
            self.handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _kzg_cp(b: bytes):
    return ctypes.cast(ctypes.c_char_p(b or b"\0"), ctypes.c_void_p)


def _kzg_check_packed(blobs: bytes, n: int, other: bytes = b"", width: int = 0):
    if len(blobs) != KZG_BYTES_PER_BLOB * n or len(other) != width * n:
        raise ValueError("packed arrays do not match n")


# ---- bn254 pairing checks (include/nmsm.h nmsm_bn254_pairing_check_batch) and EIP-197 ecPairing ---------------------
def bn254_pairing_check_batch(checks) -> List[bool]:
    """pairing_check_batch on bn254: checks[j] is a list of (bn254.G1.Point, bn254.G2.Point) pairs, True iff the
    product of their pairings is 1 (noble's bn254.pairingBatch compared with Fp12.ONE).  A pair with an identity point
    contributes 1; points are not subgroup-checked.  Raises ValueError for a point off its curve."""
    args = _pack_pairing_checks(checks, bn254.G1.Point, bn254.G2.Point, "bn254")
    try:
        out = bn254_pairing_check_batch_packed(*args)
    except NmsmError as e:
        _raise_mapped(e)
    return [b == 1 for b in out]


def bn254_pairing_check_batch_packed(g1_xy: bytes, g2_xy: bytes, pair_off: bytes, n_checks: int) -> bytes:
    """The C-ABI call itself (nmsm_bn254_pairing_check_batch): packed affine G1 (64 B) and G2 (128 B) points and
    n_checks + 1 little-endian u64 pair offsets.  Returns n_checks verdict bytes; raises NmsmError (with .code and
    .index) on an error."""
    return _pairing_check_call("nmsm_bn254_pairing_check_batch", 64, g1_xy, g2_xy, pair_off, n_checks)


def bn254_eip197_pairing_batch(inputs) -> List[bool]:
    """Ethereum's ecPairing precompile (EIP-197) over a batch: one input byte string per call, one verdict per input.
    An input is k x 192 bytes, per pair G1 x, y then G2 x_imag, x_real, y_imag, y_real, each 32 B big-endian; an
    all-zero point is the identity; an empty input is True.  Everything the precompile rejects raises ValueError naming
    the input: a length that is not a multiple of 192, a coordinate >= p, a point off its curve, a G2 point outside the
    subgroup (nmsm_points_torsion_free)."""
    import struct

    inputs = list(inputs)
    if not inputs:
        return []
    g1, g2, offs, owner = [], [], [0], []
    for j, data in enumerate(inputs):
        if not isinstance(data, (bytes, bytearray, memoryview)):
            raise TypeError("input %d: bytes expected, got type=%s" % (j, type(data).__name__))
        data = bytes(data)
        if len(data) % 192:
            raise ValueError("input %d: length %d is not a multiple of 192" % (j, len(data)))
        for k in range(0, len(data), 192):
            c = [int.from_bytes(data[k + 32 * i:k + 32 * i + 32], "big") for i in range(6)]
            if any(v >= _BN_P for v in c):
                raise ValueError("input %d: pair %d has a coordinate >= p" % (j, k // 192))
            g1.append(c[0].to_bytes(32, "little") + c[1].to_bytes(32, "little"))
            g2.append(b"".join(c[i].to_bytes(32, "little") for i in (3, 2, 5, 4)))
            owner.append(j)
        offs.append(len(g1))
    n = len(owner)
    g1_xy, g2_xy = b"".join(g1), b"".join(g2)
    if n:
        for what, cid, pts in (("G1", BN254_G1, g1_xy), ("G2", BN254_G2, g2_xy)):
            bad = points_on_curve(cid, pts, n).find(b"\0")
            if bad >= 0:
                raise ValueError("input %d: %s point of pair %d is not on the curve"
                                 % (owner[bad], what, bad - offs[owner[bad]]))
        bad = torsion_free_packed(BN254_G2, g2_xy, n).find(b"\0")
        if bad >= 0:
            raise ValueError("input %d: G2 point of pair %d is not in the subgroup" % (owner[bad], bad - offs[owner[bad]]))
    try:
        out = bn254_pairing_check_batch_packed(g1_xy, g2_xy, struct.pack("<%dQ" % len(offs), *offs), len(inputs))
    except NmsmError as e:
        _raise_mapped(e)
    return [b == 1 for b in out]


DECODE_ZIP215 = 1  # include/nmsm.h NMSM_DECODE_ZIP215


def points_on_curve(curve_id: int, pts: bytes, n: int) -> bytes:
    """Batch curve-equation check (nmsm_points_on_curve; weierstrass.ts:617-624 isValidXY, edwards.ts:461-480): one
    byte per point, 1 = coordinates in range and on the curve (the affine identity encoding counts as on-curve)."""
    _lib.ensure_init()
    lib = _lib.load()
    pb = lib.nmsm_point_bytes(curve_id)
    if len(pts) != n * pb:
        raise ValueError("expected %d bytes per point" % pb)
    out = ctypes.create_string_buffer(max(1, n))
    rc = lib.nmsm_points_on_curve(curve_id, ctypes.cast(ctypes.c_char_p(bytes(pts)), ctypes.c_void_p), n,
                                  ctypes.cast(out, ctypes.c_void_p))
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw[:n]


def points_decode(curve_id: int, encodings: bytes, n: int, zip215: bool = False):
    """Batched `fromBytes` decode step on the GPU (secp256k1 SEC1-33, BLS12-381 G1 Zcash-48 / G2 Zcash-96, ed25519-32):
    returns (packed points, status bytes: 0 invalid / 1 point / 2 infinity).  ed25519: strict RFC 8032 by default
    (the reference's `fromBytes(bytes, zip215 = false)`), ZIP-215 acceptance with zip215=True."""
    _lib.ensure_init()
    lib = _lib.load()
    pb = lib.nmsm_point_bytes(curve_id)
    out = ctypes.create_string_buffer(max(1, n * pb))
    st = ctypes.create_string_buffer(max(1, n))
    rc = lib.nmsm_points_decode_ex(curve_id, ctypes.cast(ctypes.c_char_p(bytes(encodings)), ctypes.c_void_p), n,
                                   DECODE_ZIP215 if zip215 else 0,
                                   ctypes.cast(out, ctypes.c_void_p), ctypes.cast(st, ctypes.c_void_p))
    try:
        _lib.check(rc)
    except NmsmError as e:
        _raise_mapped(e)
    return out.raw[: n * pb], st.raw[:n]


def last_timing():
    """(dict of per-kernel ms, PlanInfo) of the last MSM call when profiling is enabled."""
    lib = _lib.load()
    ms = (ctypes.c_float * _lib.TIMING_SLOTS)()
    info = PlanInfo()
    lib.nmsm_last_timing(ms, ctypes.byref(info))
    return {k: float(ms[i]) for i, k in enumerate(TIMING_NAMES)}, info


def set_profiling(enabled: bool) -> None:
    _lib.load().nmsm_set_profiling(1 if enabled else 0)


def set_window_bits(c: int) -> int:
    return _lib.load().nmsm_set_window_bits(c)


def set_window_groups(groups: int) -> int:
    """Force the number of window groups the MSM pipeline overlaps (0 = automatic); results never depend on it."""
    return _lib.load().nmsm_set_window_groups(groups)


def bench_modmul(field: int, blocks_per_sm: int = 8, threads: int = 128, iters: int = 2000, ilp: int = 1) -> float:
    _lib.ensure_init()
    return float(_lib.load().nmsm_bench_modmul(field, blocks_per_sm, threads, iters, ilp))
