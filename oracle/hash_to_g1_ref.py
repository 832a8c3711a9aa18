"""Hash to BLS12-381 G1, suite BLS12381G1_XMD:SHA-256_SSWU_RO_ (RFC 9380 §8.8.1; next-row f13), and short-signature
verification: the oracle nmsm_bls12_381_hash_to_g1_batch and nmsm_bls12_381_short_verify[_msg]_batch are checked
against.

A plain Python-int restatement of noble-curves' bls12_381.G1.hashToCurve(msg, { DST }) and verifyShortSignature
(abstract/hash-to-curve.ts, abstract/bls.ts, bls12-381.ts): expand_message_xmd and the oversize-tag rule are
oracle.hash_to_curve_ref's; hash_to_field (§5.2, count 2, m 1, L 64), the simplified SWU map on E1' written straight
from §6.6.2 (two square-root attempts, not the device's one-exponentiation form), the 11-isogeny to E1 (§E.2) by its
rational map, and clear_cofactor as the scalar multiplication by h_eff = 1 - x.  Points are affine (x, y) tuples, None
for the identity.  Test infrastructure only.
"""
from __future__ import annotations

from oracle import bls_pairing_ref as B
from oracle import noble_ref as R
from oracle.hash_to_curve_ref import dst_prime_tag, expand_message_xmd  # noqa: F401  (the shared expander)

P = 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB
N = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
X = -0xD201000000010000  # the BLS parameter
H_EFF = 1 - X
assert H_EFF == 0xD201000000010001

DST_G1_NUL = b"BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_"  # noble's default for short signatures
DST_G1_POP = b"BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_POP_"
DST_QUUX = b"QUUX-V01-CS02-with-BLS12381G1_XMD:SHA-256_SSWU_RO_"  # RFC 9380 J.9.1


def inv(a: int) -> int:
    return pow(a, P - 2, P)


def sqrt(a: int):
    """a square root of a mod p, or None (p = 3 mod 4)"""
    r = pow(a, (P + 1) // 4, P)
    return r if r * r % P == a % P else None


def sgn0(a: int) -> int:
    return a & 1


# ---- hash_to_field ----------------------------------------------------------------------------------------------
def hash_to_field(msg: bytes, dst: bytes):
    """count = 2, m = 1, L = 64 (len_in_bytes = 128): [u0, u1]"""
    uniform = expand_message_xmd(msg, dst, 128)
    return [int.from_bytes(uniform[64 * k:64 * k + 64], "big") % P for k in range(2)]


# ---- simplified SWU on E1' and the 11-isogeny ----------------------------------------------------------------------
A_ISO = 0x144698A3B8E9433D693A02C96D4982B0EA985383EE66A8D8E8981AEFD881AC98936F8DA0E0F97F5CF428082D584C1D
B_ISO = 0x12E2908D11688030018B12E8753EEE3B2016C1F0F24F4070A0B9C14FCEF35EF55A23215A316CEAA5D1CC48E98E172BE0
Z_SSWU = 11


def g_iso(x: int) -> int:
    return (x * x * x + A_ISO * x + B_ISO) % P


def map_to_curve_sswu(u: int):
    """§6.6.2 straight from its definition: the point (x, y) of E1': y^2 = x^3 + A' x + B'"""
    zu2 = Z_SSWU * u * u % P
    tv1 = (zu2 * zu2 + zu2) % P
    if tv1 == 0:
        x1 = B_ISO * inv(Z_SSWU * A_ISO) % P
    else:
        x1 = -B_ISO * inv(A_ISO) * (1 + inv(tv1)) % P
    x, y = x1, sqrt(g_iso(x1))
    if y is None:
        x = zu2 * x1 % P
        y = sqrt(g_iso(x))
    assert y is not None and y * y % P == g_iso(x)
    if sgn0(u) != sgn0(y):
        y = (-y) % P
    return x, y


# §E.2: x = x_num / x_den, y = y' y_num / y_den; coefficients from the constant term up (x_den, y_den monic)
ISO_XNUM = [
    0x11A05F2B1E833340B809101DD99815856B303E88A2D7005FF2627B56CDB4E2C85610C2D5F2E62D6EAEAC1662734649B7,
    0x17294ED3E943AB2F0588BAB22147A81C7C17E75B2F6A8417F565E33C70D1E86B4838F2A6F318C356E834EEF1B3CB83BB,
    0x0D54005DB97678EC1D1048C5D10A9A1BCE032473295983E56878E501EC68E25C958C3E3D2A09729FE0179F9DAC9EDCB0,
    0x1778E7166FCC6DB74E0609D307E55412D7F5E4656A8DBF25F1B33289F1B330835336E25CE3107193C5B388641D9B6861,
    0x0E99726A3199F4436642B4B3E4118E5499DB995A1257FB3F086EEB65982FAC18985A286F301E77C451154CE9AC8895D9,
    0x1630C3250D7313FF01D1201BF7A74AB5DB3CB17DD952799B9ED3AB9097E68F90A0870D2DCAE73D19CD13C1C66F652983,
    0x0D6ED6553FE44D296A3726C38AE652BFB11586264F0F8CE19008E218F9C86B2A8DA25128C1052ECADDD7F225A139ED84,
    0x17B81E7701ABDBE2E8743884D1117E53356DE5AB275B4DB1A682C62EF0F2753339B7C8F8C8F475AF9CCB5618E3F0C88E,
    0x080D3CF1F9A78FC47B90B33563BE990DC43B756CE79F5574A2C596C928C5D1DE4FA295F296B74E956D71986A8497E317,
    0x169B1F8E1BCFA7C42E0C37515D138F22DD2ECB803A0C5C99676314BAF4BB1B7FA3190B2EDC0327797F241067BE390C9E,
    0x10321DA079CE07E272D8EC09D2565B0DFA7DCCDDE6787F96D50AF36003B14866F69B771F8C285DECCA67DF3F1605FB7B,
    0x06E08C248E260E70BD1E962381EDEE3D31D79D7E22C837BC23C0BF1BC24C6B68C24B1B80B64D391FA9C8BA2E8BA2D229]
ISO_XDEN = [
    0x08CA8D548CFF19AE18B2E62F4BD3FA6F01D5EF4BA35B48BA9C9588617FC8AC62B558D681BE343DF8993CF9FA40D21B1C,
    0x12561A5DEB559C4348B4711298E536367041E8CA0CF0800C0126C2588C48BF5713DAA8846CB026E9E5C8276EC82B3BFF,
    0x0B2962FE57A3225E8137E629BFF2991F6F89416F5A718CD1FCA64E00B11ACEACD6A3D0967C94FEDCFCC239BA5CB83E19,
    0x03425581A58AE2FEC83AAFEF7C40EB545B08243F16B1655154CCA8ABC28D6FD04976D5243EECF5C4130DE8938DC62CD8,
    0x13A8E162022914A80A6F1D5F43E7A07DFFDFC759A12062BB8D6B44E833B306DA9BD29BA81F35781D539D395B3532A21E,
    0x0E7355F8E4E667B955390F7F0506C6E9395735E9CE9CAD4D0A43BCEF24B8982F7400D24BC4228F11C02DF9A29F6304A5,
    0x0772CAACF16936190F3E0C63E0596721570F5799AF53A1894E2E073062AEDE9CEA73B3538F0DE06CEC2574496EE84A3A,
    0x14A7AC2A9D64A8B230B3F5B074CF01996E7F63C21BCA68A81996E1CDF9822C580FA5B9489D11E2D311F7D99BBDCC5A5E,
    0x0A10ECF6ADA54F825E920B3DAFC7A3CCE07F8D1D7161366B74100DA67F39883503826692ABBA43704776EC3A79A1D641,
    0x095FC13AB9E92AD4476D6E3EB3A56680F682B4EE96F7D03776DF533978F31C1593174E4B4B7865002D6384D168ECDD0A,
    1]
ISO_YNUM = [
    0x090D97C81BA24EE0259D1F094980DCFA11AD138E48A869522B52AF6C956543D3CD0C7AEE9B3BA3C2BE9845719707BB33,
    0x134996A104EE5811D51036D776FB46831223E96C254F383D0F906343EB67AD34D6C56711962FA8BFE097E75A2E41C696,
    0x00CC786BAA966E66F4A384C86A3B49942552E2D658A31CE2C344BE4B91400DA7D26D521628B00523B8DFE240C72DE1F6,
    0x01F86376E8981C217898751AD8746757D42AA7B90EEB791C09E4A3EC03251CF9DE405ABA9EC61DECA6355C77B0E5F4CB,
    0x08CC03FDEFE0FF135CAF4FE2A21529C4195536FBE3CE50B879833FD221351ADC2EE7F8DC099040A841B6DAECF2E8FEDB,
    0x16603FCA40634B6A2211E11DB8F0A6A074A7D0D4AFADB7BD76505C3D3AD5544E203F6326C95A807299B23AB13633A5F0,
    0x04AB0B9BCFAC1BBCB2C977D027796B3CE75BB8CA2BE184CB5231413C4D634F3747A87AC2460F415EC961F8855FE9D6F2,
    0x0987C8D5333AB86FDE9926BD2CA6C674170A05BFE3BDD81FFD038DA6C26C842642F64550FEDFE935A15E4CA31870FB29,
    0x09FC4018BD96684BE88C9E221E4DA1BB8F3ABD16679DC26C1E8B6E6A1F20CABE69D65201C78607A360370E577BDBA587,
    0x0E1BBA7A1186BDB5223ABDE7ADA14A23C42A0CA7915AF6FE06985E7ED1E4D43B9B3F7055DD4EBA6F2BAFAAEBCA731C30,
    0x19713E47937CD1BE0DFD0B8F1D43FB93CD2FCBCB6CAF493FD1183E416389E61031BF3A5CCE3FBAFCE813711AD011C132,
    0x18B46A908F36F6DEB918C143FED2EDCC523559B8AAF0C2462E6BFE7F911F643249D9CDF41B44D606CE07C8A4D0074D8E,
    0x0B182CAC101B9399D155096004F53F447AA7B12A3426B08EC02710E807B4633F06C851C1919211F20D4C04F00B971EF8,
    0x0245A394AD1ECA9B72FC00AE7BE315DC757B3B080D4C158013E6632D3C40659CC6CF90AD1C232A6442D9D3F5DB980133,
    0x05C129645E44CF1102A159F748C4A3FC5E673D81D7E86568D9AB0F5D396A7CE46BA1049B6579AFB7866B1E715475224B,
    0x15E6BE4E990F03CE4EA50B3B42DF2EB5CB181D8F84965A3957ADD4FA95AF01B2B665027EFEC01C7704B456BE69C8B604]
ISO_YDEN = [
    0x16112C4C3A9C98B252181140FAD0EAE9601A6DE578980BE6EEC3232B5BE72E7A07F3688EF60C206D01479253B03663C1,
    0x1962D75C2381201E1A0CBD6C43C348B885C84FF731C4D59CA4A10356F453E01F78A4260763529E3532F6102C2E49A03D,
    0x058DF3306640DA276FAAAE7D6E8EB15778C4855551AE7F310C35A5DD279CD2ECA6757CD636F96F891E2538B53DBF67F2,
    0x16B7D288798E5395F20D23BF89EDB4D1D115C5DBDDBCD30E123DA489E726AF41727364F2C28297ADA8D26D98445F5416,
    0x0BE0E079545F43E4B00CC912F8228DDCC6D19C9F0F69BBB0542EDA0FC9DEC916A20B15DC0FD2EDEDDA39142311A5001D,
    0x08D9E5297186DB2D9FB266EAAC783182B70152C65550D881C5ECD87B6F0F5A6449F38DB9DFA9CCE202C6477FAAF9B7AC,
    0x166007C08A99DB2FC3BA8734ACE9824B5EECFDFA8D0CF8EF5DD365BC400A0051D5FA9C01A58B1FB93D1A1399126A775C,
    0x16A3EF08BE3EA7EA03BCDDFABBA6FF6EE5A4375EFA1F4FD7FEB34FD206357132B920F5B00801DEE460EE415A15812ED9,
    0x1866C8ED336C61231A1BE54FD1D74CC4F9FB0CE4C6AF5920ABC5750C4BF39B4852CFE2F7BB9248836B233D9D55535D4A,
    0x167A55CDA70A6E1CEA820597D94A84903216F763E13D87BB5308592E7EA7D4FBC7385EA3D529B35E346EF48BB8913F55,
    0x04D2F259EEA405BD48F010A01AD2911D9C6DD039BB61A6290E591B36E636A5C871A5C29F4F83060400F8B49CBA8F6AA8,
    0x0ACCBB67481D033FF5852C1E48C50C477F94FF8AEFCE42D28C0F9A88CEA7913516F968986F7EBBEA9684B529E2561092,
    0x0AD6B9514C767FE3C3613144B45F1496543346D98ADF02267D5CEEF9A00D9B8693000763E3B90AC11E99B138573345CC,
    0x02660400EB2E4F3B628BDD0D53CD76F2BF565B94E72927C1CB748DF27942480E420517BD8714CC80D1FADC1326ED06F7,
    0x0E0FA1D816DDC03E6B24255E0D7819C171C40F65E273B853324EFCD6356CAA205CA2F570F13497804415473A1D634B8F,
    1]


def _poly(coeffs, x: int) -> int:
    r = 0
    for c in reversed(coeffs):
        r = (r * x + c) % P
    return r


def iso_map(pt):
    """§E.2: E1' -> E1; a point of the isogeny's kernel maps to the identity (None)"""
    x, y = pt
    xd, yd = _poly(ISO_XDEN, x), _poly(ISO_YDEN, x)
    if xd == 0 or yd == 0:
        return None
    return _poly(ISO_XNUM, x) * inv(xd) % P, y * _poly(ISO_YNUM, x) * inv(yd) % P


# ---- E1: y^2 = x^3 + 4 ---------------------------------------------------------------------------------------------
def on_e1(pt) -> bool:
    return pt is None or (pt[1] * pt[1] - pt[0] ** 3 - 4) % P == 0


def point_add(p1, p2):
    """the affine group law of E1, complete (identity None, P + P, P + (-P))"""
    if p1 is None:
        return p2
    if p2 is None:
        return p1
    if p1[0] == p2[0]:
        if p1[1] != p2[1] or p1[1] == 0:
            return None
        lam = 3 * p1[0] * p1[0] * inv(2 * p1[1]) % P
    else:
        lam = (p2[1] - p1[1]) * inv(p2[0] - p1[0]) % P
    x3 = (lam * lam - p1[0] - p2[0]) % P
    return x3, (lam * (p1[0] - x3) - p1[1]) % P


def point_neg(pt):
    return None if pt is None else (pt[0], (-pt[1]) % P)


def scalar_mul(k: int, pt):
    """k pt for k >= 0 by double-and-add in Jacobian coordinates (one inversion at the end)"""
    if pt is None or k == 0:
        return None
    X1, Y1 = pt
    acc = None  # (X, Y, Z)

    def dbl(q):
        X, Y, Z = q
        if Y == 0:
            return None
        A, Bq = X * X % P, Y * Y % P
        C = Bq * Bq % P
        D = 2 * ((X + Bq) ** 2 - A - C) % P
        E = 3 * A % P
        X3 = (E * E - 2 * D) % P
        return X3, (E * (D - X3) - 8 * C) % P, 2 * Y * Z % P

    def madd(q):  # q + (X1, Y1) with Z1 = 1
        if q is None:
            return (X1, Y1, 1)
        X, Y, Z = q
        ZZ = Z * Z % P
        H, Rr = (X1 * ZZ - X) % P, (Y1 * ZZ * Z - Y) % P
        if H == 0:
            return dbl(q) if Rr == 0 else None
        HH = H * H % P
        HHH, V = HH * H % P, X * HH % P
        X3 = (Rr * Rr - HHH - 2 * V) % P
        return X3, (Rr * (V - X3) - Y * HHH) % P, Z * H % P

    for bit in bin(k)[2:]:
        if acc is not None:
            acc = dbl(acc)
        if bit == "1":
            acc = madd(acc)
    if acc is None:
        return None
    zi = inv(acc[2])
    return acc[0] * zi * zi % P, acc[1] * zi * zi * zi % P


def clear_cofactor(pt):
    return scalar_mul(H_EFF, pt)


def in_g1(pt) -> bool:
    return on_e1(pt) and scalar_mul(N, pt) is None


def map_to_curve(u: int):
    """map_to_curve of the suite: iso_map(simplified SWU(u)), a point of E1 (None: the identity)"""
    return iso_map(map_to_curve_sswu(u))


def hash_to_g1(msg: bytes, dst: bytes = DST_G1_NUL):
    """hash_to_curve (§3): clear_cofactor(map_to_curve(u0) + map_to_curve(u1))"""
    if not isinstance(msg, (bytes, bytearray)) or not isinstance(dst, (bytes, bytearray)):
        raise TypeError("bytes expected")
    if len(dst) == 0:
        raise ValueError("DST must be non-empty")
    u0, u1 = hash_to_field(bytes(msg), bytes(dst))
    return clear_cofactor(point_add(map_to_curve(u0), map_to_curve(u1)))


def g1_packed(pt) -> bytes:
    """the G1 packing of include/nmsm.h: x, y, 48 B little-endian each; the identity is all zero"""
    if pt is None:
        return bytes(96)
    return pt[0].to_bytes(48, "little") + pt[1].to_bytes(48, "little")


# ---- short signatures (bls12_381.verifyShortSignature) ----------------------------------------------------------
def g1_encode(pt) -> bytes:
    """48-byte Zcash-flag compressed encoding of an affine G1 tuple (None: the identity)"""
    if pt is None:
        return bytes([0xC0]) + bytes(47)
    b = bytearray(pt[0].to_bytes(48, "big"))
    b[0] |= 0x80 | (0x20 if (2 * pt[1]) // P else 0)
    return bytes(b)


def public_key(sk: int) -> bytes:
    """sk G2, 96-byte compressed (the short-signature scheme's key)"""
    return B.g2_encode(B.G2.BASE.multiply(sk))


def sign(sk: int, H) -> bytes:
    """sk H for the G1 point H = hash_to_g1(m) (noble's signShortSignature with the message already hashed)"""
    return g1_encode(scalar_mul(sk % N, H))


def short_verify(sig48: bytes, H, pk96: bytes) -> bool:
    """noble's bls12_381.verifyShortSignature(signature, message, publicKey) with the message already hashed to the G1
    point H (affine tuple, None or (0, 0) the identity): sig and pk must decode, be non-identity and lie in their
    subgroups; H must not be the identity; then e(H, pk) e(sig, -G2) == 1."""
    if H is None or H == (0, 0):
        return False
    if len(sig48) != 48 or len(pk96) != 96:
        return False
    try:
        sig = R.bls12_381_g1_decode(sig48)
        pk = R.bls12_381_g2_decode(pk96)
    except ValueError:
        return False
    if B.is_identity_g1(sig) or B.is_identity_g2(pk):
        return False
    if not in_g1(sig):
        return False
    if not B.torsion_free(B.G2.fromAffine({"x": pk[0], "y": pk[1]})):
        return False
    neg_g2 = B.affine(B.G2.BASE.negate())
    return B.pairing_check([(H, pk), (sig, neg_g2)])
