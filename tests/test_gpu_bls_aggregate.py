"""BLS12-381 aggregate verification on the GPU (nmsm_bls12_381_aggregate_verify_batch): the contract's edge set against
the oracle (oracle.bls_aggregate_ref), committees of many sizes with verdicts known by construction, one group of 2^20
keys, AggregateVerify checks of many messages (one across a Miller chunk), grouping invariance, agreement with single
verification, the error codes, the Python mirror and the profiling slots."""
import ctypes
import random
import struct

import pytest

import bls_agg_cases as C
from oracle import bls_pairing_ref as B

pytestmark = pytest.mark.gpu

N, P = B.N, B.P
DST = C.DST
TILE = 128  # BLS_KEY_TILE of inst_bls381_pairing.cu


@pytest.fixture(scope="module")
def nmsm():
    import nmsm as m

    m.init(0)
    return m


@pytest.fixture(scope="module")
def table(nmsm):
    t = nmsm.PointTable(nmsm.BLS12_381_G1, nmsm.bls12_381.G1.Point.BASE.to_packed())
    yield t
    t.close()


def _scalars(ks) -> bytes:
    return b"".join((k % N).to_bytes(32, "little") for k in ks)


def _keys(table, sks):
    """sk G1 for each sk (the table multiply of G1's base), 96-byte affine keys"""
    out, _ = table.mul_batch(_scalars(sks), len(sks), False)
    return [out[96 * i:96 * i + 96] for i in range(len(sks))]


def _sig_points(nmsm, msgs, scalars, dst=DST):
    """s_i H(m_i) as packed G2 points: the hash and one G2 multiplication per message on the GPU"""
    offs = [0]
    for m in msgs:
        offs.append(offs[-1] + len(m))
    hs = nmsm.bls_hash_to_g2_batch_packed(b"".join(msgs), struct.pack("<%dQ" % len(offs), *offs), len(msgs), dst)
    out, infs = nmsm.mul_batch_packed(nmsm.BLS12_381_G2, hs, _scalars(scalars), len(msgs), True)
    G2 = nmsm.bls12_381.G2.Point
    return [G2.from_packed(out[192 * i:192 * i + 192], infs[i], True) for i in range(len(msgs))]


def _sigs(nmsm, msgs, scalars, dst=DST):
    return [nmsm._bls_g2_compress(p) for p in _sig_points(nmsm, msgs, scalars, dst)]


def _pack_raw(checks):
    """[(sig96, [(msg, [96-byte keys])])] -> the C ABI's packed arrays"""
    sigs, goff, msgs, moff, keys, koff = [], [0], [], [0], [], [0]
    for sig, groups in checks:
        sigs.append(sig)
        for msg, ks in groups:
            msgs.append(msg)
            moff.append(moff[-1] + len(msg))
            keys.extend(ks)
            koff.append(len(keys))
        goff.append(len(msgs))
    u64 = lambda v: struct.pack("<%dQ" % len(v), *v)  # noqa: E731
    return b"".join(sigs), u64(goff), b"".join(msgs), u64(moff), b"".join(keys), u64(koff)


def _verify(nmsm, checks, dst=DST):
    sigs, goff, msgs, moff, keys, koff = _pack_raw(checks)
    out = nmsm.bls_aggregate_verify_batch_packed(sigs, goff, msgs, moff, keys, koff, len(checks), dst)
    return [b == 1 for b in out]


# ---- the edge set, rule by rule, against the oracle -------------------------------------------------------------------
def test_edge_set_matches_oracle(nmsm):
    cases = C.edge_checks()
    checks = [c for _, c in cases]
    want = C.oracle(checks)
    sigs, goff, msgs, moff, keys, koff = C.pack(checks)
    got = [b == 1 for b in nmsm.bls_aggregate_verify_batch_packed(sigs, goff, msgs, moff, keys, koff, len(checks), DST)]
    assert got == want, [n for (n, _), g, w in zip(cases, got, want) if g != w]
    assert want[0] and not all(want)


# ---- committees of many sizes, verdicts by construction -------------------------------------------------------------
def test_committee_sizes_with_scattered_invalid_checks(nmsm, table):
    sizes = [1, 31, 32, 33, 128, 512, 2048, TILE - 1, TILE, TILE + 1, 2 * TILE + 1]
    n = 4097
    rnd = random.Random(21)
    counts = [sizes[j % len(sizes)] for j in range(n)]
    sks = [rnd.randrange(1, N) for _ in range(sum(counts))]
    keys = _keys(table, sks)
    msgs = [j.to_bytes(32, "big") for j in range(n)]
    scal, want, groups, at = [], [], [], 0
    for j, c in enumerate(counts):
        ks, s = keys[at:at + c], sum(sks[at:at + c]) % N
        at += c
        kind = j % 53
        if kind == 5:  # the signature of another key set
            s = (s + 1) % N
        elif kind == 17:  # one key swapped for another signer's
            ks = ks[:-1] + [keys[(at + 7) % len(keys)]]
        elif kind == 29:  # an identity key next to a valid committee
            ks = ks + [bytes(96)]
        elif kind == 41:  # a wrong message
            groups.append((None, ks))
            scal.append(s)
            want.append(False)
            continue
        groups.append((msgs[j], ks))
        scal.append(s)
        want.append(kind not in (5, 17, 29))
    sigs = _sigs(nmsm, msgs, scal)
    checks = [(sig, [(m if m is not None else msgs[(j + 1) % n], ks)]) for j, (sig, (m, ks)) in
              enumerate(zip(sigs, groups))]
    got = _verify(nmsm, checks)
    assert got == want, [j for j in range(n) if got[j] != want[j]][:20]


def test_one_group_of_2_20_keys(nmsm, table):
    n = 1 << 20
    rnd = random.Random(22)
    sks = [rnd.randrange(1, N) for _ in range(n)]
    keys = _keys(table, sks)
    msg = b"sync committee root"
    sig = _sigs(nmsm, [msg], [sum(sks) % N])[0]
    assert _verify(nmsm, [(sig, [(msg, keys)])]) == [True]
    keys[777777] = _keys(table, [sks[777777] + 1])[0]
    assert _verify(nmsm, [(sig, [(msg, keys)])]) == [False]


# ---- AggregateVerify: many messages in one check ---------------------------------------------------------------------
def _many_message_check(nmsm, table, rnd, count, tag):
    sks = [rnd.randrange(1, N) for _ in range(count)]
    keys = _keys(table, sks)
    msgs = [tag + k.to_bytes(4, "big") for k in range(count)]
    pts = _sig_points(nmsm, msgs, sks)
    G2 = nmsm.bls12_381.G2.Point
    sig = nmsm._bls_g2_compress(nmsm.aggregate_points(G2, pts))
    return sig, [(m, [k]) for m, k in zip(msgs, keys)]


def test_aggregate_verify_4097_distinct_messages(nmsm, table):
    rnd = random.Random(23)
    sig, groups = _many_message_check(nmsm, table, rnd, 4097, b"msg")
    bad = list(groups)
    bad[4000] = (bad[4000][0] + b"!", bad[4000][1])
    assert _verify(nmsm, [(sig, groups), (sig, bad)]) == [True, False]


def test_aggregate_verify_across_a_miller_chunk(nmsm, table):
    """a check of 2^16 + 100 pairs between two small checks: its partial product crosses the chunk boundary"""
    rnd = random.Random(24)
    s1, g1 = _many_message_check(nmsm, table, rnd, 3, b"a")
    sb, gb = _many_message_check(nmsm, table, rnd, (1 << 16) + 99, b"big")
    s2, g2 = _many_message_check(nmsm, table, rnd, 5, b"c")
    assert _verify(nmsm, [(s1, g1), (sb, gb), (s2, g2)]) == [True, True, True]
    gb_bad = list(gb)
    gb_bad[-3] = (gb_bad[-3][0], gb[-2][1])
    assert _verify(nmsm, [(s1, g1), (sb, gb_bad), (s2, g2)]) == [True, False, True]


def test_grouping_invariance(nmsm, table):
    """one (message, key) multiset: one group per key and grouped by message give the same verdicts"""
    rnd = random.Random(25)
    sks = [rnd.randrange(1, N) for _ in range(12)]
    keys = _keys(table, sks)
    msgs = [b"m%d" % (k % 3) for k in range(12)]
    sig = nmsm._bls_g2_compress(nmsm.aggregate_points(nmsm.bls12_381.G2.Point, _sig_points(nmsm, msgs, sks)))
    other = _sigs(nmsm, [b"x"], [5])[0]
    per_key = [(m, [k]) for m, k in zip(msgs, keys)]
    by_msg = [(b"m%d" % i, [keys[k] for k in range(12) if k % 3 == i]) for i in range(3)]
    got = _verify(nmsm, [(sig, per_key), (sig, by_msg), (other, per_key), (other, by_msg)])
    assert got == [True, True, False, False]


def test_one_key_checks_agree_with_single_verification(nmsm, table):
    rnd = random.Random(26)
    n = 64
    sks = [rnd.randrange(1, N) for _ in range(n)]
    keys = _keys(table, sks)
    msgs = [bytes(rnd.randrange(256) for _ in range(rnd.randrange(80))) for _ in range(n)]
    sigs = _sigs(nmsm, msgs, sks)
    for k in range(0, n, 5):
        sigs[k] = sigs[(k + 1) % n]
    G1 = nmsm.bls12_381.G1.Point
    pks = [G1.from_packed(k, 0, True).toBytes(True) for k in keys]
    want = nmsm.bls_verify_messages_batch(sigs, msgs, pks, DST)
    assert _verify(nmsm, [(s, [(m, [k])]) for s, m, k in zip(sigs, msgs, keys)]) == want
    assert want.count(False) == len(range(0, n, 5))


# ---- errors -----------------------------------------------------------------------------------------------------------
def test_bad_key_errors_report_the_smallest_index(nmsm, table):
    keys = _keys(table, [3, 4, 5])
    sig = _sigs(nmsm, [b"m"], [12])[0]
    off_curve = (1).to_bytes(48, "little") * 2
    big_x = P.to_bytes(48, "little") + keys[0][48:]
    for checks, idx in (([(sig, [(b"m", keys)]), (sig, [(b"m", keys[:2] + [off_curve]), (b"n", [big_x])])], 5),
                        ([(sig, [(b"m", keys)]), (sig, [(b"m", [big_x] + keys[:2])])], 3)):
        with pytest.raises(nmsm.NmsmError) as e:
            _verify(nmsm, checks)
        assert e.value.code == nmsm._lib.ERR_POINT and e.value.index == idx
    assert _verify(nmsm, [(sig, [(b"m", keys)])]) == [True]  # the context is still good


def test_argument_errors(nmsm):
    lib = nmsm._lib.load()
    ERR_ARG = nmsm._lib.ERR_ARG
    u64 = lambda *v: (ctypes.c_uint64 * len(v))(*v)  # noqa: E731
    sig, key = ctypes.c_char_p(bytes(96)), ctypes.c_char_p(bytes(96))
    m, d = ctypes.c_char_p(b"m"), ctypes.c_char_p(b"D")
    goff, moff, koff = u64(0, 1), u64(0, 1), u64(0, 1)
    out = ctypes.create_string_buffer(b"\x5a" * 2, 2)
    call = lambda s, g, n, mm, mo, k, ko, dd, dl: lib.nmsm_bls12_381_aggregate_verify_batch(  # noqa: E731
        s, g, n, mm, mo, k, ko, dd, dl, out)
    assert call(sig, goff, 1, m, moff, key, koff, d, 0) == ERR_ARG  # empty tag
    assert call(sig, goff, 1, m, moff, key, koff, None, 1) == ERR_ARG
    assert call(None, goff, 1, m, moff, key, koff, d, 1) == ERR_ARG
    assert call(sig, goff, 1, None, moff, key, koff, d, 1) == ERR_ARG
    assert call(sig, goff, 1, m, moff, None, koff, d, 1) == ERR_ARG
    assert call(sig, goff, 1 << 30, m, moff, key, koff, d, 1) == ERR_ARG
    assert call(sig, u64(1, 1), 1, m, moff, key, koff, d, 1) == ERR_ARG
    assert b"group_off" in lib.nmsm_last_error()
    assert call(sig, u64(0, 2), 1, m, u64(0, 1, 0), key, u64(0, 1, 1), d, 1) == ERR_ARG
    assert b"msg_off" in lib.nmsm_last_error() and lib.nmsm_last_error_index() == 2
    assert call(sig, u64(0, 2), 1, m, u64(0, 1, 1), key, u64(0, 1, 0), d, 1) == ERR_ARG
    assert b"key_off" in lib.nmsm_last_error()
    assert call(sig, u64(0, 1 << 31), 1, m, moff, key, koff, d, 1) == ERR_ARG
    assert call(sig, goff, 1, m, moff, key, u64(0, 1 << 31), d, 1) == ERR_ARG
    assert out.raw == b"\x5a" * 2
    assert call(None, None, 0, None, None, None, None, d, 1) == 0  # n_checks == 0 writes nothing
    assert out.raw == b"\x5a" * 2


def test_empty_checks_and_groups(nmsm, table):
    keys = _keys(table, [7])
    sig = _sigs(nmsm, [b"m"], [7])[0]
    assert _verify(nmsm, [(sig, [])]) == [False]
    assert _verify(nmsm, [(sig, []), (sig, [(b"m", keys)]), (sig, [(b"m", keys), (b"n", [])])]) == [False, True, False]


# ---- the mirror, interleaved with other work, and the profiling slots --------------------------------------------------
def test_profiling_slots(nmsm, table):
    keys = _keys(table, [3, 4, 5, 6])
    sig = _sigs(nmsm, [b"m"], [18])[0]
    nmsm.set_profiling(True)
    try:
        assert _verify(nmsm, [(sig, [(b"m", keys)])] * 3) == [True] * 3
        ms, _ = nmsm.last_timing()
        slots = [ms[k] for k in ("prepare", "count", "scan", "scatter", "accumulate")]
        assert all(v > 0 for v in slots) and ms["total"] == pytest.approx(sum(slots), rel=1e-4)
    finally:
        nmsm.set_profiling(False)


def test_mirror_and_state(nmsm, table):
    rnd = random.Random(27)
    G1 = nmsm.bls12_381.G1.Point
    sks = [rnd.randrange(1, N) for _ in range(6)]
    pts = [G1.BASE.multiply(k) for k in sks]
    encs = [p.toBytes(True) for p in pts]
    msg = b"\x11" * 32
    sig = _sigs(nmsm, [msg], [sum(sks[:4])])[0]
    off = B.g1_encode(B.G1.fromAffine(dict(zip("xy", C.BC.g1_off_subgroup(rnd)))))
    for _ in range(2):
        assert nmsm.bls_fast_aggregate_verify_batch(
            [sig, sig, sig, sig], [msg, msg, msg, b"other"],
            [encs[:4], pts[:2] + encs[2:4], encs[:4] + [off], encs[:4]]) == [True, True, False, False]
        assert nmsm.bls_verify_messages_batch(_sigs(nmsm, [b"v"], [sks[5]], nmsm.DST_G2_NUL), [b"v"], [encs[5]]) == [True]
        # verifyBatch: pairs with equal messages are one group; the tag is noble's NUL tag
        vb = nmsm._bls_g2_compress(nmsm.aggregate_points(nmsm.bls12_381.G2.Point, _sig_points(
            nmsm, [b"a", b"b", b"a"], sks[:3], nmsm.DST_G2_NUL)))
        assert nmsm.bls12_381.verifyBatch(vb, [b"a", b"b", b"a"], encs[:3])
        assert not nmsm.bls12_381.verifyBatch(vb, [b"a", b"b", b"b"], encs[:3])
        assert nmsm.aggregate_points(G1, pts).toBytes(True) == G1.BASE.multiply(sum(sks) % N).toBytes(True)
        nmsm._lib.load().nmsm_shutdown()
        nmsm._lib.check(nmsm._lib.load().nmsm_init(0))
