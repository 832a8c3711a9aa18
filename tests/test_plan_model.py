"""Host-side plan selection (csrc/msm_body.cuh make_plan / make_table_plan / choose_table_bits), through the host
emulation library: structural invariants the kernels rely on, and the choices the time model makes at the BASELINE sizes."""
import ctypes

import numpy as np
import pytest

import helpers as H

NAMES = ["secp256k1", "ed25519", "bn254_G1", "bn254_G2", "bls12_381_G1", "bls12_381_G2", "bls12_381_G1_any", "bls12_381_G2_any"]
# sub-terms per term (msm_body.cuh split_of): endomorphism halves, or the four psi digits of BLS12-381 G2
SPLIT = {"secp256k1": 2, "bn254_G1": 2, "bls12_381_G1": 2, "bls12_381_G2": 4}


def plan(name, n, table_c=0):
    out = np.zeros(12, np.uint32)
    assert H.hostemu().emu_plan(H.CURVE_IDS[name], n, table_c, out.ctypes.data_as(ctypes.c_void_p)) == 0
    keys = ("c", "W", "B", "L", "K", "chunks", "D", "wb", "r", "stride", "auto_c", "T")
    return dict(zip(keys, (int(v) for v in out)))


@pytest.mark.parametrize("name", NAMES)
def test_ordinary_plans(name):
    for logn in (0, 3, 8, 12, 16, 20, 22):
        p = plan(name, 1 << logn)
        assert 2 <= p["c"] <= 16 and p["B"] == 1 << (p["c"] - 1)
        assert p["W"] * p["c"] >= p["T"] > (p["W"] - 1) * p["c"]          # the windows cover bits + 1 exactly once
        assert p["D"] == p["W"] and p["stride"] == 0 and p["wb"] == p["c"] and p["r"] == 0
        assert p["K"] >= 1 and p["K"] * p["chunks"] == p["B"] and p["K"] & (p["K"] - 1) == 0
        assert 4 <= p["L"] <= 64  # msm_body.cuh plan_seg_len
    big = plan(name, 1 << 20)
    if name == "secp256k1":  # 130 half-scalar bits: c = 16 would leave a 2-bit top window (two giant buckets)
        assert big["c"] == 13 and big["W"] == 10
    elif name in ("bls12_381_G1", "bn254_G1", "bls12_381_G2", "bls12_381_G1_any", "bls12_381_G2_any"):
        assert big["c"] == 16
    else:
        assert 13 <= big["c"] <= 16


@pytest.mark.parametrize("name", NAMES)
def test_table_plans_spread_the_digits_evenly(name):
    for n in (5, 1 << 10, 1 << 20):
        for c_req in range(4, 23):
            p = plan(name, n, c_req)
            T = p["T"]
            assert p["W"] == 1 and p["stride"] == n * SPLIT.get(name, 1)
            assert p["c"] <= c_req and p["B"] == 1 << (p["c"] - 1)
            widths = [p["wb"] + (1 if w < p["r"] else 0) for w in range(p["D"])]
            assert sum(widths) == T and max(widths) == p["c"] and max(widths) - min(widths) <= 1
            # canonical pair: D = ceil(T / c) and c = ceil(T / D)
            assert p["D"] == -(-T // p["c"]) and p["c"] == -(-T // p["D"])
            assert p["K"] * p["chunks"] == p["B"]


def test_table_window_choice_tracks_the_measurements():
    assert plan("bls12_381_G1", 1 << 20)["auto_c"] == 19   # 7 digits
    assert plan("bls12_381_G1", 1 << 16)["auto_c"] == 16
    assert plan("bls12_381_G2", 1 << 18)["auto_c"] == 16
    assert plan("bn254_G1", 1 << 20)["auto_c"] == 19
