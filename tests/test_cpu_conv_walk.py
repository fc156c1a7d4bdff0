"""Tile walk of the tensor-core conv's persistent grid, as the host-only planner (sy_conv2d_plan) reports it.

M-band (walk 1): each CTA keeps one N tile and the n_tiles CTAs of a slot walk the same M tiles together, so the
activation operand crosses HBM -> L2 about once per layer.  The planner must take it only where it adds no round of the persistent grid, and
its grid must be a multiple of n_tiles that fits the SMs (one CTA per SM: the BatchNorm grid barrier needs them all)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from streamyolo_b200 import ops  # noqa: E402
from test_gpu_parity_l import L_SHAPES  # noqa: E402


def cdiv(a, b):
    return -(-a // b)


@pytest.mark.parametrize("case", L_SHAPES, ids=lambda c: "x".join(map(str, c)))
def test_walk_never_adds_a_round(case):
    n, ci, co, h, w, k, s, _ = case
    sms = ops.conv_stat_rows()
    p = ops.conv2d_plan(n, h, w, ci, co, k, s)
    tiles = p["m_tiles"] * p["n_tiles"]
    assert p["rounds"] == cdiv(tiles, sms)
    assert 1 <= p["grid"] <= sms
    if p["walk"] == 1:
        assert p["n_tiles"] > 1 and p["grid"] % p["n_tiles"] == 0
        slots = sms // p["n_tiles"]
        assert p["grid"] == slots * p["n_tiles"]
        # slot j walks the M-tile classes j, j + slots, ... < SMs; class rho holds the M tiles rho, rho + SMs, ...
        busiest = max(sum(cdiv(p["m_tiles"] - r, sms) for r in range(j, sms, slots) if r < p["m_tiles"]) for j in range(slots))
        assert busiest <= p["rounds"]
    else:
        assert p["grid"] == min(tiles, sms)


def test_walk_choices():
    sms = ops.conv_stat_rows()
    if sms != 132:
        pytest.skip("choices pinned for 132 SMs (H100 SXM)")
    p = ops.conv2d_plan(16, 19, 30, 2048, 1024, 1, 1)       # 72 x 8 tiles: 16 slots of 8 CTAs, 5 rounds
    assert (p["walk"], p["grid"], p["rounds"]) == (1, 128, 5)
    p = ops.conv2d_plan(16, 38, 60, 512, 512, 1, 1)         # 285 x 4 tiles: 33 slots of 4 CTAs, 9 rounds
    assert (p["walk"], p["grid"], p["rounds"]) == (1, 132, 9)
    p = ops.conv2d_plan(16, 75, 120, 128, 128, 1, 1)        # one N tile: nothing to share
    assert (p["walk"], p["grid"]) == (0, 132)
    p = ops.conv2d_plan(8, 19, 30, 1024, 256, 1, 1)         # 36 x 2 tiles: one round either way
    assert (p["walk"], p["grid"]) == (0, 72)
