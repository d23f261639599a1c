"""GPU tests of the ping-pong GEMM kernel's shared stage ring: one producer loads the k-blocks of all a CTA's tiles into
one ring of 6 stages, and the two MMA warpgroups take its tiles in turn, so a warpgroup's tile starts at a ring
position offset by the k-blocks of the other's tiles; and of its tile order.  The outputs must stay bitwise equal to
gemm_f16_kernel's."""
import pytest

from test_gemm_pingpong_gpu import check_equal, ops, sms  # noqa: F401  (ops is a fixture)

pytestmark = pytest.mark.gpu


# k-blocks per tile below, equal to and co-prime with the ring's 6 stages
@pytest.mark.parametrize("num_kb", [1, 2, 5, 6, 7, 13])
# tiles per CTA: fewer tiles than SMs (the second MMA warpgroup has no tile at all), one and a half (some CTAs take
# a second tile) and three (the first warpgroup takes one tile more than the second)
@pytest.mark.parametrize("per_cta", [0.5, 1.5, 3])
@pytest.mark.parametrize("ln", [False, True])
@pytest.mark.parametrize("geglu", [False, True])
def test_ring_positions(ops, num_kb, per_cta, ln, geglu):
    k = 64 * num_kb
    tiles = max(1, int(per_cta * sms()))
    n_out = 128 * 8
    per_row = n_out // (64 if geglu else 128)
    m = 128 * (-(-tiles // per_row)) - 37   # ragged last row of tiles
    check_equal(ops, m, 2 * n_out if geglu else n_out, k, geglu, ln=ln, seed=num_kb)


# the kernel walks tiles in bands of 16 row tiles, M fastest inside a band: row-tile counts below, at and past a band
# (a narrower last band), with a column-tile count that is not a multiple of anything
@pytest.mark.parametrize("m_tiles", [15, 16, 17, 33, 50])
@pytest.mark.parametrize("geglu", [False, True])
def test_tile_bands(ops, m_tiles, geglu):
    n_out = 64 * 13 + 40   # 14 column tiles of 64 outputs (GEGLU), 7 of 128 (plain), the last one ragged
    check_equal(ops, 128 * m_tiles - 5, 2 * n_out if geglu else n_out, 320, geglu, seed=m_tiles)
