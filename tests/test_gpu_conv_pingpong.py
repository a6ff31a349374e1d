"""conv_tc_kernel's ping-pong schedule: the two consumer warpgroups take alternate tiles of a CTA's static tile list
(grid = min(tiles, 132)).  Cases at the schedule's edges -- one, exactly two and an odd number of tiles per CTA, the
two warpgroups on different N tiles, every A-feeding mode, the head scatter, residual + out1 + out2, K-step
skipping -- against the float64 bound of _conv_case, and two launches bit-identical."""
import numpy as np
import pytest

from test_gpu_conv import _conv_case

pytestmark = pytest.mark.gpu

# id: (B, H, W, Cin, Cout, k, stride, dil), _conv_case keywords, environment
CASES = {
    # halo-flat, Cout 128 (one N tile): Q = B*(H+2)*(W+2) over 128-row tiles
    "flat_one_tile_per_cta": ((1, 62, 126, 64, 128, 3, 1, 1), {"in_halo": 1}, {}),            # 64 tiles
    "flat_two_tiles_per_cta": ((1, 130, 254, 64, 128, 3, 1, 1), {"in_halo": 1}, {}),          # 264 tiles
    "flat_three_tiles_per_cta": ((1, 174, 286, 64, 128, 3, 1, 1), {"in_halo": 1}, {}),        # 396 tiles
    "flat_ragged_tiles_per_cta": ((3, 75, 75, 64, 128, 3, 1, 1), {"in_halo": 1, "out_halo": 1}, {}),  # 139 tiles
    # im2col, Cout 640 = five N tiles of 128: 132 % 5 != 0, so a CTA's consecutive tiles (one per warpgroup)
    # sit on different N tiles and each warpgroup stages its own parameters
    "im2col_odd_n_tiles": ((8, 38, 38, 128, 640, 3, 1, 1), {"act": "leaky"}, {}),             # 455 tiles
    "im2col_one_tile_per_cta": ((1, 19, 19, 256, 256, 3, 1, 1), {}, {}),
    # row-block + fused pool: one, and five or six tiles per CTA
    "rowblock_pool_one_tile_per_cta": ((1, 16, 130, 64, 28, 3, 1, 1), {"in_halo": 1, "pool": 2}, {"ODT_TC_TAPN": "0"}),
    "rowblock_pool_many_tiles": ((1, 300, 300, 64, 64, 3, 1, 1), {"in_halo": 1, "out_halo": 1, "pool": 2},
                                 {"ODT_TC_TAPN": "0"}),
    # fp32 head scatter (column-wise reads of the staged slice) from the halo-flat and the im2col modes
    "head_flat": ((8, 64, 64, 256, 36, 3, 1, 1), {"in_halo": 1, "act": None, "f32_out": True}, {"ODT_TC_TAPN": "0"}),
    "head_im2col_ragged": ((4, 100, 100, 256, 189, 3, 1, 1), {"act": None, "f32_out": True}, {}),
    # residual + two pre-activated outputs, two N tiles
    "residual_out1_out2": ((8, 75, 75, 128, 256, 3, 1, 1), {"residual": True, "pre": True, "pre2": True}, {}),
    # thin Cin with K-step skipping (1 of 4 and 1 of 4 / 3 of 4 steps issued)
    "kskip_flat": ((8, 64, 64, 16, 28, 3, 1, 1), {"in_halo": 1, "out_halo": 1},
                   {"ODT_TC_TAPN": "0"}),
    "kskip_im2col": ((16, 40, 40, 100, 64, 3, 1, 1), {}, {}),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_conv_tc_pingpong_schedule(built, monkeypatch, case):
    shape, kw, env = CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    a = _conv_case(*shape, mode="tc", seed=sum(shape), **kw)
    assert a.kernel.startswith("conv_tc_kernel<"), a.kernel
    b = _conv_case(*shape, mode="tc", seed=sum(shape), **kw)
    np.testing.assert_array_equal(a.got, b.got)
    if a.got1 is not None:
        np.testing.assert_array_equal(a.got1, b.got1)
