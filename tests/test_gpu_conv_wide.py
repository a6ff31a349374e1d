"""conv_tc_kernel's wide tile (BN = 256, im2col mode): both consumer warpgroups share one 128 x 256 tile, one m64n256k16
accumulator set each, and one parameter block of 256 columns.  Cases at its edges -- Cout 256 / 512 / 1024, a ragged
last M tile, one, two, three and a ragged number of tiles per CTA, dilation 2, stride 2, 1x1, a thin last channel
chunk (K-step skipping), ragged Cout, residual + out1 + out2, the generic and the head-scatter output paths -- against
the fp32 reference at the tolerances of test_gpu_conv.py, two launches bit-identical, and bit-identical to the
128-wide ping-pong tile (each output element sees the same K order).  The plan: which layers take the wide tile."""
import numpy as np
import pytest

from test_gpu_conv import _conv_case

# id: (B, H, W, Cin, Cout, k, stride, dil), _conv_case keywords, environment
CASES = {
    # grid = min(tiles, 132): tiles per CTA = ceil(tiles / 132)
    "cout256_one_tile_per_cta": ((8, 38, 38, 128, 256, 3, 1, 1), {}, {}),                        # 91 tiles
    "cout256_two_tiles_per_cta": ((33, 32, 32, 64, 256, 3, 1, 1), {}, {}),                       # 264 tiles
    "cout256_three_tiles_per_cta": ((48, 33, 32, 64, 256, 3, 1, 1), {}, {}),                     # 396 tiles
    "cout256_ragged_tiles_per_cta": ((5, 75, 75, 64, 256, 3, 1, 1), {"act": "leaky"}, {}),       # 220, last ragged
    "cout512_ragged_m": ((16, 38, 38, 256, 512, 3, 1, 1), {}, {}),                               # 181 x 2 tiles
    "cout1024_dil2_conv6": ((4, 19, 19, 512, 1024, 3, 1, 2), {}, {}),                            # 12 x 4 tiles
    "cout1024_1x1_conv7": ((8, 19, 19, 1024, 1024, 1, 1, 1), {}, {}),                            # 23 x 4 tiles
    "cout512_stride2_conv8_2": ((16, 19, 19, 256, 512, 3, 2, 1), {}, {}),                        # 13 x 2 tiles
    "halo_in_out": ((4, 38, 38, 256, 512, 3, 1, 1), {"in_halo": 1, "out_halo": 1}, {}),
    # thin last 64-channel chunk: 3 of 4 and 1 of 4 K steps issued
    "kskip_cin100": ((8, 38, 38, 100, 256, 3, 1, 1), {}, {}),
    "kskip_cin16": ((8, 38, 38, 16, 512, 3, 1, 1), {}, {}),
    # Cout 500 padded to 512: the last 32-column slice is partly padding, the lanes of its upper half hold none
    "ragged_cout": ((8, 38, 38, 128, 500, 3, 1, 1), {}, {}),
    # RetinaNet's pattern: residual added, two consumer pre-activations stored
    "residual_out1_out2": ((8, 38, 38, 256, 512, 3, 1, 1), {"residual": True, "pre": True, "pre2": True}, {}),
    # fp32 outputs: the head scatter (column-wise slice reads) and the generic element path
    "head_f32": ((4, 38, 38, 256, 256, 3, 1, 1), {"act": None, "f32_out": True}, {}),
    "generic_f32_residual": ((4, 38, 38, 256, 256, 3, 1, 1), {"f32_out": True, "residual": True}, {}),
}


def _run(monkeypatch, case, wide):
    shape, kw, env = CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("ODT_TC_WIDE", wide)
    return _conv_case(*shape, mode="tc", seed=sum(shape), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_conv_tc_wide_tile(built, monkeypatch, case):
    a, ref, a1, r1 = _run(monkeypatch, case, "2")
    tol = 2e-3 * max(np.abs(ref).max(), 1.0)
    assert np.abs(a - ref).max() <= tol, (case, float(np.abs(a - ref).max()), tol)
    if a1 is not None:
        assert np.abs(a1 - r1).max() <= 3 * tol, case
    b, _, b1, _ = _run(monkeypatch, case, "2")
    np.testing.assert_array_equal(a, b)
    if a1 is not None:
        np.testing.assert_array_equal(a1, b1)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cout512_ragged_m", "cout1024_1x1_conv7", "kskip_cin100", "residual_out1_out2",
                                  "head_f32"])
def test_conv_tc_wide_matches_narrow(built, monkeypatch, case):
    """The wide tile only regroups who computes which columns: every output element is the same sum in the same
    K order as on the 128-wide tile."""
    a, _, a1, _ = _run(monkeypatch, case, "2")
    b, _, b1, _ = _run(monkeypatch, case, "0")
    np.testing.assert_array_equal(a, b)
    if a1 is not None:
        np.testing.assert_array_equal(a1, b1)


@pytest.mark.gpu
def test_conv_tc_wide_needs_cout_pad_multiple_of_256(built, monkeypatch):
    """Cout_pad 384 cannot take the wide tile even where it is forced; the layer still runs correctly."""
    from odt_b200 import lib as L
    monkeypatch.setenv("ODT_TC_WIDE", "2")
    assert L.load().odt_conv_tc_pick_bn(384, 16 * 38 * 38, 36) <= 128
    a, ref, _, _ = _conv_case(16, 38, 38, 256, 384, 3, 1, 1, mode="tc", seed=1)
    assert np.abs(a - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0)


# SSD300 at B = 64: (layer, output size, Cin, Cout, k) of the im2col-mode layers whose Cout_pad is a multiple of 256
SSD300_B64 = [("conv3_1", 75, 128, 256, 3), ("conv3_2", 75, 256, 256, 3), ("conv3_3", 75, 256, 256, 3),
              ("conv4_1", 38, 256, 512, 3), ("conv4_2", 38, 512, 512, 3), ("conv4_3", 38, 512, 512, 3), ("conv5_1", 19, 512, 512, 3),
              ("conv5_2", 19, 512, 512, 3), ("conv5_3", 19, 512, 512, 3), ("conv6", 19, 512, 1024, 3),
              ("conv7", 19, 1024, 1024, 1)]


def test_conv_tc_wide_plan_ssd300_b64(built, monkeypatch):
    """The wide VGG layers of the headline workload take the 128 x 256 tile from the cost model alone, and the
    switch turns it off."""
    from odt_b200 import lib as L
    lib = L.load()
    monkeypatch.delenv("ODT_TC_WIDE", raising=False)
    for name, hw, cin, cout, k in SSD300_B64:
        assert lib.odt_conv_tc_pick_bn(cout, 64 * hw * hw, k * k * cin // 64) == 256, name
    monkeypatch.setenv("ODT_TC_WIDE", "0")
    for name, hw, cin, cout, k in SSD300_B64:
        assert lib.odt_conv_tc_pick_bn(cout, 64 * hw * hw, k * k * cin // 64) <= 128, name


def test_conv_tc_wide_plan_small_m(built, monkeypatch):
    """Small-M layers keep narrow tiles spread over the SMs where one wide tile per CTA would leave most of them idle:
    the SSD extras at B = 1 and RetinaNet's P6 / P7 heads at B = 16 (Cout 256, 3x3)."""
    from odt_b200 import lib as L
    lib = L.load()
    monkeypatch.delenv("ODT_TC_WIDE", raising=False)
    assert lib.odt_conv_tc_pick_bn(512, 1 * 10 * 10, 36) <= 128     # conv8_2, B = 1
    assert lib.odt_conv_tc_pick_bn(256, 16 * 13 * 13, 36) <= 128    # P6 tower, B = 16
    assert lib.odt_conv_tc_pick_bn(256, 16 * 7 * 7, 36) <= 128      # P7 tower, B = 16
