"""The planner of the transposed tensor-core tiles (odt_conv_tc_swap_plan, csrc/conv_tc_swap.cu), on the host: which
3x3 / stride-1 halo layers of the five detectors it takes at their benchmark batches, the row-block RP it chooses and
the share of computed positions that are no output pixel.  Needs no GPU."""
import ctypes as C

import pytest


def _plan(B, H, W, Cin, Cout, pool=0, out_halo=1, **over):
    from odt_b200 import lib as L
    ld, cpad, old = (Cin + 63) // 64 * 64, (Cout + 31) // 32 * 32, (Cout + 63) // 64 * 64
    yh, yw = (H // 2, W // 2) if pool else (H, W)
    p = L.ConvParams()
    p.B, p.H, p.W, p.Cin, p.in_ld, p.OH, p.OW, p.Cout = B, H, W, Cin, ld, H, W, Cout
    p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l, p.w_ld, p.Cout_pad = 3, 3, 1, 1, 1, 1, ld, cpad
    p.out0, p.out0_dtype, p.out0_pix_stride = 4096, L.ODT_F16, old
    p.out0_img_stride = (yh + 2 * out_halo) * (yw + 2 * out_halo) * old
    p.in_halo, p.out0_halo, p.out0_pool = 1, out_halo, pool
    for k, v in over.items():
        setattr(p, k, v)
    rp, tiles, waste = C.c_int(-1), C.c_longlong(-1), C.c_int(-1)
    taken = L.load().odt_conv_tc_swap_plan(C.byref(p), C.byref(rp), C.byref(tiles), C.byref(waste))
    return (taken, rp.value, tiles.value, waste.value) if taken else (0, None, None, None)


@pytest.mark.parametrize("name,args,rp,tiles_per_img,max_waste", [
    # SSD300, B = 64 (the benchmark's headline workload)
    ("ssd300 conv1_2", (64, 300, 300, 64, 64, 2), 4, 375, 67),
    ("ssd300 conv2_1", (64, 150, 150, 64, 128, 0), 0, None, 30),      # halo-flat: the 2 x 152 + 150 border positions
    ("ssd300 conv2_2", (64, 150, 150, 128, 128, 2), 8, 95, 80),
    # SSD512, B = 16
    ("ssd512 conv1_2", (16, 512, 512, 64, 64, 2), 8, 1024, 0),
    ("ssd512 conv2_1", (16, 256, 256, 64, 128, 0), 0, None, 20),
    ("ssd512 conv2_2", (16, 256, 256, 128, 128, 2), 8, 256, 0),
])
def test_layers_taken(built, monkeypatch, name, args, rp, tiles_per_img, max_waste):
    monkeypatch.delenv("ODT_TC_SWAP", raising=False)
    taken, got_rp, tiles, waste = _plan(*args)
    assert taken == 1 and got_rp == rp, name
    if tiles_per_img is not None:
        assert tiles == args[0] * tiles_per_img, name
    assert 0 <= waste <= max_waste, (name, waste)


@pytest.mark.parametrize("name,args,over", [
    ("ssd300 conv3_1: 256 output channels", (64, 75, 75, 128, 256), {}),
    ("ssd300 conv1_2 at B = 1: too few units per SM", (1, 300, 300, 64, 64, 2), {}),
    ("ssd300 conv10_2-sized map", (64, 5, 5, 128, 128), {}),
    ("retinanet P7 tower-sized map, B = 16", (16, 7, 7, 128, 128), {}),
    ("yolov3 residual block 3x3 (adds its input)", (32, 208, 208, 32, 64), {"residual": 4096}),
    ("retinanet bottleneck 3x3 with a pre-activated second output", (16, 200, 200, 64, 64), {"out1": 4096}),
    ("fp32 head output", (64, 150, 150, 128, 128), {"out0_dtype": 1}),
    ("Cout_pad 96", (64, 150, 150, 64, 96), {}),
    ("stride 2", (64, 150, 150, 64, 64), {"stride": 2}),
    ("no input halo", (64, 150, 150, 64, 64), {"in_halo": 0}),
    ("halo-flat output without a halo", (64, 150, 150, 64, 128, 0, 0), {}),
])
def test_layers_not_taken(built, monkeypatch, name, args, over):
    monkeypatch.delenv("ODT_TC_SWAP", raising=False)
    assert _plan(*args, **over)[0] == 0, name


def test_switch(built, monkeypatch):
    small = (1, 16, 16, 64, 64)
    big = (64, 150, 150, 64, 128)
    monkeypatch.setenv("ODT_TC_SWAP", "0")
    assert _plan(*big)[0] == 0
    monkeypatch.setenv("ODT_TC_SWAP", "1")
    assert _plan(*big)[0] == 1 and _plan(*small)[0] == 0
    monkeypatch.setenv("ODT_TC_SWAP", "2")
    assert _plan(*small)[:3] == (1, 0, 2)
    assert _plan(1, 16, 16, 64, 96)[0] == 0  # never past what the tile computes


def test_rowblock_rp_minimises_tiles(built, monkeypatch):
    monkeypatch.setenv("ODT_TC_SWAP", "2")
    for H, W in [(300, 300), (150, 150), (2, 300), (4, 64), (8, 32), (38, 38), (512, 512), (6, 4), (16, 130)]:
        _, rp, tiles, waste = _plan(1, H, W, 64, 64, 2)
        counts = {r: -(-H // r) * -(-W // (256 // r)) for r in (2, 4, 8)}
        assert tiles == min(counts.values()) and counts[rp] == tiles, (H, W)
        assert rp == max(r for r in counts if counts[r] == tiles), "ties keep the larger RP"
        assert waste == (tiles * 256 - H * W) * 1000 // (tiles * 256)
