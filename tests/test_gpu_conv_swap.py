"""The transposed tensor-core tiles of csrc/conv_tc_swap.cu (64 output channels x 256 pixels per wgmma, pixels on the N
side) behind odt_conv2d_f16_tc: halo-flat layers and the row-block pooled mode with RP = 8 / 4 / 2, Cout_pad = 64
(resident and streamed filter bank) and 128 (two channel halves per pixel tile), against the float64 bound AND bit for
bit against the pixel-major path (ODT_TC_SWAP=0): same products, same K order.  Ragged tiles, one-row-pair images,
B = 1, ragged Cout; guard bands around the output; SSD300's three layers at full size."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_gpu_conv import _conv_case, _tc_raw
from test_gpu_conv_tma_store import SENTINEL, _guarded

pytestmark = pytest.mark.gpu


def _both(monkeypatch, *geom, **kw):
    """The layer on the transposed tiles (ODT_TC_SWAP=2) and on the pixel-major path (=0); the other opt-in paths off."""
    monkeypatch.setenv("ODT_TC_TAPN", "0")
    monkeypatch.setenv("ODT_TC_SWAP", "2")
    a = _conv_case(*geom, 3, 1, 1, mode="tc", in_halo=1, seed=sum(geom), **kw)
    assert a.kernel == "conv_tc_swap_kernel", a.kernel
    monkeypatch.setenv("ODT_TC_SWAP", "0")
    b = _conv_case(*geom, 3, 1, 1, mode="tc", in_halo=1, seed=sum(geom), **kw)
    assert b.kernel.startswith("conv_tc_kernel<"), b.kernel
    return a.got, b.got


def _plan(B, H, W, Cin, Cout, pool, out_halo=1, ld_extra=0):
    """odt_conv_tc_swap_plan of a 3x3 / stride-1 halo layer -> (taken, RP, tiles, waste per thousand)."""
    from odt_b200 import lib as L
    ld, cpad = (Cin + 63) // 64 * 64, (Cout + 31) // 32 * 32
    old = (Cout + 63) // 64 * 64 + ld_extra
    yh, yw = (H // 2, W // 2) if pool else (H, W)
    p = L.ConvParams()
    p.B, p.H, p.W, p.Cin, p.in_ld, p.OH, p.OW, p.Cout = B, H, W, Cin, ld, H, W, Cout
    p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l, p.w_ld, p.Cout_pad = 3, 3, 1, 1, 1, 1, ld, cpad
    p.out0, p.out0_dtype, p.out0_pix_stride = 4096, L.ODT_F16, old
    p.out0_img_stride = (yh + 2 * out_halo) * (yw + 2 * out_halo) * old
    p.in_halo, p.out0_halo, p.out0_pool = 1, out_halo, pool
    rp, tiles, waste = C.c_int(-1), C.c_longlong(-1), C.c_int(-1)
    taken = L.load().odt_conv_tc_swap_plan(C.byref(p), C.byref(rp), C.byref(tiles), C.byref(waste))
    return taken, rp.value, tiles.value, waste.value


# B, H, W, Cin, Cout
FLAT = [
    (1, 16, 16, 64, 64),      # B = 1, two tiles, the second ragged
    (2, 37, 41, 64, 128),     # odd sizes, two channel halves
    (3, 21, 23, 128, 64),     # Cin = 128: streamed filter bank
    (2, 20, 23, 192, 128),
    (1, 1, 300, 64, 64),      # one-row image
    (2, 33, 5, 64, 56),       # rows shorter than a register octet, ragged Cout
    (1, 150, 150, 64, 128),   # SSD300 conv2_1, one image
    (2, 30, 30, 64, 100),     # ragged Cout in the second half
]


@pytest.mark.parametrize("shape", FLAT)
@pytest.mark.parametrize("act", ["relu", "leaky", None])
def test_swap_halo_flat(built, monkeypatch, shape, act):
    if act != "relu" and shape[1] > 40:
        pytest.skip("every activation on the small shapes")
    a, b = _both(monkeypatch, *shape, out_halo=1, act=act)   # _conv_case checks the zero border and pad lanes
    np.testing.assert_array_equal(a, b)


POOLED = [
    (1, 8, 32, 64, 64),       # RP 8: exactly one tile
    (2, 150, 150, 128, 128),  # RP 8, ragged row and column blocks, two channel halves (SSD300 conv2_2)
    (1, 300, 300, 64, 64),    # RP 4 (SSD300 conv1_2), ragged column block
    (2, 4, 64, 64, 64),       # RP 4: exactly one tile per image
    (2, 2, 300, 64, 128),     # RP 2: one row pair, ragged column block
    (3, 38, 38, 64, 96 + 4),  # ragged Cout, ragged blocks
    (2, 6, 4, 128, 64),       # tiny map, streamed filter bank
    (1, 16, 130, 64, 120),
]


@pytest.mark.parametrize("shape", POOLED)
@pytest.mark.parametrize("out_halo", [0, 1])
def test_swap_pooled(built, monkeypatch, shape, out_halo):
    B, H, W, Cin, Cout = shape
    act = ["relu", "leaky", None][(H + out_halo) % 3]
    a, b = _both(monkeypatch, *shape, out_halo=out_halo, pool=2, act=act)
    np.testing.assert_array_equal(a, b)


def test_swap_rowblock_plan(built, monkeypatch):
    monkeypatch.setenv("ODT_TC_SWAP", "2")
    assert _plan(1, 8, 32, 64, 64, 2)[:3] == (1, 8, 1)
    assert _plan(1, 300, 300, 64, 64, 2)[:3] == (1, 4, 375)
    assert _plan(2, 150, 150, 128, 128, 2)[:3] == (1, 8, 190)
    assert _plan(2, 2, 300, 64, 128, 2)[:3] == (1, 2, 6)
    assert _plan(1, 16, 16, 64, 64, 0)[:3] == (1, 0, 2)


@pytest.mark.parametrize("case", [
    # B, H, W, Cin, Cout, k, stride, in_halo, out_halo, pool, extra channels in the row
    (2, 37, 37, 64, 56, 3, 1, 1, 1, 0, 0),        # halo-flat, ragged Cout
    (2, 23, 31, 64, 128, 3, 1, 1, 1, 0, 64),      # halo-flat, channels past Cout_pad in the row
    (2, 300, 300, 64, 64, 3, 1, 1, 1, 2, 0),      # pooled RP 4, ragged column block
    (2, 38, 38, 64, 112, 3, 1, 1, 0, 2, 0),       # pooled, ragged column and row blocks
    (2, 150, 150, 128, 128, 3, 1, 1, 0, 2, 64),   # pooled RP 8
    (2, 2, 260, 64, 64, 3, 1, 1, 1, 2, 0),        # pooled RP 2
])
def test_swap_guard_bands(built, monkeypatch, case):
    monkeypatch.setenv("ODT_TC_TAPN", "0")
    monkeypatch.setenv("ODT_TC_SWAP", "2")
    (sent, zero), guard, n, shape, cpad = _guarded(*case)
    B, H, W, Cin, Cout, k, stride, in_halo, oh, pool, extra = case
    assert _plan(B, H, W, Cin, Cout, pool, oh, extra)[0] == 1, "the layer did not take the transposed tiles"
    assert bool((sent[:guard] == SENTINEL).all()) and bool((sent[guard + n:] == SENTINEL).all()), "guard band written"
    ys, yz = sent[guard:guard + n].view(shape), zero[guard:guard + n].view(shape)
    inner = (slice(None), slice(oh, shape[1] - oh), slice(oh, shape[2] - oh))
    assert torch.equal(ys[inner][..., :Cout], yz[inner][..., :Cout]), "a store missed the interior"
    assert float(ys[inner][..., :Cout].float().abs().max()) > 0
    assert bool((ys[inner][..., Cout:cpad] == 0).all()), "pad lanes up to Cout_pad are zeros"
    assert bool((ys[inner][..., cpad:] == SENTINEL).all()), "channels past Cout_pad written"
    if oh:  # (_guarded zeroes the border rows and columns whole)
        for border in (ys[:, 0], ys[:, -1], ys[:, :, 0], ys[:, :, -1]):
            assert bool((border == 0).all()), "halo written"
    monkeypatch.setenv("ODT_TC_SWAP", "0")
    (sent0, _), _, _, _, _ = _guarded(*case)
    assert torch.equal(sent0, sent), "differs from the pixel-major path"


@pytest.mark.parametrize("name,geom,pool", [
    ("conv1_2", (300, 300, 64, 64), 2),
    ("conv2_1", (150, 150, 64, 128), 0),
    ("conv2_2", (150, 150, 128, 128), 2),
])
def test_swap_ssd300_layers_full_size(built, monkeypatch, name, geom, pool):
    """SSD300's three narrow layers at the benchmark batch (64): taken by the planner, equal bit for bit to the
    pixel-major path; the same layer at B = 2 against the float64 bound."""
    monkeypatch.delenv("ODT_TC_SWAP", raising=False)
    monkeypatch.setenv("ODT_TC_TAPN", "0")
    H, W, Cin, Cout = geom
    assert _plan(64, H, W, Cin, Cout, pool)[0] == 1, name
    g = torch.Generator(device="cuda").manual_seed(11)
    x = (torch.randn((64, H, W, Cin), generator=g, device="cuda") * 0.5).half()
    w = (torch.randn((Cout, 3, 3, Cin), generator=g, device="cuda") * (2.0 / (9 * Cin)) ** 0.5).half()
    y = _tc_raw(x, w, pool=pool)
    assert float(y.float().abs().max()) > 0.1
    monkeypatch.setenv("ODT_TC_SWAP", "0")
    assert torch.equal(_tc_raw(x, w, pool=pool), y), name
    del x, y
    a, b = _both(monkeypatch, 2, H, W, Cin, Cout, out_halo=1, pool=pool)
    np.testing.assert_array_equal(a, b)
