"""conv_tc_kernel's fp16 output path: the epilogue on the accumulator fragments and TMA stores of staged 32-column
chunks, in every mode it covers -- im2col (every N tile, the wide tile included), halo-flat with an output halo, and
the row-block pooled mode with RP = 2 and RP = 4 -- against the float64 bound; ragged M, ragged Cout and ragged
column / row blocks, which the output tensor map clips.  Guard bands: the output sits inside a larger sentinel-filled
buffer, and no byte before or after it, no halo position and no channel past Cout_pad may change.  The layers the path
does not cover (residual + two extra outputs, the fp32 head scatter, an im2col output with a halo) still pass."""
import ctypes as C

import numpy as np
import pytest
import torch

from gpu_harness import SENT as SENTINEL
from gpu_harness import Guarded, mask
from test_gpu_conv import _conv_case

pytestmark = pytest.mark.gpu


# B, H, W, Cin, Cout, k, stride, ODT_TC_WIDE
IM2COL = [
    (2, 19, 19, 128, 64, 3, 1, "0"),     # BN 64
    (3, 17, 23, 64, 96, 3, 1, "0"),      # BN 96, ragged M
    (2, 38, 38, 128, 128, 3, 1, "0"),    # BN 128
    (1, 5, 5, 128, 32, 3, 1, "0"),       # BN 32, one partial tile
    (4, 38, 38, 128, 256, 3, 1, "2"),    # wide tile
    (3, 19, 19, 256, 512, 3, 2, "2"),    # wide tile, stride 2, ragged M
    (3, 21, 21, 64, 56, 1, 1, "0"),      # ragged Cout inside the last chunk
    (2, 26, 26, 128, 112, 3, 1, "0"),
    (2, 19, 19, 128, 200, 3, 1, "0"),    # ragged Cout, two N tiles
    (2, 38, 38, 256, 500, 3, 1, "2"),    # wide tile, ragged Cout
]


@pytest.mark.parametrize("shape", IM2COL)
def test_tma_store_im2col(built, monkeypatch, shape):
    *geom, wide = shape
    monkeypatch.setenv("ODT_TC_WIDE", wide)
    a = _conv_case(*geom, 1, mode="tc", seed=sum(geom))   # also checks the pad channels
    assert a.kernel.endswith(",true>"), a.kernel
    b = _conv_case(*geom, 1, mode="tc", seed=sum(geom))
    np.testing.assert_array_equal(a.got, b.got)


@pytest.mark.parametrize("shape", [(1, 150, 150, 64, 128), (3, 37, 37, 64, 64), (2, 20, 23, 192, 96), (1, 16, 16, 64, 28)])
def test_tma_store_halo_flat(built, monkeypatch, shape):
    monkeypatch.setenv("ODT_TC_TAPN", "0")
    monkeypatch.setenv("ODT_TC_SWAP", "0")   # the transposed tiles would take the larger halo layers
    B, H, W, Cin, Cout = shape
    a = _conv_case(B, H, W, Cin, Cout, 3, 1, 1, mode="tc", in_halo=1, out_halo=1, seed=sum(shape))
    assert a.kernel.endswith(",true>"), a.kernel   # _conv_case checks the zero border


@pytest.mark.parametrize("shape", [(2, 300, 300, 64, 64), (2, 150, 150, 128, 128), (2, 38, 38, 64, 96),
                                   (1, 16, 130, 64, 28), (2, 6, 4, 64, 64)])
@pytest.mark.parametrize("out_halo", [0, 1])
def test_tma_store_pooled(built, monkeypatch, shape, out_halo):
    monkeypatch.setenv("ODT_TC_TAPN", "0")
    monkeypatch.setenv("ODT_TC_SWAP", "0")   # the transposed tiles would take the larger halo layers
    B, H, W, Cin, Cout = shape
    a = _conv_case(B, H, W, Cin, Cout, 3, 1, 1, mode="tc", in_halo=1, out_halo=out_halo, pool=2, seed=sum(shape))
    assert a.kernel.endswith(",true>"), a.kernel


def _guarded(B, H, W, Cin, Cout, k, stride, in_halo, out_halo, pool, ld_extra=0, guard=4096):
    """Run one layer into an output placed inside a sentinel-filled buffer; returns (whole buffer, offset, shape, ld,
    Cout_pad) and the same layer written into a zeroed tight tensor."""
    from odt_b200 import lib as L
    from odt_b200.engine import same_pad
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(B * H * W + Cout)
    ld = (Cin + 63) // 64 * 64
    old = (Cout + 63) // 64 * 64 + ld_extra
    cpad = (Cout + 31) // 32 * 32
    x = torch.zeros((B, H + 2 * in_halo, W + 2 * in_halo, ld), dtype=torch.float16, device="cuda")
    x[:, in_halo:in_halo + H, in_halo:in_halo + W, :Cin] = torch.randn((B, H, W, Cin), generator=g, device="cuda").half()
    w = torch.zeros((cpad, k, k, ld), dtype=torch.float16, device="cuda")
    w[:Cout, :, :, :Cin] = (torch.randn((Cout, k, k, Cin), generator=g, device="cuda") * (2.0 / (k * k * Cin)) ** 0.5).half()
    shift = torch.randn(Cout, generator=g, device="cuda") * 0.2
    OH, pt, _ = same_pad(H, k, stride)
    OW, pl, _ = same_pad(W, k, stride)
    yh, yw = (OH // 2, OW // 2) if pool else (OH, OW)
    oh = out_halo
    shape = (B, yh + 2 * oh, yw + 2 * oh, old)
    n = int(np.prod(shape))
    outs = []
    for fill in (SENTINEL, 0.0):
        init = torch.full(shape, fill, dtype=torch.float16, device="cuda")
        if oh:  # the halo of a halo tensor is zero by contract
            init[mask(shape, 1)] = 0
        y = Guarded(shape, torch.float16, guard=guard, fill=init)
        p = L.ConvParams()
        p.B, p.H, p.W, p.Cin, p.in_ld = B, H, W, Cin, ld
        p.OH, p.OW, p.Cout = OH, OW, Cout
        p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = k, k, stride, 1, pt, pl
        p.w_ld, p.Cout_pad = ld, cpad
        p.shift, p.act = shift.data_ptr(), 2
        p.out0, p.out0_dtype = y.ptr(), L.ODT_F16
        p.out0_img_stride, p.out0_pix_stride = shape[1] * shape[2] * old, old
        p.in_halo, p.out0_halo, p.out0_pool = in_halo, oh, pool
        L.check(lib.odt_conv2d_f16_tc(x.data_ptr(), w.data_ptr(), C.byref(p), torch.cuda.current_stream().cuda_stream),
                "conv")
        torch.cuda.synchronize()
        y.assert_outside_untouched()
        outs.append(y.buf)
    return outs, guard, n, shape, cpad


@pytest.mark.parametrize("case", [
    # B, H, W, Cin, Cout, k, stride, in_halo, out_halo, pool, extra channels in the row, ODT_TC_WIDE
    (3, 17, 23, 64, 96, 3, 1, 0, 0, 0, 0, "0"),       # im2col, ragged M
    (2, 19, 19, 128, 200, 3, 1, 0, 0, 0, 64, "0"),    # im2col, ragged Cout, channels past Cout_pad in the row
    (2, 19, 19, 256, 500, 3, 1, 0, 0, 0, 0, "2"),     # wide tile, ragged M and Cout
    (2, 37, 37, 64, 56, 3, 1, 1, 1, 0, 0, "0"),       # halo-flat
    (2, 300, 300, 64, 64, 3, 1, 1, 1, 2, 0, "0"),     # pooled RP = 2, ragged column block
    (2, 38, 38, 64, 112, 3, 1, 1, 0, 2, 0, "0"),      # pooled, ragged column and row blocks
    (2, 150, 150, 128, 128, 3, 1, 1, 0, 2, 0, "0"),   # pooled RP = 4
])
def test_tma_store_guard_bands(built, monkeypatch, case):
    *geom, wide = case
    monkeypatch.setenv("ODT_TC_WIDE", wide)
    monkeypatch.setenv("ODT_TC_TAPN", "0")
    monkeypatch.setenv("ODT_TC_SWAP", "0")   # the transposed tiles would take the larger halo layers
    (sent, zero), guard, n, shape, cpad = _guarded(*geom)
    B, H, W, Cin, Cout, k, stride, in_halo, oh, pool, extra = geom
    assert bool((sent[:guard] == SENTINEL).all()) and bool((sent[guard + n:] == SENTINEL).all()), "guard band written"
    ys, yz = sent[guard:guard + n].view(shape), zero[guard:guard + n].view(shape)
    inner = (slice(None), slice(oh, shape[1] - oh), slice(oh, shape[2] - oh))
    assert torch.equal(ys[inner][..., :Cout], yz[inner][..., :Cout]), "a store missed the interior"
    assert float(ys[inner][..., :Cout].float().abs().max()) > 0
    assert bool((ys[inner][..., Cout:cpad] == 0).all()), "pad lanes up to Cout_pad are zeros"
    assert bool((ys[..., cpad:] == SENTINEL).all()), "channels past Cout_pad written"
    if oh:
        for border in (ys[:, 0], ys[:, -1], ys[:, :, 0], ys[:, :, -1]):
            assert bool((border == 0).all()), "halo written"


@pytest.mark.parametrize("shape,kw", [
    ((4, 38, 38, 256, 512, 3, 1, 1), {"residual": True, "pre": True, "pre2": True}),   # residual + out1 + out2
    ((2, 38, 38, 256, 189, 3, 1, 1), {"act": None, "f32_out": True}),                  # fp32 head scatter
    ((2, 26, 26, 128, 64, 1, 1, 1), {"in_halo": 1, "out_halo": 1}),                    # im2col output with a halo
])
def test_staged_path_layers(built, shape, kw):
    a = _conv_case(*shape, mode="tc", seed=sum(shape), **kw)
    assert a.kernel.endswith(",false>"), a.kernel
