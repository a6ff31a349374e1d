"""Index arithmetic of the thin-layer CUDA-core convolution (csrc/conv_thin.cu) restated in numpy: one output
pixel per "thread", taps addressed as iy = oy*stride - pad_t + r inside a tensor stored with or without a one-pixel
zero halo, anything outside the stored extent read as zero.  Checked against the oracle's TF-SAME convolution.
CPU only; the CUDA kernel itself is checked on the GPU (tests/test_gpu_conv.py)."""
import numpy as np
import pytest

from oracle import tfops as T


def thin_conv(x, w_hwio, stride, in_halo):
    B, H, W, Cin = x.shape
    ks, Cout = w_hwio.shape[0], w_hwio.shape[3]
    OH, pad_t, _ = T.same_pad(H, ks, stride)
    OW, pad_l, _ = T.same_pad(W, ks, stride)
    ih = in_halo
    stored = np.zeros((B, H + 2 * ih, W + 2 * ih, Cin), np.float64)
    stored[:, ih:ih + H, ih:ih + W] = x
    out = np.zeros((B, OH, OW, Cout), np.float64)
    oy, ox = np.meshgrid(np.arange(OH), np.arange(OW), indexing="ij")
    for r in range(ks):
        for s in range(ks):
            iy = oy * stride - pad_t + r
            ix = ox * stride - pad_l + s
            inside = (iy >= -ih) & (iy < H + ih) & (ix >= -ih) & (ix < W + ih)
            v = stored[:, np.clip(iy + ih, 0, H + 2 * ih - 1), np.clip(ix + ih, 0, W + 2 * ih - 1)]
            v = np.where(inside[None, :, :, None], v, 0.0)
            out += v @ w_hwio[r, s]
    return out


@pytest.mark.parametrize("H,W,ks,stride,halo", [(9, 11, 3, 1, 1), (9, 11, 3, 1, 0), (10, 12, 3, 2, 1), (11, 13, 3, 2, 0),
                                                (10, 10, 3, 2, 0), (7, 5, 1, 1, 1), (8, 6, 1, 2, 0)])
def test_thin_conv_indexing_equals_same_convolution(H, W, ks, stride, halo):
    rng = np.random.default_rng(H * 100 + W * 10 + ks + stride)
    x = rng.standard_normal((2, H, W, 7)).astype(np.float32)
    w = rng.standard_normal((ks, ks, 7, 5)).astype(np.float32)
    ref = T.conv2d_same(x, w, None, stride)
    np.testing.assert_allclose(thin_conv(x.astype(np.float64), w.astype(np.float64), stride, halo), ref, rtol=1e-4,
                               atol=1e-4)
