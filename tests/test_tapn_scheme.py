"""Index arithmetic of the "taps as N" convolution (csrc/conv_tapn.cu), restated in numpy and checked against
a direct 3x3 SAME convolution: tile = 4 rows x 32 columns (30 outputs per row), one [128 x Cin] activation tile
per filter row, N = (tap s, channel n), out[p] = P[p-1, s=0] + P[p, s=1] + P[p+1, s=2]; optional 2x2/2 max-pool
pairing (odd lane, next lane) x (even row, next row).  CPU only: the CUDA kernel itself is opt-in until it has
run on an H100."""
import numpy as np
import pytest

XV, ROWS = 30, 4


def tapn_conv(x, w, pool):
    """x [B,H,W,C] float64, w [N,3,3,C] -> [B,H,W,N] (or pooled [B,H/2,W/2,N]) following the kernel's tiling."""
    B, H, W, C = x.shape
    N = w.shape[0]
    xp = np.zeros((B, H + 2 + ROWS + 2, W + 2 + 34, C))            # halo tensor + room for the TMA zero fill
    xp[:, 1:H + 1, 1:W + 1] = x
    out = np.full((B, H // 2, W // 2, N) if pool else (B, H, W, N), np.nan)
    wn = np.concatenate([w[:, :, s, :] for s in range(3)], 0)      # rows s*N + n, [3N, r, C]
    for b in range(B):
        for yq in range(-(-H // ROWS)):
            for xq in range(-(-W // XV)):
                P = np.zeros((ROWS * 32, 3 * N))
                for r in range(3):                                  # one activation tile per filter row
                    a = xp[b, ROWS * yq + r:ROWS * yq + r + ROWS, XV * xq:XV * xq + 32].reshape(ROWS * 32, C)
                    P += a @ wn[:, r, :].T
                P = P.reshape(ROWS, 32, 3, N)
                v = np.full((ROWS, 32, N), np.nan)
                v[:, 1:31] = P[:, 0:30, 0] + P[:, 1:31, 1] + P[:, 2:32, 2]   # shfl_up / own / shfl_down
                for row in range(ROWS):
                    for lx in range(1, XV + 1):
                        y, xx = ROWS * yq + row, XV * xq - 1 + lx
                        if y >= H or xx >= W:
                            continue
                        if not pool:
                            out[b, y, xx] = v[row, lx]
                        elif (lx & 1) and not (row & 1):            # top-left pixel of a window
                            out[b, y >> 1, xx >> 1] = np.maximum(np.maximum(v[row, lx], v[row, lx + 1]),
                                                                 np.maximum(v[row + 1, lx], v[row + 1, lx + 1]))
    return out


def direct_conv(x, w):
    B, H, W, C = x.shape
    xp = np.zeros((B, H + 2, W + 2, C))
    xp[:, 1:-1, 1:-1] = x
    out = np.zeros((B, H, W, w.shape[0]))
    for r in range(3):
        for s in range(3):
            out += xp[:, r:r + H, s:s + W] @ w[:, r, s, :].T
    return out


@pytest.mark.parametrize("H,W,pool", [(8, 30, False), (7, 41, False), (12, 60, True), (10, 34, True), (4, 300, True)])
def test_taps_as_n_tiling_equals_direct_convolution(H, W, pool):
    rng = np.random.default_rng(H * 1000 + W)
    x = rng.standard_normal((2, H, W, 5))
    w = rng.standard_normal((6, 3, 3, 5))
    got = tapn_conv(x, w, pool)
    ref = direct_conv(x, w)
    if pool:
        ref = ref.reshape(2, H // 2, 2, W // 2, 2, 6).max(axis=(2, 4))
    assert not np.isnan(got).any()                                  # every output is written exactly by some tile
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-10)
