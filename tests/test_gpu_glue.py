"""The glue kernels of glue.cu (pools, channel L2-norm, affine + activation, FPN up-sampling, nearest concat, input
normalisation / packing, GroupNorm) on every dispatch path, at their edges and in situ at the models' full sizes.

Exactness is stated per check and holds by construction:
  * bit-exact: max-pooling (a maximum of stored values is a stored value), nearest concat (a copy), input
    normalisation (one correctly rounded fp32 subtraction, rounded once to the output type), the legacy bilinear
    up-sampling + add (the kernel and the restatement below execute the same correctly rounded fp32 operations one
    for one, no FMA; in fp16 the fp32 result is rounded once);
  * at most one ulp of the output type: affine + activation (the kernel's fmaf is x*s+h rounded once; the float64
    x*s+h rounded to fp32 can differ from it by double rounding only);
  * l2norm and GroupNorm: forward-error bounds derived next to their checks.
Every output is written inside a sentinel-filled buffer: nothing outside the tensor, no channel in [C, ld), no halo
position and no NULL output may change.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_harness import Guarded
from gpu_harness import interior as _interior
from gpu_harness import mask as _mask
from gpu_harness import model as _model

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24   # unit roundoff of fp32
U16 = 2.0 ** -11   # unit roundoff of fp16
GN_EPS = 1e-6
DTYPES = {"f16": torch.float16, "f32": torch.float32}


@pytest.fixture(scope="module")
def lib(built):
    from odt_b200 import lib as L
    return L.load()


def _code(dt):
    from odt_b200 import lib as L
    return L.ODT_F16 if dt == torch.float16 else L.ODT_F32


def _st():
    return torch.cuda.current_stream().cuda_stream


def _check(rc, what=""):
    from odt_b200 import lib as L
    L.check(rc, what)


def _ulps(got, ref):
    """Distance in units in the last place of the (common) floating type: ordered-integer difference."""
    assert got.dtype == ref.dtype
    if got.dtype == torch.float16:
        a, b = got.view(torch.int16).int(), ref.view(torch.int16).int()
        a, b = torch.where(a < 0, -32768 - a, a), torch.where(b < 0, -32768 - b, b)
    else:
        a, b = got.view(torch.int32).long(), ref.view(torch.int32).long()
        a, b = torch.where(a < 0, -2 ** 31 - a, a), torch.where(b < 0, -2 ** 31 - b, b)
    return (a - b).abs()


# ---- restatements on the device (torch), checked against oracle/tfops.py in test_restatements_match_oracle ----------
def ref_maxpool(x, k, s):
    """TF SAME max-pool of NHWC x (exact in any dtype)."""
    from odt_b200.engine import same_pad
    _, pt, pb = same_pad(x.shape[1], k, s)
    _, pl, pr = same_pad(x.shape[2], k, s)
    t = F.pad(x.permute(0, 3, 1, 2).double(), (pl, pr, pt, pb), value=float("-inf"))
    return F.max_pool2d(t, k, s).permute(0, 2, 3, 1).to(x.dtype)


def ref_affine(x, s, h, act, dt):
    """act(x*s + h): float64 product and sum rounded once to fp32, the activation in fp32, rounded to dt."""
    z = (x.double() * s.double() + h.double()).float()
    if act == 1:
        z = torch.clamp_min(z, 0.0)
    elif act == 2:
        z = torch.maximum(z, torch.tensor(0.1, dtype=torch.float32, device=z.device) * z)
    return z.to(dt)


def ref_l2norm(x, gamma):
    """x * rsqrt(max(sum_c x^2, 1e-12)) * gamma in float64, and the kernel's sum of squares in exact arithmetic."""
    x = x.double()
    ss = (x * x).sum(-1, keepdim=True)
    return x * torch.rsqrt(torch.clamp_min(ss, 1e-12)) * gamma, ss


def ref_bilinear(top, H, W):
    """TF1 legacy resize_bilinear in fp32, one correctly rounded operation at a time (as the kernel)."""
    f32 = torch.float32
    t = top.float()
    TH, TW = t.shape[1], t.shape[2]
    hs = torch.tensor(TH, dtype=f32) / torch.tensor(H, dtype=f32)
    ws = torch.tensor(TW, dtype=f32) / torch.tensor(W, dtype=f32)
    ys = torch.arange(H, dtype=f32) * hs
    xs = torch.arange(W, dtype=f32) * ws
    y0, x0 = torch.floor(ys).long(), torch.floor(xs).long()
    y1, x1 = torch.clamp_max(torch.ceil(ys).long(), TH - 1), torch.clamp_max(torch.ceil(xs).long(), TW - 1)
    ly = (ys - y0.to(f32)).to(t.device).view(1, H, 1, 1)
    lx = (xs - x0.to(f32)).to(t.device).view(1, 1, W, 1)
    y0, y1, x0, x1 = (v.to(t.device) for v in (y0, y1, x0, x1))
    tl, tr = t[:, y0][:, :, x0], t[:, y0][:, :, x1]
    bl, br = t[:, y1][:, :, x0], t[:, y1][:, :, x1]
    top_ = tl + (tr - tl) * lx
    bot = bl + (br - bl) * lx
    return top_ + (bot - top_) * ly


def ref_nearest(b, H, W):
    f32 = torch.float32
    BH, BW = b.shape[1], b.shape[2]
    hs = torch.tensor(BH, dtype=f32) / torch.tensor(H, dtype=f32)
    ws = torch.tensor(BW, dtype=f32) / torch.tensor(W, dtype=f32)
    yi = torch.clamp_max(torch.floor(torch.arange(H, dtype=f32) * hs).long(), BH - 1).to(b.device)
    xi = torch.clamp_max(torch.floor(torch.arange(W, dtype=f32) * ws).long(), BW - 1).to(b.device)
    return b[:, yi][:, :, xi]


def ref_groupnorm(x, gamma, beta, groups, act, eps=GN_EPS):
    """GroupNorm of the stored x [B,H,W,C]: float64 two-pass moments, then TF's formula
    (gain = rstd*gamma; off = -mean*gain + beta) in float64.  Returns (y, mean, rstd, sigma) per element."""
    B, H, W, Cc = x.shape
    xg = x.double().reshape(B, H * W, groups, Cc // groups)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(var + float(np.float32(eps)))
    g = gamma.double().view(1, 1, groups, Cc // groups)
    bt = beta.double().view(1, 1, groups, Cc // groups)
    gain = rstd * g
    y = xg * gain + (-mean * gain + bt)
    if act == 1:
        y = torch.clamp_min(y, 0.0)
    elif act == 2:
        y = torch.maximum(y, 0.1 * y)
    shp = (B, H, W, Cc)
    ex = lambda t: t.expand(B, H * W, groups, Cc // groups).reshape(shp)  # noqa: E731
    return y.reshape(shp), ex(mean), ex(rstd), ex(torch.sqrt(var))


def gn_bound(x, gamma, beta, mean, rstd, sigma, dt, k):
    """Per-element forward-error bound of the kernels' GroupNorm against ref_groupnorm.

    The kernels evaluate gain = fl(rstd*gamma), off = fl(fl(-mean*gain) + beta), y = fl(fl(x*gain) + off) in fp32 from
    their fp32 (mean, rstd): at most 6 fp32 roundings of terms bounded by |x*gain| + |mean*gain| + |beta| (the last
    one of |y| itself), plus the rounding to fp16 (U16*|y|, and half the smallest fp16 subnormal).  The statistics
    carry a relative error eps = (k + 16) * U32, where k is the number of terms a thread sums in fp32 (the fp32 partial
    sums of the deviations dominate; 16 covers the rounding of the deviations, the fp32 reduction tree of the
    fallback, the fp64 merges and the final rounding to fp32): it moves y by at most eps * (|x - mean| + sigma) *
    |gamma| * rstd (rstd's error scales x - mean, the mean's error is at most eps * sigma)."""
    Cc = x.shape[-1]
    g = gamma.double().view(1, 1, 1, Cc)
    bt = beta.double().view(1, 1, 1, Cc)
    xd = x.double()
    gain = rstd * g
    s = (xd * gain).abs() + (mean * gain).abs() + bt.abs()
    eps = (k + 16) * U32
    tol = 6 * U32 * s + eps * ((xd - mean).abs() + sigma) * g.abs() * rstd
    if dt == torch.float16:
        # |fl16(y') - y| <= |y' - y| (1 + U16) + U16 |y| for the kernel's fp32 result y' (half an ulp; the fp16
        # rounding of a value just above a power of two reaches it: measured up to 0.99 of this bound in FCOS)
        y = (xd - mean) * gain + bt
        tol = tol * (1 + U16) + U16 * y.abs() + 2.0 ** -25
    return tol


def gn_terms_fused(dt, Cc, groups):
    V = 8 if dt == torch.float16 else 4
    return 8 * min(V, Cc // groups)  # 8 vectors per thread per slice


def gn_terms_fallback(hw, Cc, groups):
    return -(-hw * (Cc // groups) // 1024)  # 1024 threads per (group, image)


def test_restatements_match_oracle(built):
    """The device restatements used below (and in the in-situ checks) against oracle/tfops.py on the CPU."""
    from oracle import tfops as T
    rng = np.random.default_rng(0)
    for (h, w, k, s) in [(9, 11, 2, 2), (10, 7, 3, 2), (8, 8, 3, 1)]:
        x = rng.standard_normal((2, h, w, 5)).astype(np.float32)
        np.testing.assert_array_equal(ref_maxpool(torch.from_numpy(x), k, s).numpy(), T.max_pool_same(x, k, s))
    for (th, tw, hh, ww) in [(13, 7, 25, 13), (4, 4, 8, 8), (25, 25, 50, 50), (5, 3, 7, 11)]:
        t = rng.standard_normal((2, th, tw, 3)).astype(np.float32)
        np.testing.assert_array_equal(ref_bilinear(torch.from_numpy(t), hh, ww).numpy(),
                                      T.resize_bilinear_legacy(t, hh, ww))
        np.testing.assert_array_equal(ref_nearest(torch.from_numpy(t), hh, ww).numpy(),
                                      T.resize_nearest_legacy(t, hh, ww))
    x = rng.standard_normal((2, 5, 6, 32)).astype(np.float32)
    y, _ = ref_l2norm(torch.from_numpy(x), 20.0)
    np.testing.assert_allclose(y.numpy(), 20.0 * T.l2_normalize_channels(x), rtol=1e-6, atol=0)
    g, b = rng.uniform(.5, 1.5, 32).astype(np.float32), rng.standard_normal(32).astype(np.float32)
    y = ref_groupnorm(torch.from_numpy(x), torch.from_numpy(g), torch.from_numpy(b), 8, 0)[0]
    np.testing.assert_allclose(y.numpy(), T.group_norm(x, g, b), rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# a. dispatch matrix at small shapes
# ---------------------------------------------------------------------------------------------------------------------
def _rnd(shape, dt, seed, scale=1.0, shift=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale + shift).to(dt)


# (B, H, W, C, ld, k, stride): odd sizes, pad_t != pad_b, ld > C; off = 1 forces the scalar path
POOLS = [(2, 75, 75, 64, 64, 2, 2), (2, 19, 21, 64, 72, 3, 1), (2, 20, 17, 32, 40, 3, 2), (1, 10, 10, 16, 64, 2, 2),
         (3, 7, 9, 24, 24, 3, 2), (1, 5, 6, 12, 12, 2, 2)]


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("shape", POOLS)
@pytest.mark.parametrize("halo", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("off", [0, 1])
def test_maxpool_dispatch(lib, dtype, shape, halo, off):
    """odt_maxpool: maxpool_h8 (fp16, 2/2 and 3/1, C % 8 == 0), the vectorised and the scalar generic kernel; exact,
    nothing written outside [C) of the interior."""
    from odt_b200.engine import same_pad
    dt = DTYPES[dtype]
    B, H, W, Cc, ld, k, s = shape
    ih, oh = halo
    OH, OW = same_pad(H, k, s)[0], same_pad(W, k, s)[0]
    x = torch.zeros((B, H + 2 * ih, W + 2 * ih, ld), dtype=dt, device="cuda")
    _interior(x, ih)[..., :Cc] = _rnd((B, H, W, Cc), dt, B * H + Cc)
    xg = Guarded(x.shape, dt, off=off, fill=x)
    y = Guarded((B, OH + 2 * oh, OW + 2 * oh, ld), dt, off=off)
    _check(lib.odt_maxpool(xg.ptr(), y.ptr(), _code(dt), B, H, W, Cc, ld, k, s, ih, oh, _st()))
    torch.cuda.synchronize()
    ref = ref_maxpool(_interior(x, ih)[..., :Cc], k, s)
    assert torch.equal(_interior(y.t, oh)[..., :Cc], ref)
    y.assert_outside_untouched()
    y.assert_untouched(_mask(y.t.shape, oh, Cc), "halo / channel >= C")
    xg.assert_outside_untouched()


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("shape", [(2, 20, 22, 16, 64, 3, 2), (2, 9, 7, 8, 8, 3, 2), (1, 11, 13, 12, 12, 2, 2),
                                   (2, 16, 16, 64, 64, 3, 2)])
@pytest.mark.parametrize("outs", ["all", "raw+1", "1", "2", "1+2"])
@pytest.mark.parametrize("variant", [(0, 0, 0, 0, 1, 2), (1, 1, 1, 0, 0, 1), (0, 1, 0, 1, 2, 0)])
@pytest.mark.parametrize("off", [0, 1])
def test_maxpool_affine_dispatch(lib, dtype, shape, outs, variant, off):
    """odt_maxpool_affine: raw out / out1 / out2 each optional, halos on every tensor, NULL scale / shift (identity),
    act in {0, 1, 2}; the scalar path through a misaligned base pointer.  Raw output exact, affine outputs within one
    ulp of the output type."""
    from odt_b200.engine import same_pad
    dt = DTYPES[dtype]
    B, H, W, Cc, ld, k, s = shape
    ih, oh, h1, h2, act1, act2 = variant
    null_params = variant[3] == 1
    OH, OW = same_pad(H, k, s)[0], same_pad(W, k, s)[0]
    x = torch.zeros((B, H + 2 * ih, W + 2 * ih, ld), dtype=dt, device="cuda")
    _interior(x, ih)[..., :Cc] = _rnd((B, H, W, Cc), dt, 7 + Cc)
    xg = Guarded(x.shape, dt, off=off, fill=x)
    raw = Guarded((B, OH + 2 * oh, OW + 2 * oh, ld), dt, off=off)
    o1 = Guarded((B, OH + 2 * h1, OW + 2 * h1, ld), dt, off=off)
    o2 = Guarded((B, OH + 2 * h2, OW + 2 * h2, ld), dt, off=off)
    gen = torch.Generator(device="cuda").manual_seed(11)
    s1 = torch.rand(ld, generator=gen, device="cuda") + 0.5
    t1 = torch.randn(ld, generator=gen, device="cuda")
    s2 = torch.rand(ld, generator=gen, device="cuda") - 0.5
    t2 = torch.randn(ld, generator=gen, device="cuda")
    want_raw = outs in ("all", "raw+1")
    want1 = outs in ("all", "raw+1", "1", "1+2")
    want2 = outs in ("all", "2", "1+2")
    p = lambda t: None if null_params else t.data_ptr()  # noqa: E731
    _check(lib.odt_maxpool_affine(
        xg.ptr(), raw.ptr() if want_raw else None, _code(dt), B, H, W, Cc, ld, k, s, ih, oh,
        p(s1), p(t1), act1, o1.ptr() if want1 else None, h1, p(s2), p(t2), act2, o2.ptr() if want2 else None, h2,
        _st()))
    torch.cuda.synchronize()
    pooled = ref_maxpool(_interior(x, ih)[..., :Cc], k, s)
    one, zero = torch.ones(Cc, device="cuda"), torch.zeros(Cc, device="cuda")
    for g, want, halo, sc, sh, act in ((raw, want_raw, oh, None, None, None), (o1, want1, h1, s1, t1, act1),
                                       (o2, want2, h2, s2, t2, act2)):
        g.assert_outside_untouched()
        if not want:
            g.assert_untouched(torch.ones(g.t.shape, dtype=torch.bool, device="cuda"), "NULL output")
            continue
        g.assert_untouched(_mask(g.t.shape, halo, Cc), "halo / channel >= C")
        got = _interior(g.t, halo)[..., :Cc]
        if act is None:
            assert torch.equal(got, pooled)
        else:
            sc_, sh_ = (one, zero) if null_params else (sc[:Cc], sh[:Cc])
            ref = ref_affine(pooled, sc_, sh_, act, dt)
            assert int(_ulps(got, ref).max()) <= 1


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("shape", [(98, 64, 64), (37, 24, 40), (50, 7, 7), (33, 512, 512), (5, 3, 8)])
@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("off", [0, 1])
def test_affine_act_dispatch(lib, dtype, shape, act, off):
    """odt_affine_act (vectorised / scalar, ld > C, NULL scale or shift): within one ulp of the output type."""
    dt = DTYPES[dtype]
    P, Cc, ld = shape
    x = _rnd((P, ld), dt, P + Cc, scale=3.0)
    xg = Guarded(x.shape, dt, off=off, fill=x)
    y = Guarded(x.shape, dt, off=off)
    gen = torch.Generator(device="cuda").manual_seed(P)
    sc = torch.randn(ld, generator=gen, device="cuda")
    sh = torch.randn(ld, generator=gen, device="cuda")
    for use_sc, use_sh in ((True, True), (False, True), (True, False)):
        _check(lib.odt_affine_act(xg.ptr(), y.ptr(), _code(dt), P, Cc, ld, sc.data_ptr() if use_sc else None,
                                  sh.data_ptr() if use_sh else None, act, _st()))
        torch.cuda.synchronize()
        ref = ref_affine(x[:, :Cc], sc[:Cc] if use_sc else torch.ones(Cc, device="cuda"),
                         sh[:Cc] if use_sh else torch.zeros(Cc, device="cuda"), act, dt)
        assert int(_ulps(y.t[:, :Cc], ref).max()) <= 1, (use_sc, use_sh)
        y.assert_outside_untouched()
        y.assert_untouched(_mask(y.t.shape, 0, Cc), "channel >= C")


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("shape", [(162, 512, 512), (40, 30, 33), (64, 1024, 1024), (7, 5, 8)])
@pytest.mark.parametrize("off", [0, 1])
def test_l2norm_dispatch(lib, dtype, shape, off):
    """odt_l2norm_scale.  Bound: each lane sums ceil(C/32) squares with fmaf, then a 5-level shuffle tree: the sum of
    squares has a relative error of at most (C/32 + 6) * U32 (all terms >= 0); the correctly rounded rsqrt adds half
    of that plus U32, the two products 2 U32; fp16 adds its rounding U16.  An all-zero pixel gives zeros (the
    max(., 1e-12) clamp keeps rsqrt finite) and tiny pixels hit the clamp."""
    dt = DTYPES[dtype]
    P, Cc, ld = shape
    x = _rnd((P, ld), dt, P * 3 + Cc)
    x[0] = 0                     # all-zero pixel
    x[1, :Cc] = 0
    x[1, 0] = 1e-7 if dt == torch.float32 else 2.0 ** -20  # sum of squares < 1e-12: the clamp applies
    xg = Guarded(x.shape, dt, off=off, fill=x)
    y = Guarded(x.shape, dt, off=off)
    _check(lib.odt_l2norm_scale(xg.ptr(), y.ptr(), _code(dt), P, Cc, ld, 20.0, _st()))
    torch.cuda.synchronize()
    ref, ss = ref_l2norm(x[:, :Cc], 20.0)
    got = y.t[:, :Cc]
    assert torch.isfinite(got).all()
    assert torch.equal(got[0], torch.zeros_like(got[0]))
    assert float(ss[1]) < 1e-12
    eps = (1.5 * (-(-Cc // 32) + 6) + 3) * U32 + (U16 if dt == torch.float16 else 0.0)
    floor = 2.0 ** -24 if dt == torch.float16 else 0.0
    err = (got.double() - ref).abs()
    assert bool((err <= eps * ref.abs() + floor).all()), float((err - eps * ref.abs()).max())
    y.assert_outside_untouched()
    y.assert_untouched(_mask(y.t.shape, 0, Cc), "channel >= C")


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("geom", [(2, 13, 13, 25, 25, 64), (2, 4, 4, 8, 8, 64), (1, 25, 25, 50, 50, 256),
                                  (2, 5, 7, 9, 13, 24), (1, 7, 5, 14, 10, 12)])
@pytest.mark.parametrize("with_out1", [None, 0, 1, 2])
@pytest.mark.parametrize("off", [0, 1])
def test_upsample_bilinear_add_dispatch(lib, dtype, geom, with_out1, off):
    """odt_upsample_bilinear_add: out bit-exact against the fp32 restatement (rounded once in fp16); the consumer
    pre-activation out1 = act(stored out * s + h) within one ulp; NULL scale2 / shift2 when act is 0."""
    dt = DTYPES[dtype]
    B, TH, TW, H, W, Cc = geom
    top = _rnd((B, TH, TW, Cc), dt, 3 + Cc)
    a = _rnd((B, H, W, Cc), dt, 5 + Cc)
    tg, ag = Guarded(top.shape, dt, off=off, fill=top), Guarded(a.shape, dt, off=off, fill=a)
    y, y1 = Guarded(a.shape, dt, off=off), Guarded(a.shape, dt, off=off)
    gen = torch.Generator(device="cuda").manual_seed(Cc)
    s2, h2 = torch.randn(Cc, generator=gen, device="cuda"), torch.randn(Cc, generator=gen, device="cuda")
    null = with_out1 == 0
    _check(lib.odt_upsample_bilinear_add(
        tg.ptr(), ag.ptr(), y.ptr(), _code(dt), B, TH, TW, H, W, Cc, Cc,
        None if (with_out1 is None or null) else s2.data_ptr(), None if (with_out1 is None or null) else h2.data_ptr(),
        with_out1 or 0, y1.ptr() if with_out1 is not None else None, _st()))
    torch.cuda.synchronize()
    ref = (a.float() + ref_bilinear(top, H, W)).to(dt)
    assert torch.equal(y.t, ref)
    y.assert_outside_untouched()
    y1.assert_outside_untouched()
    if with_out1 is None:
        y1.assert_untouched(torch.ones(a.shape, dtype=torch.bool, device="cuda"), "NULL out1")
    else:
        sc = torch.ones(Cc, device="cuda") if null else s2
        sh = torch.zeros(Cc, device="cuda") if null else h2
        assert int(_ulps(y1.t, ref_affine(ref, sc, sh, with_out1, dt)).max()) <= 1


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("geom", [(2, 26, 26, 64, 64, 13, 13, 32, 32, 128), (2, 52, 52, 128, 128, 26, 26, 256, 256, 384),
                                  (1, 9, 7, 24, 32, 5, 4, 16, 24, 48), (2, 6, 6, 3, 5, 3, 3, 5, 7, 9)])
@pytest.mark.parametrize("off", [0, 1])
def test_upsample_nearest_concat_dispatch(lib, dtype, geom, off):
    """odt_upsample_nearest_concat: a copy, exact; channels [Ca + Cb, ldo) untouched."""
    dt = DTYPES[dtype]
    B, H, W, Ca, lda, BH, BW, Cb, ldb, ldo = geom
    a, b = _rnd((B, H, W, lda), dt, 1 + Ca), _rnd((B, BH, BW, ldb), dt, 2 + Cb)
    agd, bgd = Guarded(a.shape, dt, off=off, fill=a), Guarded(b.shape, dt, off=off, fill=b)
    y = Guarded((B, H, W, ldo), dt, off=off)
    _check(lib.odt_upsample_nearest_concat(agd.ptr(), bgd.ptr(), y.ptr(), _code(dt), B, H, W, Ca, lda, BH, BW, Cb, ldb,
                                           ldo, _st()))
    torch.cuda.synchronize()
    assert torch.equal(y.t[..., :Ca], a[..., :Ca])
    assert torch.equal(y.t[..., Ca:Ca + Cb], ref_nearest(b[..., :Cb], H, W))
    y.assert_outside_untouched()
    y.assert_untouched(_mask(y.t.shape, 0, Ca + Cb), "channel >= Ca + Cb")


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("geom", [(2, 9, 11, 8), (1, 300, 300, 64), (3, 5, 7, 3)])
def test_normalize_input(lib, dtype, geom):
    """odt_normalize_input: fp32 image - mean (one correctly rounded subtraction) rounded once; channels >= 3 zero."""
    dt = DTYPES[dtype]
    B, H, W, ld = geom
    img = torch.randint(0, 256, (B, H, W, 3), device="cuda").float()
    mean = (C.c_float * 3)(123.68, 116.779, 103.979)
    m = torch.tensor(list(mean), dtype=torch.float32, device="cuda")
    y = Guarded((B, H, W, ld), dt)
    _check(lib.odt_normalize_input(img.data_ptr(), y.ptr(), _code(dt), B, H, W, ld, mean, _st()))
    torch.cuda.synchronize()
    assert torch.equal(y.t[..., :3], (img - m).to(dt))
    assert bool((y.t[..., 3:] == 0).all())
    y.assert_outside_untouched()


@pytest.mark.parametrize("geom", [(2, 16, 20, 4), (1, 13, 9, 1), (2, 8, 12, 3), (1, 33, 47, 0)])
@pytest.mark.parametrize("img_off", [0, 1])
def test_pack_input_rgbx(lib, geom, img_off):
    """odt_pack_input_rgbx: (image - mean) in fp16 RGBX, X = 0; the border of `pad` pixels is never written.  W % 4
    and the image's alignment pick the 4-pixel or the 1-pixel kernel; odd pads take the 8-byte stores."""
    B, H, W, pad = geom
    img = Guarded((B, H, W, 3), torch.float32, off=img_off,
                  fill=torch.randint(0, 256, (B, H, W, 3), device="cuda").float())
    mean = (C.c_float * 3)(123.68, 116.779, 103.979)
    m = torch.tensor(list(mean), dtype=torch.float32, device="cuda")
    out = Guarded((B, H + 2 * pad, W + 2 * pad, 4), torch.float16)
    _check(lib.odt_pack_input_rgbx(img.ptr(), out.ptr(), B, H, W, pad, mean, _st()))
    torch.cuda.synchronize()
    inner = out.t[:, pad:pad + H, pad:pad + W]
    assert torch.equal(inner[..., :3], (img.t - m).half())
    assert bool((inner[..., 3] == 0).all())
    border = torch.ones(out.t.shape, dtype=torch.bool, device="cuda")
    border[:, pad:pad + H, pad:pad + W] = False
    out.assert_untouched(border, "border")
    out.assert_outside_untouched()


# ---------------------------------------------------------------------------------------------------------------------
# b. GroupNorm at its edges
# ---------------------------------------------------------------------------------------------------------------------
def _gn_fused(lib, x, ld, Cc, groups, gamma, beta, act, out=None):
    B, H, W = x.shape[:3]
    dt = x.dtype
    nbytes = lib.odt_groupnorm_act_workspace_bytes(_code(dt), B, H * W, Cc, groups)
    assert nbytes > 0
    ws = torch.zeros((nbytes + 7) // 8, dtype=torch.float64, device="cuda")
    y = out if out is not None else Guarded(x.shape, dt)
    rc = lib.odt_groupnorm_act(x.data_ptr(), y.ptr(), ws.data_ptr(), _code(dt), B, H * W, Cc, ld, groups, GN_EPS,
                               gamma.data_ptr(), beta.data_ptr(), act, _st())
    _check(rc, "groupnorm_act")
    torch.cuda.synchronize()
    return y, ws


def _gn_fallback(lib, x, ld, Cc, groups, gamma, beta, act):
    B, H, W = x.shape[:3]
    dt = x.dtype
    stats = torch.zeros(B * groups * 2, dtype=torch.float32, device="cuda")
    y = Guarded(x.shape, dt)
    _check(lib.odt_groupnorm_stats(x.data_ptr(), stats.data_ptr(), _code(dt), B, H * W, Cc, ld, groups, GN_EPS, _st()))
    _check(lib.odt_groupnorm_apply(x.data_ptr(), y.ptr(), stats.data_ptr(), _code(dt), B, H * W, Cc, ld, groups,
                                   gamma.data_ptr(), beta.data_ptr(), act, _st()))
    torch.cuda.synchronize()
    return y


def _gn_input(B, H, W, Cc, ld, dt, ratio, seed):
    """x = m + N(0, 1) per (image, group), m = ratio (alternating sign across images), stored in dt."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.zeros((B, H, W, ld), dtype=dt, device="cuda")
    sign = torch.tensor([1.0 if b % 2 == 0 else -1.0 for b in range(B)], device="cuda").view(B, 1, 1, 1)
    x[..., :Cc] = (torch.randn((B, H, W, Cc), generator=g, device="cuda") + ratio * sign).to(dt)
    gamma = torch.rand(Cc, generator=g, device="cuda") + 0.5
    beta = torch.randn(Cc, generator=g, device="cuda")
    return x, gamma, beta


def _gn_assert(y, x, Cc, groups, gamma, beta, act, k, what):
    ref, mean, rstd, sigma = ref_groupnorm(x[..., :Cc], gamma, beta, groups, act)
    tol = gn_bound(x[..., :Cc], gamma, beta, mean, rstd, sigma, x.dtype, k)
    err = (y.t[..., :Cc].double() - ref).abs()
    assert torch.isfinite(y.t[..., :Cc]).all(), what
    worst = float((err / tol).max())
    assert worst <= 1.0, "%s: error reaches %.3g x the bound (max err %.3g)" % (what, worst, float(err.max()))
    y.assert_outside_untouched()
    y.assert_untouched(_mask(y.t.shape, 0, Cc), "channel >= C")
    return worst


# (B, H, W, C, ld, groups): cpg < V (16 channels stored 64 wide, 8 groups; 64 channels, 32 / 64 groups), = V, > V;
# hw = 1, hw below one slice (256 * 8 vectors), hw not a multiple of the slice
GN_SHAPES = [(3, 17, 19, 16, 64, 8), (1, 1, 1, 64, 64, 8), (4, 5, 7, 64, 64, 32), (2, 9, 9, 64, 64, 64),
             (4, 33, 31, 256, 256, 8), (1, 40, 40, 256, 256, 32), (16, 3, 5, 512, 512, 8), (3, 64, 64, 256, 256, 8),
             (1, 23, 29, 512, 512, 64), (2, 1, 3, 32, 32, 8)]


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("shape", GN_SHAPES)
@pytest.mark.parametrize("act", [0, 1, 2])
def test_groupnorm_shapes(lib, dtype, shape, act):
    """odt_groupnorm_act and odt_groupnorm_stats + apply against float64 two-pass moments (gn_bound)."""
    dt = DTYPES[dtype]
    B, H, W, Cc, ld, groups = shape
    x, gamma, beta = _gn_input(B, H, W, Cc, ld, dt, 0.5, B * H * W + Cc + groups)
    y, _ = _gn_fused(lib, x, ld, Cc, groups, gamma, beta, act)
    _gn_assert(y, x, Cc, groups, gamma, beta, act, gn_terms_fused(dt, Cc, groups), "fused")
    y2 = _gn_fallback(lib, x, ld, Cc, groups, gamma, beta, act)
    _gn_assert(y2, x, Cc, groups, gamma, beta, act, gn_terms_fallback(H * W, Cc, groups), "stats + apply")


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("ratio", [0, 10, 100, 1000])
@pytest.mark.parametrize("shape", [(4, 64, 64, 256, 256, 8), (2, 33, 47, 64, 64, 32)])
def test_groupnorm_large_mean(lib, dtype, ratio, shape):
    """|mean| / sigma up to 1000: the statistics are two-pass, so the variance does not cancel.  (A one-pass
    E[x^2] - mean^2 from fp32 partial sums misses the fp32 bound by orders of magnitude at 100.)"""
    dt = DTYPES[dtype]
    B, H, W, Cc, ld, groups = shape
    x, gamma, beta = _gn_input(B, H, W, Cc, ld, dt, float(ratio), 17 + ratio)
    y, _ = _gn_fused(lib, x, ld, Cc, groups, gamma, beta, 0)
    w1 = _gn_assert(y, x, Cc, groups, gamma, beta, 0, gn_terms_fused(dt, Cc, groups), "fused")
    y2 = _gn_fallback(lib, x, ld, Cc, groups, gamma, beta, 0)
    w2 = _gn_assert(y2, x, Cc, groups, gamma, beta, 0, gn_terms_fallback(H * W, Cc, groups), "stats + apply")
    print("%s |mean|/sigma=%d %s: worst error / bound: fused %.3f, stats + apply %.3f" % (dtype, ratio, shape, w1, w2))


@pytest.mark.parametrize("dtype", ["f16", "f32"])
def test_groupnorm_constant_group(lib, dtype):
    """A constant group: variance 0, rstd = 1/sqrt(eps), the output is beta (up to the rounding of the formula)."""
    dt = DTYPES[dtype]
    x, gamma, beta = _gn_input(2, 20, 20, 64, 64, dt, 0.0, 5)
    x[0, ..., :8] = 0.3   # group 0 of image 0
    x[1, ..., 8:16] = -2.0
    for y in (_gn_fused(lib, x, 64, 64, 8, gamma, beta, 0)[0], _gn_fallback(lib, x, 64, 64, 8, gamma, beta, 0)):
        _gn_assert(y, x, 64, 8, gamma, beta, 0, gn_terms_fallback(400, 64, 8), "constant group")
        ref = beta[:8].to(dt).double()
        assert float((y.t[0, ..., :8].double() - ref).abs().max()) <= 1e-3


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("shape", [(96, 3, 4, 64, 64, 64), (768, 1, 2, 8, 8, 8)])
def test_groupnorm_at_shared_memory_limit(lib, dtype, shape):
    """B * groups = 6144: the apply kernel's shared-memory copy of the statistics is exactly 48 KiB; one more image
    is outside the two-launch path (workspace query 0, ODT_ERR_UNSUPPORTED)."""
    from odt_b200 import lib as L
    dt = DTYPES[dtype]
    B, H, W, Cc, ld, groups = shape
    x, gamma, beta = _gn_input(B, H, W, Cc, ld, dt, 1.0, 3)
    y, _ = _gn_fused(lib, x, ld, Cc, groups, gamma, beta, 1)
    _gn_assert(y, x, Cc, groups, gamma, beta, 1, gn_terms_fused(dt, Cc, groups), "48 KiB")
    assert lib.odt_groupnorm_act_workspace_bytes(_code(dt), B + 1, H * W, Cc, groups) == 0
    x2 = torch.zeros((B + 1, H, W, ld), dtype=dt, device="cuda")
    ws = torch.zeros(1024, dtype=torch.float64, device="cuda")
    out = Guarded(x2.shape, dt)
    rc = lib.odt_groupnorm_act(x2.data_ptr(), out.ptr(), ws.data_ptr(), _code(dt), B + 1, H * W, Cc, ld, groups,
                               GN_EPS, gamma.data_ptr(), beta.data_ptr(), 1, _st())
    torch.cuda.synchronize()
    assert rc == L.ERR_UNSUPPORTED
    out.assert_untouched(torch.ones(x2.shape, dtype=torch.bool, device="cuda"), "output of a refused launch")


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("case", ["C=96", "groups=128", "misaligned"])
def test_groupnorm_act_unsupported(lib, dtype, case):
    """Shapes outside the two-launch path return ODT_ERR_UNSUPPORTED and leave the output untouched."""
    from odt_b200 import lib as L
    dt = DTYPES[dtype]
    Cc, groups, off = {"C=96": (96, 8, 0), "groups=128": (256, 128, 0), "misaligned": (64, 8, 1)}[case]
    x = Guarded((2, 6, 6, Cc), dt, off=off, fill=_rnd((2, 6, 6, Cc), dt, 1))
    out = Guarded((2, 6, 6, Cc), dt, off=off)
    ws = torch.zeros(1 << 16, dtype=torch.float64, device="cuda")
    g = torch.ones(Cc, device="cuda")
    rc = lib.odt_groupnorm_act(x.ptr(), out.ptr(), ws.data_ptr(), _code(dt), 2, 36, Cc, Cc, groups, GN_EPS,
                               g.data_ptr(), g.data_ptr(), 0, _st())
    torch.cuda.synchronize()
    assert rc == L.ERR_UNSUPPORTED
    out.assert_untouched(torch.ones(out.t.shape, dtype=torch.bool, device="cuda"), "output of a refused launch")
    out.assert_outside_untouched()
    if case != "misaligned":
        assert lib.odt_groupnorm_act_workspace_bytes(_code(dt), 2, 36, Cc, groups) == 0


@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("shape", [(4, 64, 64, 256, 256, 8), (4, 33, 35, 16, 64, 8), (4, 128, 128, 64, 64, 32)])
def test_groupnorm_batch_invariant_and_reproducible(lib, dtype, shape):
    """Bit for bit: image b alone equals its slice of a batch of 4 (the slice partition depends on hw and C only), two
    launches give the same output (fixed-order reductions, no float atomics), on both paths; fused and fallback agree
    within the sum of their bounds."""
    dt = DTYPES[dtype]
    B, H, W, Cc, ld, groups = shape
    x, gamma, beta = _gn_input(B, H, W, Cc, ld, dt, 3.0, 99)
    y, ws = _gn_fused(lib, x, ld, Cc, groups, gamma, beta, 1)
    first = y.t.clone()
    _gn_fused(lib, x, ld, Cc, groups, gamma, beta, 1, out=y)   # fresh workspace
    assert torch.equal(y.t, first), "two launches differ"
    # the same workspace again without re-zeroing: the kernel left its arrival counters at zero
    lib.odt_groupnorm_act(x.data_ptr(), y.ptr(), ws.data_ptr(), _code(dt), B, H * W, Cc, ld, groups, GN_EPS,
                          gamma.data_ptr(), beta.data_ptr(), 1, _st())
    torch.cuda.synchronize()
    assert torch.equal(y.t, first), "a reused workspace changes the output"
    for b in (0, 3):
        xb = x[b:b + 1].clone()
        yb, _ = _gn_fused(lib, xb, ld, Cc, groups, gamma, beta, 1)
        assert torch.equal(yb.t, first[b:b + 1]), "image %d alone differs from its slice of the batch" % b
    f1 = _gn_fallback(lib, x, ld, Cc, groups, gamma, beta, 1).t.clone()
    assert torch.equal(_gn_fallback(lib, x, ld, Cc, groups, gamma, beta, 1).t, f1)
    assert torch.equal(_gn_fallback(lib, x[1:2].clone(), ld, Cc, groups, gamma, beta, 1).t, f1[1:2])
    ref, mean, rstd, sigma = ref_groupnorm(x[..., :Cc], gamma, beta, groups, 1)
    tol = (gn_bound(x[..., :Cc], gamma, beta, mean, rstd, sigma, dt, gn_terms_fused(dt, Cc, groups))
           + gn_bound(x[..., :Cc], gamma, beta, mean, rstd, sigma, dt, gn_terms_fallback(H * W, Cc, groups)))
    assert bool(((first[..., :Cc].double() - f1[..., :Cc].double()).abs() <= tol).all())


# ---------------------------------------------------------------------------------------------------------------------
# c. in situ at full size
# ---------------------------------------------------------------------------------------------------------------------
def _check_pad_lanes(buf, C, what):
    if buf.shape[-1] > C:
        assert not bool(buf[..., C:].ne(0).any()), "%s: channel >= C written" % what


def _check_halo_zero(buf, halo, what):
    if halo:
        m = _mask(buf.shape, 1)
        assert not bool(buf[m].ne(0).any()), "%s: halo written" % what


def _insitu_pool(net, op):
    x = op.x
    c = min(x.ld, (x.C + 7) // 8 * 8)
    xin = _interior(x.buf, x.halo)[..., :c]
    pooled = ref_maxpool(xin, op.k, op.stride)
    if op.y.needed and op.y.buf is not None:
        assert torch.equal(_interior(op.y.buf, op.y.halo)[..., :c], pooled), "pool raw output"
        _check_pad_lanes(op.y.buf[..., c:], 0, "pool")
        _check_halo_zero(op.y.buf, op.y.halo, "pool")
    for a in op.aff:
        if a is None:
            continue
        sc, sh, act, t = a
        got = _interior(t.buf, t.halo)[..., :c]
        assert int(_ulps(got, ref_affine(pooled, sc[:c], sh[:c], act, got.dtype)).max()) <= 1, "pool affine output"
        _check_pad_lanes(t.buf, c, "pool affine")
        _check_halo_zero(t.buf, t.halo, "pool affine")
    return "exact" + ("" if all(a is None for a in op.aff) else ", fused affine outputs <= 1 ulp")


def _insitu_l2norm(net, op):
    x = op.x
    assert x.halo == 0 and op.y.halo == 0
    xin = x.buf[..., :x.C]
    ref, _ = ref_l2norm(xin, op.gamma)
    got = op.y.buf[..., :x.C]
    eps = (1.5 * (-(-x.C // 32) + 6) + 3) * U32 + (U16 if got.dtype == torch.float16 else 0.0)
    floor = 2.0 ** -24 if got.dtype == torch.float16 else 0.0
    err = (got.double() - ref).abs()
    assert bool((err <= eps * ref.abs() + floor).all()), "l2norm"
    _check_pad_lanes(op.y.buf, x.C, "l2norm")
    return "max err %.3g" % float(err.max())


def _insitu_affine(net, op):
    x, y = op.x, op.y
    assert x.halo == 0 and y.halo == 0
    got = y.buf
    ref = ref_affine(x.buf, op.scale, op.shift, {None: 0, "relu": 1, "leaky": 2}[op.act], got.dtype)
    assert int(_ulps(got, ref).max()) <= 1, "affine_act"
    return "<= 1 ulp"


def _insitu_gn(net, op):
    x, y = op.x, op.y
    assert x.halo == 0 and y.halo == 0
    act = {None: 0, "relu": 1, "leaky": 2}[op.act]
    xin = x.buf[..., :x.C]
    ref, mean, rstd, sigma = ref_groupnorm(xin, op.gamma, op.beta, op.groups, act)
    k = (gn_terms_fused(xin.dtype, x.C, op.groups) if op.two_launch
         else gn_terms_fallback(x.H * x.W, x.C, op.groups))
    tol = gn_bound(xin, op.gamma, op.beta, mean, rstd, sigma, xin.dtype, k)
    err = (y.buf[..., :x.C].double() - ref).abs()
    worst = float((err / tol).max())
    ratio = float((mean.abs() / sigma.clamp_min(1e-30)).max())
    assert worst <= 1.0, "GroupNorm %s: %.3g x the bound" % (op.gn, worst)
    _check_pad_lanes(y.buf, x.C, "GroupNorm")
    return "C=%d hw=%d max|mean|/sigma %.3g, max err %.3g (rel. to max|ref| %.2e), %.3f of the bound" % (
        x.C, x.H * x.W, ratio, float(err.max()), float(err.max()) / max(float(ref.abs().max()), 1e-30), worst)


def _insitu_upsample(net, op):
    t, a, y = op.top, op.a, op.y
    assert t.halo == 0 and a.halo == 0 and y.halo == 0
    ref = (a.buf.float() + ref_bilinear(t.buf, y.H, y.W)).to(y.buf.dtype)
    assert torch.equal(y.buf, ref), "upsample_add"
    if op.pre is not None:
        t1 = op.pre[2]
        assert t1.halo == 0
        sc = op.s2 if op.s2 is not None else torch.ones(y.ld, device="cuda")
        sh = op.h2 if op.h2 is not None else torch.zeros(y.ld, device="cuda")
        act = {None: 0, "relu": 1, "leaky": 2}[op.pre[1]]
        assert int(_ulps(t1.buf, ref_affine(ref, sc, sh, act, y.buf.dtype)).max()) <= 1, "upsample_add out1"
    return "exact" + (" + out1 <= 1 ulp" if op.pre is not None else "")


def _insitu_concat(net, op):
    a, b, y = op.a, op.b, op.y
    assert a.halo == 0 and b.halo == 0 and y.halo == 0
    assert torch.equal(y.buf[..., :a.C], a.buf[..., :a.C])
    assert torch.equal(y.buf[..., a.C:a.C + b.C], ref_nearest(b.buf[..., :b.C], y.H, y.W))
    _check_pad_lanes(y.buf, a.C + b.C, "nearest_concat")
    return "exact"


INSITU = [("ssd300", "fp16", 64, {}), ("retinanet", "fp16", 16, {"data_shape": [800, 800, 3]}),
          ("yolov3", "fp16", 32, {"data_shape": [416, 416, 3]}), ("fcos", "fp16", 4, {"data_shape": [1024, 1024, 3]}),
          ("fcos", "fp32", 4, {"data_shape": [1024, 1024, 3]}), ("ssd512", "fp16", 1, {}),
          ("yolov2", "fp16", 64, {}), ("yolov2", "fp16", 8, {"size": 200}), ("yolov2", "fp32", 2, {})]


@pytest.mark.parametrize("kind,precision,B,over", INSITU, ids=["%s-%s-B%d%s" % (k, p, b, "-%d" % o["size"] if "size" in o
                                                                            else "") for k, p, b, o in INSITU])
def test_glue_ops_in_situ(built, kind, precision, B, over):
    """Every glue op of the network at its full per-GPU geometry, checked on its actual input and output buffers
    after one eager forward (every activation owns its buffer, so all of them are live): the planner's own launch
    arguments (fused pre-activations, halos, pooled channel counts) on real activation statistics."""
    from odt_b200 import engine as E
    m = _model(kind, precision, **over)
    net = m.engine(B, graph=False)
    h, w = net.in_h, net.in_w
    img = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (B, h, w, 3)).astype(np.float32))
    net.image_buf.copy_(img)
    net.forward()
    torch.cuda.synchronize()
    fns = {E.PoolOp: _insitu_pool, E.L2NormOp: _insitu_l2norm, E.AffineActOp: _insitu_affine,
           E.GroupNormActOp: _insitu_gn, E.UpsampleAddOp: _insitu_upsample, E.NearestConcatOp: _insitu_concat}
    seen = {}
    for i, op in enumerate(net.ops):
        fn = fns.get(type(op))
        if fn is None:
            continue
        if any(t.buf is None for t in op.reads):
            continue  # an input the plan dropped
        res = fn(net, op)
        seen[type(op).__name__] = seen.get(type(op).__name__, 0) + 1
        print("%s %s B=%d op %d %s: %s" % (kind, precision, B, i, type(op).__name__, res))
    print("%s %s B=%d glue ops checked: %s" % (kind, precision, B, seen))
    assert seen, "no glue op found"
    if kind == "fcos":
        assert seen.get("GroupNormActOp", 0) > 0
        assert all(op.two_launch for op in net.ops if isinstance(op, E.GroupNormActOp))
    del net, m
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# d. FCOS whole network
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_fcos_replay_and_batch_invariance(built, precision):
    """FCOS 256^2: two replays of the captured graph give bit-identical head rows and packed detection records; one
    image alone equals its slice of a batch of 2 when every layer runs the same kernel at both batch sizes (checked
    on the op plan); otherwise only the GroupNorm outputs are compared in situ."""
    from odt_b200 import engine as E
    m = _model("fcos", precision, data_shape=[256, 256, 3])
    img = np.random.default_rng(2).integers(0, 256, (2, 256, 256, 3)).astype(np.float32)
    net2 = m.engine(2)
    net2.image_buf.copy_(torch.from_numpy(img))
    net2.run()
    torch.cuda.synchronize()
    rows, rec = net2.head_buf.clone(), net2.tail.rec.clone()
    net2.run()
    torch.cuda.synchronize()
    assert torch.equal(net2.head_buf, rows), "graph replay changed the head rows"
    assert torch.equal(net2.tail.rec, rec), "graph replay changed the detection records"
    net1 = m.engine(1)
    net1.image_buf.copy_(torch.from_numpy(img[:1]))
    net1.run()
    torch.cuda.synchronize()

    def plan(net):
        out = []
        for op in net.ops:
            if isinstance(op, E.ConvOp):
                out.append(("conv", op.kernel, op.use_tc, getattr(op, "rgbx", 0), op.pool,
                            op.pre is not None, op.pre2 is not None))
            elif isinstance(op, E.GroupNormActOp):
                out.append(("gn", op.gn, op.two_launch))
            else:
                out.append((type(op).__name__,))
        return out

    same_plan = plan(net1) == plan(net2)
    # the tensor-core convolution's tile choice depends on the GEMM size (and so on B): compare picks per layer
    picks = []
    for o1, o2 in zip(net1.ops, net2.ops):
        if isinstance(o1, E.ConvOp) and o1.use_tc:
            p1, p2 = o1.params(net1), o2.params(net2)
            M1 = p1.B * p1.OH * p1.OW
            kb = p1.R * p1.S * p1.in_ld // 64
            picks.append(net1.lib.odt_conv_tc_pick_bn(p1.Cout_pad, M1, kb) ==
                         net2.lib.odt_conv_tc_pick_bn(p2.Cout_pad, p2.B * p2.OH * p2.OW, kb))
    same_kernels = same_plan and all(picks)
    gn1 = [op for op in net1.ops if isinstance(op, E.GroupNormActOp)]
    gn2 = [op for op in net2.ops if isinstance(op, E.GroupNormActOp)]
    assert gn1 and len(gn1) == len(gn2)
    if same_kernels:
        assert torch.equal(net1.head_buf[0], net2.head_buf[0]), "image 0 alone differs from its slice of the batch"
        print("FCOS %s: same kernels at B=1 and B=2; head rows bit-identical" % precision)
    else:
        print("FCOS %s: the planner picks different kernels at B=1 and B=2 (plan equal: %s, tile picks equal: %d/%d);"
              " comparing the GroupNorm outputs in situ only" % (precision, same_plan, sum(picks), len(picks)))
    # GroupNorm in situ: the same input image gives the same output bits at both batch sizes
    net2.image_buf[1:].copy_(net2.image_buf[:1])
    net2.forward()
    net1.forward()
    torch.cuda.synchronize()
    for a, b in zip(gn1, gn2):
        x1, x2 = a.x.buf[0], b.x.buf[1]
        if same_kernels or torch.equal(x1, x2):
            assert torch.equal(a.y.buf[0], b.y.buf[1]), a.gn
            assert torch.equal(b.y.buf[0], b.y.buf[1]), a.gn
