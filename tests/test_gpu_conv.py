"""GPU parity, stage (ii): convolution and glue kernels against plain fp32
references (torch / the oracle's TF-op restatements) on the same inputs.
Tolerances: fp16 tensor-core path -- fp16 operands are exact in both, fp32
accumulation, fp16-rounded output => |err| <= 2e-3 * max|ref|; fp32 CUDA-core
path => 2e-5 * max|ref| (accumulation order only)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _conv_case(B, H, W, Cin, Cout, k, stride, dil, mode, act="relu", residual=False, pre=False,
               bn=True, f32_out=False, seed=0, in_halo=0, out_halo=0, pool=0, pre2=False, no_out0=False, aux_halo=0):
    """mode: 'tc' (fp16 wgmma), 'direct16', 'direct32'.  Returns (got, ref, got1, ref1)."""
    from odt_b200 import lib as L
    from odt_b200.engine import same_pad
    from oracle import tfops as T
    lib = L.load()
    rng = np.random.default_rng(seed)
    f16 = mode != "direct32"
    tdt = torch.float16 if f16 else torch.float32
    ld = (Cin + 63) // 64 * 64 if mode == "tc" else Cin
    x = (rng.standard_normal((B, H, W, Cin)) * 1.0).astype(np.float32)
    w = (rng.standard_normal((k, k, Cin, Cout)) * np.sqrt(2.0 / (k * k * Cin))).astype(np.float32)
    if f16:
        x = x.astype(np.float16).astype(np.float32)
        w = w.astype(np.float16).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32) if bn else None
    shift = (rng.standard_normal(Cout) * 0.2).astype(np.float32)
    OH, pt, _ = same_pad(H, k, stride, dil)
    OW, pl, _ = same_pad(W, k, stride, dil)
    old = (Cout + 63) // 64 * 64 if mode == "tc" else Cout
    dev = "cuda"
    xd = torch.zeros((B, H + 2 * in_halo, W + 2 * in_halo, ld), dtype=tdt, device=dev)
    xd[:, in_halo:in_halo + H, in_halo:in_halo + W, :Cin] = torch.from_numpy(x).to(dev).to(tdt)
    ohwi = np.transpose(w, (3, 0, 1, 2))
    if mode == "tc":
        cpad = (Cout + 31) // 32 * 32
        wp = np.zeros((cpad, k, k, ld), np.float32)
        wp[:Cout, :, :, :Cin] = ohwi
    else:
        cpad, wp = Cout, np.ascontiguousarray(ohwi)
    wd = torch.from_numpy(wp).to(dev).to(tdt)
    res = None
    if residual:
        res = (rng.standard_normal((B, OH, OW, Cout))).astype(np.float32)
        if f16:
            res = res.astype(np.float16).astype(np.float32)
    out_dt = torch.float32 if (f32_out or not f16) else torch.float16
    oh = out_halo
    cOH, cOW = OH, OW                       # the convolution's own output size
    if pool:                                # out0 is the 2x2/2 max-pooled tensor
        OH, OW = OH // 2, OW // 2
    yd = torch.zeros((B, OH + 2 * oh, OW + 2 * oh, old), dtype=out_dt, device=dev)
    rd = None
    if residual:
        rd = torch.zeros((B, OH + 2 * oh, OW + 2 * oh, old), dtype=tdt, device=dev)
        rd[:, oh:oh + OH, oh:oh + OW, :Cout] = torch.from_numpy(res).to(dev).to(tdt)
    p = L.ConvParams()
    p.B, p.H, p.W, p.Cin, p.in_ld = B, H, W, Cin, ld
    p.OH, p.OW, p.Cout = cOH, cOW, Cout
    p.out0_pool = pool
    p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = k, k, stride, dil, pt, pl
    p.w_ld, p.Cout_pad = (ld if mode == "tc" else Cin), cpad
    sd = torch.from_numpy(scale).to(dev) if scale is not None else None
    hd = torch.from_numpy(shift).to(dev)
    p.scale = sd.data_ptr() if sd is not None else None
    p.shift = hd.data_ptr()
    p.act = {"relu": 1, "leaky": 2, None: 0}[act]
    p.residual = rd.data_ptr() if rd is not None else None
    p.out0 = yd.data_ptr()
    p.out0_dtype = L.ODT_F32 if out_dt == torch.float32 else L.ODT_F16
    p.out0_img_stride, p.out0_pix_stride = (OH + 2 * oh) * (OW + 2 * oh) * old, old
    p.in_halo, p.out0_halo = in_halo, out_halo
    s2 = h2 = y1 = None
    if pre:
        s2 = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
        h2 = (rng.standard_normal(Cout) * 0.2).astype(np.float32)
        s2d, h2d = torch.from_numpy(s2).to(dev), torch.from_numpy(h2).to(dev)
        ah = aux_halo
        y1 = torch.zeros((B, OH + 2 * ah, OW + 2 * ah, old), dtype=tdt, device=dev)
        p.scale2, p.shift2, p.act2 = s2d.data_ptr(), h2d.data_ptr(), 1
        p.out1, p.out1_img_stride, p.out1_pix_stride = y1.data_ptr(), (OH + 2 * ah) * (OW + 2 * ah) * old, old
        p.out1_halo = ah
    s3 = h3 = y2 = None
    if pre2:  # third epilogue output (checked in here against the rounded out0 like out1)
        s3 = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
        h3 = (rng.standard_normal(Cout) * 0.2).astype(np.float32)
        s3d, h3d = torch.from_numpy(s3).to(dev), torch.from_numpy(h3).to(dev)
        ah = aux_halo
        y2 = torch.zeros((B, OH + 2 * ah, OW + 2 * ah, old), dtype=tdt, device=dev)
        p.scale3, p.shift3, p.act3 = s3d.data_ptr(), h3d.data_ptr(), 2
        p.out2, p.out2_img_stride, p.out2_pix_stride = y2.data_ptr(), (OH + 2 * ah) * (OW + 2 * ah) * old, old
        p.out2_halo = ah
    if no_out0:
        p.out0 = None
    st = torch.cuda.current_stream().cuda_stream
    if mode == "tc":
        rc = lib.odt_conv2d_f16_tc(xd.data_ptr(), wd.data_ptr(), C.byref(p), st)
    else:
        rc = lib.odt_conv2d_direct(xd.data_ptr(), wd.data_ptr(), L.ODT_F16 if f16 else L.ODT_F32,
                                   C.byref(p), st)
    L.check(rc, "conv")
    torch.cuda.synchronize()
    ref = T.conv2d_same(x, w, None, stride, dil)
    ref = ref * (scale if scale is not None else 1.0) + shift
    if act == "relu":
        ref = np.maximum(ref, 0)
    elif act == "leaky":
        ref = np.maximum(ref, 0.1 * ref)
    if residual:
        ref = ref + res
    if pool:
        ref = T.max_pool_same(ref, 2, 2)
    got = yd[:, oh:oh + OH, oh:oh + OW, :Cout].float().cpu().numpy()
    if oh:  # the zero border must never be dirtied
        full = yd.float().cpu().numpy()
        assert np.abs(full[:, 0]).max() == 0 and np.abs(full[:, -1]).max() == 0
        assert np.abs(full[:, :, 0]).max() == 0 and np.abs(full[:, :, -1]).max() == 0
    got1 = ref1 = None
    if pre:
        base = got if (f16 and not f32_out and not no_out0) else ref
        ref1 = np.maximum(base * s2 + h2, 0)
        ah = aux_halo
        got1 = y1[:, ah:ah + OH, ah:ah + OW, :Cout].float().cpu().numpy()
        if ah:  # the zero border of a halo output is never dirtied
            f1 = y1.float().cpu().numpy()
            assert np.abs(f1[:, 0]).max() == 0 and np.abs(f1[:, -1]).max() == 0
            assert np.abs(f1[:, :, 0]).max() == 0 and np.abs(f1[:, :, -1]).max() == 0
    if pre2:
        base = got if (f16 and not f32_out and not no_out0) else ref
        t = base * s3 + h3
        ref2 = np.maximum(t, 0.1 * t)
        ah = aux_halo
        got2 = y2[:, ah:ah + OH, ah:ah + OW, :Cout].float().cpu().numpy()
        if ah:
            f2 = y2.float().cpu().numpy()
            assert np.abs(f2[:, 0]).max() == 0 and np.abs(f2[:, :, -1]).max() == 0
        tol2 = (6e-3 if f16 else 4e-5) * max(np.abs(ref2).max(), 1.0)
        assert np.abs(got2 - ref2).max() <= tol2, ("out2", float(np.abs(got2 - ref2).max()))
    if mode == "tc" and old > Cout and not f32_out:
        assert float(yd[..., Cout:].abs().max()) == 0.0, "pad channels must stay zero"
    return got, ref.astype(np.float32), got1, ref1


TC_SHAPES = [
    # B, H, W, Cin, Cout, k, stride, dil      (SSD300 / RetinaNet / YOLOv3 layer shapes, small B)
    (2, 38, 38, 512, 512, 3, 1, 1),
    (2, 19, 19, 512, 1024, 3, 1, 2),   # conv6, dilation 2
    (2, 19, 19, 1024, 1024, 1, 1, 1),  # conv7, 1x1
    (2, 19, 19, 256, 512, 3, 2, 1),    # conv8_2: 19 -> 10 pads (1,1)
    (3, 10, 10, 128, 256, 3, 2, 1),    # conv9_2: 10 -> 5 pads (0,1)
    (1, 5, 5, 128, 256, 3, 1, 1),      # conv10_2 (tile larger than the whole problem)
    (3, 75, 75, 64, 128, 3, 1, 1),     # odd width, tiles wrap rows and images
    (1, 150, 150, 64, 64, 3, 1, 1),
    (2, 26, 26, 768, 128, 1, 1, 1),    # YOLOv3 head after concat
    (2, 52, 52, 128, 256, 3, 2, 1),    # darknet down-sampling 52 -> 26 pads (0,1)
    (1, 50, 50, 256, 256, 3, 1, 1),    # RetinaNet tower
    (2, 13, 13, 256, 256, 3, 2, 1),    # P6 -> P7: 13 -> 7 pads (1,1)
    (1, 25, 25, 28, 7, 1, 1, 1),       # RetinaNet 7*2^i widths: padded Cin, tiny ragged Cout
]


@pytest.mark.parametrize("shape", TC_SHAPES)
def test_conv_tc_vs_fp32_reference(built, shape):
    got, ref, _, _ = _conv_case(*shape, mode="tc", seed=hash(shape) % 1000)
    err = np.abs(got - ref).max()
    assert err <= 2e-3 * max(np.abs(ref).max(), 1.0), (shape, float(err), float(np.abs(ref).max()))


def test_conv_tc_epilogue_variants(built):
    base = (2, 19, 19, 256, 256, 3, 1, 1)
    for kw in (dict(act="leaky", residual=True), dict(act=None, bn=False, pre=True),
               dict(act=None, residual=True, pre=True), dict(act="relu", f32_out=True)):
        got, ref, got1, ref1 = _conv_case(*base, mode="tc", **kw)
        tol = 2e-3 * max(np.abs(ref).max(), 1.0)
        assert np.abs(got - ref).max() <= tol, kw
        if got1 is not None:
            assert np.abs(got1 - ref1).max() <= 4e-3 * max(np.abs(ref1).max(), 1.0), kw
    # fp32 head scatter out of the halo-flat mode (RetinaNet regression head fed by a halo'd pre-activation)
    for cout in (36, 20):
        got, ref, _, _ = _conv_case(2, 24, 24, 256, cout, 3, 1, 1, mode="tc", act=None, f32_out=True, in_halo=1)
        assert np.abs(got - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0), ("flat head", cout)
    # head-style output: ragged Cout (100, 150), fp32, through the generic store path
    for cout in (100, 150, 75, 36, 189, 20, 4, 1):
        got, ref, _, _ = _conv_case(1, 10, 10, 256, cout, 3, 1, 1, mode="tc", act=None, f32_out=True)
        assert np.abs(got - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0), cout


@pytest.mark.parametrize("mode,tol", [("direct32", 2e-5), ("direct16", 2e-3)])
def test_conv_direct_vs_fp32_reference(built, mode, tol):
    for shape in [(2, 19, 19, 64, 96, 3, 1, 2), (2, 20, 20, 3, 16, 7, 2, 1), (1, 10, 10, 7, 28, 3, 2, 1),
                  (2, 13, 13, 100, 75, 1, 1, 1), (1, 38, 38, 32, 64, 3, 1, 1)]:
        got, ref, got1, ref1 = _conv_case(*shape, mode=mode, act="leaky", residual=True, pre=True)
        assert np.abs(got - ref).max() <= tol * max(np.abs(ref).max(), 1.0), (mode, shape)
        assert np.abs(got1 - ref1).max() <= 2 * tol * max(np.abs(ref1).max(), 1.0), (mode, shape)


def test_conv_tc_matches_direct_on_device(built):
    """The two independent device implementations agree (cross-check of im2col TMA)."""
    a, _, _, _ = _conv_case(2, 38, 38, 128, 128, 3, 1, 1, mode="tc")
    b, _, _, _ = _conv_case(2, 38, 38, 128, 128, 3, 1, 1, mode="direct16")
    assert np.abs(a - b).max() <= 4e-3 * max(np.abs(b).max(), 1.0)


def _dev(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda().to(dt)


@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_glue_kernels_vs_oracle_ops(built, dtype):
    from odt_b200 import lib as L
    from oracle import tfops as T
    lib = L.load()
    dt, code, tol = (torch.float32, L.ODT_F32, 1e-5) if dtype == "f32" else (torch.float16, L.ODT_F16, 2e-3)
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(3)

    def rnd(*s):
        a = rng.standard_normal(s).astype(np.float32)
        return a.astype(np.float16).astype(np.float32) if dtype == "f16" else a

    # max-pool 2/2 on 75 -> 38 (pads 0,1), 3/1 on 19, 3/2 on 20 -> 10
    for (h, k, s) in [(75, 2, 2), (19, 3, 1), (20, 3, 2)]:
        x = rnd(2, h, h, 64)
        ref = T.max_pool_same(x, k, s)
        y = torch.zeros(ref.shape, dtype=dt, device="cuda")
        xd = _dev(x, dt)
        L.check(lib.odt_maxpool(xd.data_ptr(), y.data_ptr(), code, 2, h, h, 64, 64, k, s, 0, 0, st))
        np.testing.assert_allclose(y.float().cpu().numpy(), ref, atol=0)
    # max-pool 3/2 + two affine/activation outputs of the pooled value, raw output optional (RetinaNet pooled stem)
    x = rnd(2, 20, 22, 16)
    ref = T.max_pool_same(x, 3, 2)
    s1, h1 = rng.uniform(.5, 1.5, 64).astype(np.float32), rng.standard_normal(64).astype(np.float32)
    s2, h2 = rng.uniform(.5, 1.5, 64).astype(np.float32), rng.standard_normal(64).astype(np.float32)
    xd = torch.zeros((2, 20, 22, 64), dtype=dt, device="cuda")
    xd[..., :16] = _dev(x, dt)
    s1d, h1d, s2d, h2d = (_dev(a, torch.float32) for a in (s1, h1, s2, h2))   # kept alive across the launches
    for with_raw in (True, False):
        y = torch.zeros((2, 10, 11, 64), dtype=dt, device="cuda")
        y1 = torch.zeros_like(y)
        y2h = torch.zeros((2, 12, 13, 64), dtype=dt, device="cuda")      # out2 in the halo layout
        L.check(lib.odt_maxpool_affine(xd.data_ptr(), y.data_ptr() if with_raw else None, code, 2, 20, 22, 16, 64, 3, 2,
                                       0, 0, s1d.data_ptr(), h1d.data_ptr(), 1, y1.data_ptr(), 0, s2d.data_ptr(),
                                       h2d.data_ptr(), 2, y2h.data_ptr(), 1, st))
        torch.cuda.synchronize()
        y2 = y2h[:, 1:11, 1:12]
        assert float(y2h[:, 0].abs().max()) == 0 and float(y2h[:, :, 12].abs().max()) == 0
        if with_raw:
            np.testing.assert_array_equal(y[..., :16].float().cpu().numpy(), ref)
        else:
            assert float(y.abs().max()) == 0.0
        t2 = ref * s2[:16] + h2[:16]
        np.testing.assert_allclose(y1[..., :16].float().cpu().numpy(), np.maximum(ref * s1[:16] + h1[:16], 0),
                                   atol=tol * 8, rtol=tol)
        np.testing.assert_allclose(y2[..., :16].float().cpu().numpy(), np.maximum(t2, 0.1 * t2), atol=tol * 8, rtol=tol)
        assert float(y1[..., 16:].abs().max()) == 0.0
    # channel L2 norm x scale
    x = rnd(2, 9, 9, 512)
    ref = 20.0 * T.l2_normalize_channels(x)
    y = torch.zeros(x.shape, dtype=dt, device="cuda")
    xd = _dev(x, dt)
    L.check(lib.odt_l2norm_scale(xd.data_ptr(), y.data_ptr(), code, 2 * 81, 512, 512, 20.0, st))
    np.testing.assert_allclose(y.float().cpu().numpy(), ref, atol=tol * 4, rtol=tol)
    # affine + relu
    x = rnd(2, 7, 7, 64)
    sc, sh = rng.uniform(.5, 1.5, 64).astype(np.float32), rng.standard_normal(64).astype(np.float32)
    y = torch.zeros(x.shape, dtype=dt, device="cuda")
    xd, scd, shd = _dev(x, dt), _dev(sc, torch.float32), _dev(sh, torch.float32)
    L.check(lib.odt_affine_act(xd.data_ptr(), y.data_ptr(), code, 98, 64, 64, scd.data_ptr(), shd.data_ptr(), 1, st))
    np.testing.assert_allclose(y.float().cpu().numpy(), np.maximum(x * sc + sh, 0), atol=tol * 8, rtol=tol)
    # FPN: a + legacy bilinear(top), 13 -> 25 and 4 -> 8
    for th, h in [(13, 25), (4, 8), (25, 50)]:
        top, a = rnd(2, th, th, 64), rnd(2, h, h, 64)
        ref = a + T.resize_bilinear_legacy(top, h, h)
        y = torch.zeros(a.shape, dtype=dt, device="cuda")
        topd, ad = _dev(top, dt), _dev(a, dt)
        L.check(lib.odt_upsample_bilinear_add(topd.data_ptr(), ad.data_ptr(), y.data_ptr(),
                                              code, 2, th, th, h, h, 64, 64, None, None, 0, None, st))
        np.testing.assert_allclose(y.float().cpu().numpy(), ref, atol=tol * 8, rtol=tol)
    # YOLOv3 nearest + concat
    a, b = rnd(2, 26, 26, 64), rnd(2, 13, 13, 32)
    ref = np.concatenate([a, T.resize_nearest_legacy(b, 26, 26)], axis=3)
    y = torch.zeros((2, 26, 26, 128), dtype=dt, device="cuda")
    ad, bd = _dev(a, dt), _dev(b, dt)
    L.check(lib.odt_upsample_nearest_concat(ad.data_ptr(), bd.data_ptr(), y.data_ptr(), code,
                                            2, 26, 26, 64, 64, 13, 13, 32, 32, 128, st))
    np.testing.assert_array_equal(y[..., :96].float().cpu().numpy(), ref)
    # GroupNorm(8) + relu
    x = rnd(2, 11, 13, 64)
    g, bt = rng.uniform(.5, 1.5, 64).astype(np.float32), rng.standard_normal(64).astype(np.float32)
    ref = np.maximum(T.group_norm(x, g, bt), 0)
    stats = torch.zeros(2 * 8 * 6, dtype=torch.float32, device="cuda")
    y = torch.zeros(x.shape, dtype=dt, device="cuda")
    xd, gd, btd = _dev(x, dt), _dev(g, torch.float32), _dev(bt, torch.float32)
    L.check(lib.odt_groupnorm_stats(xd.data_ptr(), stats.data_ptr(), code, 2, 11 * 13, 64, 64, 8, 1e-6, st))
    L.check(lib.odt_groupnorm_apply(xd.data_ptr(), y.data_ptr(), stats.data_ptr(), code, 2, 11 * 13, 64, 64, 8,
                                    gd.data_ptr(), btd.data_ptr(), 1, st))
    np.testing.assert_allclose(y.float().cpu().numpy(), ref, atol=tol * 8, rtol=tol)
    # a1: images - RGB mean into a padded NHWC tensor (SSD300.py:52-66); channels >= 3 are written as zero
    img = rng.integers(0, 256, (2, 9, 11, 3)).astype(np.float32)
    mean = (C.c_float * 3)(123.68, 116.779, 103.979)
    y = torch.full((2, 9, 11, 8), 7.0, dtype=dt, device="cuda")
    imgd = _dev(img, torch.float32)
    L.check(lib.odt_normalize_input(imgd.data_ptr(), y.data_ptr(), code, 2, 9, 11, 8, mean, st))
    got = y.float().cpu().numpy()
    ref = img - np.array([123.68, 116.779, 103.979], np.float32)
    np.testing.assert_allclose(got[..., :3], ref.astype(np.float16).astype(np.float32) if dtype == "f16" else ref,
                               atol=0)
    assert np.all(got[..., 3:] == 0)
    torch.cuda.synchronize()


STEM_SHAPES = [
    (2, 300, 300, 64, 3, 1),   # SSD conv1_1
    (3, 37, 53, 64, 3, 1),     # ragged tile tail
    (2, 64, 64, 32, 3, 1),     # YOLOv3 stem
    (2, 128, 128, 16, 7, 2),   # RetinaNet / FCOS stem (K = 147, 3 swizzle blocks)
    (1, 33, 47, 16, 7, 2),
    (1, 20, 20, 24, 5, 1),     # no specialised variant -> generic CUDA-core stem
]


# the packed-image stem ('rgbx') exists for 7x7 filters only: no 3x3 case is generated for it
@pytest.mark.parametrize("dtype,shape", [
    pytest.param(d, s, id="%s-shape%d" % (d, i)) for d in ("f16", "f32", "rgbx") for i, s in enumerate(STEM_SHAPES)
    if d != "rgbx" or s[4] != 3])
def test_stem_conv_vs_oracle(built, shape, dtype):
    """odt_conv2d_stem: fp32 image - RGB mean -> conv -> bias/BN -> ReLU.  fp16 takes the
    tensor-core stem (A tile built in swizzled smem), fp32 the CUDA-core stem; 'rgbx' = odt_pack_input_rgbx +
    odt_conv2d_stem_rgbx (the tensor-core stem on the packed fp16 image, which the engine runs for the 7x7/2 stems)."""
    from odt_b200 import lib as L
    from odt_b200.engine import same_pad
    from oracle import tfops as T
    lib = L.load()
    B, H, W, Cout, k, stride = shape
    rng = np.random.default_rng(7)
    img = rng.integers(0, 256, (B, H, W, 3)).astype(np.float32)
    w = (rng.standard_normal((k, k, 3, Cout)) * np.sqrt(2.0 / (k * k * 3)) / 64).astype(np.float32)
    rgbx = dtype == "rgbx"
    f16 = dtype in ("f16", "rgbx")
    if f16:
        w = w.astype(np.float16).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    shift = (rng.standard_normal(Cout) * 0.2).astype(np.float32)
    tdt = torch.float16 if f16 else torch.float32
    ld = (Cout + 63) // 64 * 64 if f16 else Cout
    OH, pt, _ = same_pad(H, k, stride)
    OW, pl, _ = same_pad(W, k, stride)
    P = 4 if (k, stride) == (7, 2) else 0
    if rgbx and (P == 0 or Cout != 16 or W % 2 or pl % 2):
        pytest.skip("no packed-image variant for this shape (the engine falls back to odt_conv2d_stem)")
    imgd = torch.from_numpy(img).cuda()
    wd = torch.from_numpy(np.ascontiguousarray(np.transpose(w, (3, 0, 1, 2)))).cuda().to(tdt)
    sd, hd = torch.from_numpy(scale).cuda(), torch.from_numpy(shift).cuda()
    oh = 1 if (f16 and (k, stride, Cout) in [(3, 1, 64), (7, 2, 16)] and B == 2) else 0  # halo output variants
    yd = torch.zeros((B, OH + 2 * oh, OW + 2 * oh, ld), dtype=tdt, device="cuda")
    p = L.ConvParams()
    p.B, p.H, p.W, p.Cin, p.in_ld = B, H, W, 3, 3
    p.OH, p.OW, p.Cout = OH, OW, Cout
    p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = k, k, stride, 1, pt, pl
    p.w_ld, p.Cout_pad = 3, Cout
    p.scale, p.shift, p.act = sd.data_ptr(), hd.data_ptr(), 1
    p.out0, p.out0_dtype = yd.data_ptr(), (L.ODT_F16 if f16 else L.ODT_F32)
    p.out0_img_stride, p.out0_pix_stride = (OH + 2 * oh) * (OW + 2 * oh) * ld, ld
    p.out0_halo = oh
    mean = (C.c_float * 3)(123.68, 116.779, 103.979)
    st = torch.cuda.current_stream().cuda_stream
    if rgbx:
        packed = torch.zeros((B, H + 2 * P, W + 2 * P, 4), dtype=torch.float16, device="cuda")
        L.check(lib.odt_pack_input_rgbx(imgd.data_ptr(), packed.data_ptr(), B, H, W, P, mean, st), "pack")
        pk = packed.float().cpu().numpy()
        exp = (img - np.array([123.68, 116.779, 103.979], np.float32)).astype(np.float16).astype(np.float32)
        np.testing.assert_array_equal(pk[:, P:P + H, P:P + W, :3], exp)
        assert np.all(pk[..., 3] == 0) and np.all(pk[:, :P] == 0) and np.all(pk[:, :, W + P:] == 0)
        p.in_ld, p.in_halo = 4, P
        L.check(lib.odt_conv2d_stem_rgbx(packed.data_ptr(), wd.data_ptr(), C.byref(p), st), "stem_rgbx")
    else:
        L.check(lib.odt_conv2d_stem(imgd.data_ptr(), mean, wd.data_ptr(), L.ODT_F16 if f16 else L.ODT_F32,
                                    C.byref(p), st), "stem")
    torch.cuda.synchronize()
    x = img - T.RGB_MEAN.reshape(1, 1, 1, 3)
    xr = x.astype(np.float16).astype(np.float32) if f16 else x  # the fp16 stem rounds the operand
    ref = np.maximum(T.conv2d_same(xr, w, None, stride) * scale + shift, 0)
    got = yd[:, oh:oh + OH, oh:oh + OW, :Cout].float().cpu().numpy()
    if oh:
        assert float(yd[:, 0].abs().max()) == 0 and float(yd[:, :, 0].abs().max()) == 0
    tol = (3e-3 if f16 else 2e-5) * max(np.abs(ref).max(), 1.0)
    assert np.abs(got - ref).max() <= tol, (shape, dtype, float(np.abs(got - ref).max()), float(np.abs(ref).max()))
    if ld > Cout:
        assert float(yd[..., Cout:].abs().max()) == 0.0


FLAT_SHAPES = [
    # B, H, W, Cin, Cout, k, stride, dil : 3x3 s1 with a halo input -> halo-flat path (Cout_pad <= 128)
    (2, 38, 38, 64, 64, 3, 1, 1),
    (3, 75, 75, 64, 128, 3, 1, 1),     # odd width: tiles wrap padded rows and images
    (1, 150, 150, 128, 128, 3, 1, 1),  # two channel chunks
    (2, 20, 23, 192, 96, 3, 1, 1),     # non-square, three chunks, N = 96
    (1, 16, 16, 64, 28, 3, 1, 1),      # ragged Cout
]


@pytest.mark.parametrize("shape", FLAT_SHAPES)
@pytest.mark.parametrize("out_halo", [0, 1])
@pytest.mark.parametrize("tapn", ["0", "1"])   # 0: conv_tc's own flat modes; 1: the default planner (taps-as-N where it pays)
def test_conv_tc_flat_halo_vs_fp32_reference(built, monkeypatch, shape, out_halo, tapn):
    monkeypatch.setenv("ODT_TC_TAPN", tapn)
    got, ref, _, _ = _conv_case(*shape, mode="tc", in_halo=1, out_halo=out_halo, seed=sum(shape))
    assert np.abs(got - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0), (shape, out_halo)


POOL_SHAPES = [
    # 3x3 s1 halo-flat conv + fused 2x2/2 max-pool (SSD300 conv1_2 / conv2_2 and friends)
    (2, 300, 300, 64, 64, 3, 1, 1),    # conv1_2: 2-row x 64-column tiles, ragged last column block
    (2, 150, 150, 128, 128, 3, 1, 1),  # conv2_2: 4-row x 32-column tiles, ragged last row block
    (3, 38, 38, 64, 96, 3, 1, 1),      # small map, N = 96
    (1, 16, 130, 64, 28, 3, 1, 1),     # ragged Cout, non-square
    (2, 6, 4, 64, 64, 3, 1, 1),        # tile larger than the image
]


@pytest.mark.parametrize("shape", POOL_SHAPES)
@pytest.mark.parametrize("out_halo", [0, 1])
@pytest.mark.parametrize("tapn", ["0", "1"])
def test_conv_tc_fused_maxpool(built, monkeypatch, shape, out_halo, tapn):
    """Pooled epilogue against max_pool(fp32 conv reference), and bit-exact against the
    same conv followed by the stand-alone pooling kernel (max commutes with fp16 rounding)."""
    from odt_b200 import lib as L
    monkeypatch.setenv("ODT_TC_TAPN", tapn)
    got, ref, _, _ = _conv_case(*shape, mode="tc", in_halo=1, out_halo=out_halo, pool=2, seed=sum(shape))
    assert np.abs(got - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0), (shape, out_halo)
    full, _, _, _ = _conv_case(*shape, mode="tc", in_halo=1, out_halo=0, seed=sum(shape))
    B, H, W, _, Cout = shape[:5]
    ld = (Cout + 63) // 64 * 64
    xd = torch.zeros((B, H, W, ld), dtype=torch.float16, device="cuda")
    xd[..., :Cout] = torch.from_numpy(full).cuda().half()
    yd = torch.zeros((B, H // 2, W // 2, ld), dtype=torch.float16, device="cuda")
    L.check(L.load().odt_maxpool(xd.data_ptr(), yd.data_ptr(), L.ODT_F16, B, H, W, ld, ld, 2, 2, 0, 0,
                                 torch.cuda.current_stream().cuda_stream))
    np.testing.assert_array_equal(got, yd[..., :Cout].float().cpu().numpy())


def test_conv_tc_fused_maxpool_rejects_bad_shapes(built):
    from odt_b200 import lib as L
    with pytest.raises(L.OdtError):   # odd size
        _conv_case(1, 75, 75, 64, 64, 3, 1, 1, mode="tc", in_halo=1, pool=2)
    with pytest.raises(L.OdtError):   # no halo input
        _conv_case(1, 16, 16, 64, 64, 3, 1, 1, mode="tc", in_halo=0, pool=2)


@pytest.mark.parametrize("shape,pool", [((2, 38, 38, 64, 64, 3, 1, 1), 0), ((3, 75, 75, 64, 128, 3, 1, 1), 0),
                                        ((2, 300, 300, 64, 64, 3, 1, 1), 2), ((1, 40, 40, 128, 64, 3, 1, 1), 2)])
def test_conv_tc_resident_filter_bank_is_bit_identical(built, shape, pool):
    """Layers whose filter bank stays resident in shared memory, against the fp32 reference, and two launches
    bit-identical."""
    a, ref, _, _ = _conv_case(*shape, mode="tc", in_halo=1, out_halo=1, pool=pool)
    b, _, _, _ = _conv_case(*shape, mode="tc", in_halo=1, out_halo=1, pool=pool)
    assert np.abs(a - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0)
    np.testing.assert_array_equal(a, b)


LARGE_SHAPES = [
    # hundreds of tiles, several rounds of the persistent grid: B, H, W, Cin, Cout, k, stride, dil
    (5, 88, 88, 128, 256, 3, 1, 1),    # 303 M tiles: odd count + ragged last tile
    (4, 69, 69, 128, 512, 3, 1, 1),    # four N tiles of 128, 149 M tiles
    (8, 75, 75, 256, 128, 1, 1, 1),    # 1x1, N = 128
    (8, 150, 150, 64, 192, 3, 2, 1),   # stride 2, N = 192
    (6, 80, 80, 64, 96, 3, 1, 2),      # dilation 2, N = 96
]


@pytest.mark.parametrize("shape", LARGE_SHAPES)
def test_conv_tc_large_tile_counts(built, shape):
    """Layers of hundreds of tiles (odd tile counts, ragged last tiles, several N tiles, stride, dilation) against the
    fp32 reference, and two launches bit-identical (static tile schedule, fixed K order)."""
    a, ref, a1, r1 = _conv_case(*shape, mode="tc", act="leaky", residual=True, pre=True, seed=sum(shape))
    tol = 2e-3 * max(np.abs(ref).max(), 1.0)
    assert np.abs(a - ref).max() <= tol and np.abs(a1 - r1).max() <= 2 * tol
    b, _, b1, _ = _conv_case(*shape, mode="tc", act="leaky", residual=True, pre=True, seed=sum(shape))
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(a1, b1)


def test_conv_tc_large_head_scatter_and_halo(built):
    # fp32 head rows (RetinaNet cls head shape class) and halo in/out layouts at large tile counts
    g, ref, _, _ = _conv_case(4, 100, 100, 256, 189, 3, 1, 1, mode="tc", act=None, f32_out=True)
    assert np.abs(g - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0)
    h, ref2, _, _ = _conv_case(4, 100, 100, 128, 256, 3, 1, 1, mode="tc", in_halo=1, out_halo=1)
    assert np.abs(h - ref2).max() <= 2e-3 * max(np.abs(ref2).max(), 1.0)
    h0, _, _, _ = _conv_case(4, 100, 100, 128, 256, 3, 1, 1, mode="tc", in_halo=1, out_halo=1)
    np.testing.assert_array_equal(h, h0)


@pytest.mark.parametrize("shape,pool", [((2, 38, 38, 64, 64, 3, 1, 1), 0), ((3, 75, 75, 64, 128, 3, 1, 1), 0),
                                        ((2, 300, 300, 64, 64, 3, 1, 1), 2), ((2, 150, 150, 128, 128, 3, 1, 1), 2),
                                        ((1, 150, 150, 128, 128, 3, 1, 1), 0), ((1, 17, 23, 64, 28, 3, 1, 1), 0)])
def test_conv_tc_flat_modes_bit_identical(built, shape, pool):
    """Halo-flat / row-block modes against the fp32 reference, and two launches bit-identical."""
    a, ref, _, _ = _conv_case(*shape, mode="tc", in_halo=1, out_halo=1, pool=pool)
    assert np.abs(a - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0)
    b, _, _, _ = _conv_case(*shape, mode="tc", in_halo=1, out_halo=1, pool=pool)
    np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("shape,kw", [
    ((2, 38, 38, 128, 256, 3, 1, 1), {}),                       # im2col mode
    ((8, 75, 75, 128, 256, 3, 1, 1), {"residual": True}),       # two N tiles + residual
    ((2, 40, 40, 64, 96, 3, 1, 1), {"in_halo": 1}),             # halo-flat mode
    ((2, 26, 26, 512, 28, 1, 1, 1), {"no_out0": True}),         # ragged Cout, only the two pre-activations wanted
])
def test_conv_tc_two_preactivation_outputs(built, shape, kw):
    """out1 and out2 (two consumer BN+activation variants of the same conv output)."""
    got, ref, g1, r1 = _conv_case(*shape, mode="tc", pre=True, pre2=True, **kw)
    tol = 2e-3 * max(np.abs(ref).max(), 1.0)
    if not kw.get("no_out0"):
        assert np.abs(got - ref).max() <= tol
    assert np.abs(g1 - r1).max() <= 3 * tol


@pytest.mark.parametrize("shape,kw,env", [
    ((2, 40, 40, 7, 28, 1, 1, 1), {"residual": True}, {}),                        # im2col mode, 1x1 expand (RetinaNet)
    ((2, 40, 40, 28, 28, 3, 1, 1), {"in_halo": 1}, {"ODT_TC_TAPN": "0"}),         # halo-flat mode
    ((2, 40, 40, 28, 28, 3, 1, 1), {"in_halo": 1}, {"ODT_TC_TAPN": "2"}),         # taps-as-N
    ((2, 40, 40, 16, 7, 1, 1, 1), {}, {"ODT_TC_THIN": "2"}),                      # thin CUDA-core kernel
    ((2, 37, 41, 128, 256, 3, 2, 1), {"act": "leaky"}, {}),                       # stride 2, odd sizes, N = 256
])
def test_conv_extra_outputs_in_halo_layout(built, monkeypatch, shape, kw, env):
    """out1 / out2 (the consumer pre-activations) written as [B][OH+2][OW+2][ld] with an untouched zero border, by
    every kernel behind odt_conv2d_f16_tc: the 3x3 convolutions that read them then take the halo modes."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    got, ref, g1, r1 = _conv_case(*shape, mode="tc", seed=sum(shape), pre=True, pre2=True, aux_halo=1, **kw)
    tol = 2e-3 * max(np.abs(ref).max(), 1.0)
    assert np.abs(got - ref).max() <= tol, shape
    assert np.abs(g1 - r1).max() <= 3 * tol


def test_conv_direct_two_preactivation_outputs(built):
    got, ref, g1, r1 = _conv_case(2, 20, 20, 24, 40, 3, 1, 1, mode="direct32", pre=True, pre2=True)
    assert np.abs(got - ref).max() <= 2e-5 * max(np.abs(ref).max(), 1.0)


@pytest.mark.parametrize("shape,kw", [
    ((2, 40, 40, 7, 7, 3, 1, 1), {"in_halo": 1, "out_halo": 1}),     # thin flat layer: 1 of 4 K steps issued
    ((2, 40, 40, 28, 7, 1, 1, 1), {}),                               # thin 1x1: 2 of 4
    ((2, 26, 26, 40, 64, 3, 2, 1), {}),                              # 3 of 4, stride 2
    ((8, 75, 75, 100, 256, 3, 1, 1), {}),                            # second chunk holds 36 channels, two N tiles
    ((2, 64, 64, 16, 28, 3, 1, 1), {"in_halo": 1, "pool": 2}),       # row-block pooled mode
])
def test_conv_tc_thin_input_channels(built, shape, kw):
    """Cin that does not fill its 64-channel chunk (RetinaNet's 7*2^i widths, zero-padded operands) in every
    tensor-core mode; the all-zero 16-deep K steps are not issued."""
    got, ref, _, _ = _conv_case(*shape, mode="tc", seed=sum(shape), **kw)
    assert np.abs(got - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0), shape


def test_conv_tc_flat_equals_im2col_path(built):
    """The same operands through both tensor-core paths: stored with a halo (halo-flat mode) and densely (im2col
    mode; _conv_case draws the same values whatever the layout)."""
    shape = (2, 38, 38, 128, 128, 3, 1, 1)
    a, ref, a1, r1 = _conv_case(*shape, mode="tc", in_halo=1, out_halo=1, act="leaky", residual=True, pre=True)
    b, _, b1, _ = _conv_case(*shape, mode="tc", in_halo=0, out_halo=0, act="leaky", residual=True, pre=True)
    tol = 2e-3 * max(np.abs(ref).max(), 1.0)
    assert np.abs(a - ref).max() <= tol and np.abs(b - ref).max() <= tol
    assert np.abs(a1 - r1).max() <= 2 * tol and np.abs(b1 - r1).max() <= 2 * tol
    # identical operand values and accumulation order per tap chunk -> (near) identical results
    assert np.abs(a - b).max() <= 1e-3 * max(np.abs(ref).max(), 1.0)


@pytest.mark.parametrize("shape", [
    (2, 19, 19, 256, 512, 3, 2, 1),   # im2col path reading a halo input (stride 2)
    (2, 38, 38, 256, 256, 3, 1, 1),   # 3x3 s1 but N = 256: im2col path with halo input
    (2, 26, 26, 128, 64, 1, 1, 1),    # 1x1 writing a halo output
])
def test_conv_tc_im2col_with_halo_layouts(built, shape):
    got, ref, _, _ = _conv_case(*shape, mode="tc", in_halo=1, out_halo=1)
    assert np.abs(got - ref).max() <= 2e-3 * max(np.abs(ref).max(), 1.0), shape


def test_maxpool_halo_layouts(built):
    from odt_b200 import lib as L
    from oracle import tfops as T
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    x = np.random.default_rng(1).standard_normal((2, 75, 75, 64)).astype(np.float16).astype(np.float32)
    ref = T.max_pool_same(x, 2, 2)
    for ih, oh in [(1, 1), (1, 0), (0, 1)]:
        xd = torch.zeros((2, 75 + 2 * ih, 75 + 2 * ih, 64), dtype=torch.float16, device="cuda")
        xd[:, ih:ih + 75, ih:ih + 75] = torch.from_numpy(x).cuda().half()
        yd = torch.zeros((2, 38 + 2 * oh, 38 + 2 * oh, 64), dtype=torch.float16, device="cuda")
        L.check(lib.odt_maxpool(xd.data_ptr(), yd.data_ptr(), L.ODT_F16, 2, 75, 75, 64, 64, 2, 2, ih, oh, st))
        got = yd[:, oh:oh + 38, oh:oh + 38].float().cpu().numpy()
        np.testing.assert_array_equal(got, ref)
        if oh:
            assert float(yd[:, 0].abs().max()) == 0 and float(yd[:, :, -1].abs().max()) == 0


@pytest.mark.parametrize("geom", [(3, 75, 75, 256, 2, 2), (2, 38, 37, 512, 2, 2), (3, 19, 19, 512, 3, 1), (2, 10, 13, 64, 3, 1)])
@pytest.mark.parametrize("halo", [(0, 0), (1, 1), (1, 0)])
def test_maxpool_specialised_kernel_is_bit_identical_to_the_generic_one(built, geom, halo):
    """maxpool_h8_kernel<K,S> (compile-time window, clamped taps, loads in flight) against the oracle's TF-SAME
    pooling, odd sizes and halo layouts included.  Max-pooling is exact, so equality with the oracle is equality with
    the generic maxpool_kernel too (tests/test_gpu_glue.py runs that one)."""
    from odt_b200 import lib as L
    from oracle import tfops as T
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    B, H, W, Cc, k, s = geom
    ih, oh = halo
    x = np.random.default_rng(H * W + Cc).standard_normal((B, H, W, Cc)).astype(np.float16)
    ref = T.max_pool_same(x.astype(np.float32), k, s)
    OH, OW = ref.shape[1:3]
    xd = torch.zeros((B, H + 2 * ih, W + 2 * ih, Cc), dtype=torch.float16, device="cuda")
    xd[:, ih:ih + H, ih:ih + W] = torch.from_numpy(x).cuda()
    yd = torch.zeros((B, OH + 2 * oh, OW + 2 * oh, Cc), dtype=torch.float16, device="cuda")
    L.check(lib.odt_maxpool(xd.data_ptr(), yd.data_ptr(), L.ODT_F16, B, H, W, Cc, Cc, k, s, ih, oh, st))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(yd[:, oh:oh + OH, oh:oh + OW].float().cpu().numpy(), ref)
    border = yd.clone()
    border[:, oh:oh + OH, oh:oh + OW] = 0
    assert not border.any()  # nothing written into an output halo


# The "taps as N" kernel (csrc/conv_tapn.cu) and the thin-layer kernel (csrc/conv_thin.cu) are default paths since
# the round-2 A/B (mode 1 = where their cost rules take a layer); the tests force mode 2 (wherever a layer qualifies).
@pytest.mark.parametrize("shape,kw", [
    ((2, 40, 40, 64, 64, 3, 1, 1), {"in_halo": 1, "out_halo": 1}),
    ((2, 37, 61, 64, 64, 3, 1, 1), {"in_halo": 1}),                              # ragged rows / columns
    ((2, 40, 40, 7, 7, 3, 1, 1), {"in_halo": 1, "out_halo": 1}),                 # thin: N = 96, one K step
    ((2, 40, 40, 28, 28, 3, 1, 1), {"in_halo": 1, "residual": True, "pre": True, "pre2": True}),
    ((2, 26, 26, 128, 64, 3, 1, 1), {"in_halo": 1, "act": "leaky"}),             # two channel chunks
    ((2, 64, 64, 64, 64, 3, 1, 1), {"in_halo": 1, "pool": 2}),
    ((1, 8, 300, 64, 64, 3, 1, 1), {"in_halo": 1, "out_halo": 1, "pool": 2}),    # ten full column blocks
    ((2, 30, 46, 16, 28, 3, 1, 1), {"in_halo": 1, "pool": 2}),
])
def test_conv_tapn_matches_reference(built, monkeypatch, shape, kw):
    from odt_b200 import lib as L
    monkeypatch.setenv("ODT_TC_TAPN", "2")   # 2 = wherever the layer qualifies (1 also asks the cost model)
    before = L.load().odt_debug_tapn_launches()
    got, ref, g1, r1 = _conv_case(*shape, mode="tc", seed=sum(shape), **kw)
    assert L.load().odt_debug_tapn_launches() == before + 1, "the layer did not take the taps-as-N path"
    tol = 2e-3 * max(np.abs(ref).max(), 1.0)
    assert np.abs(got - ref).max() <= tol, shape
    if g1 is not None:
        assert np.abs(g1 - r1).max() <= 3 * tol


def _tc_raw(x, w, pool=0, in_halo=1, out_halo=1):
    """x [B,H,W,Cin] fp16 device tensor (unpadded), w [Cout,3,3,Cin] fp16 -> raw kernel output (no CPU reference):
    3x3 / stride 1 / SAME, zero shift, ReLU.  For size-independent properties at BASELINE sizes."""
    from odt_b200 import lib as L
    lib = L.load()
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    ld, old, cpad = (Cin + 63) // 64 * 64, (Cout + 63) // 64 * 64, (Cout + 31) // 32 * 32
    ih, oh = in_halo, out_halo
    xd = torch.zeros((B, H + 2 * ih, W + 2 * ih, ld), dtype=torch.float16, device="cuda")
    xd[:, ih:ih + H, ih:ih + W, :Cin] = x
    wd = torch.zeros((cpad, 3, 3, ld), dtype=torch.float16, device="cuda")
    wd[:Cout, :, :, :Cin] = w
    yh, yw = (H // 2, W // 2) if pool else (H, W)
    y = torch.zeros((B, yh + 2 * oh, yw + 2 * oh, old), dtype=torch.float16, device="cuda")
    shift = torch.zeros(Cout, device="cuda")
    p = L.ConvParams()
    p.B, p.H, p.W, p.Cin, p.in_ld = B, H, W, Cin, ld
    p.OH, p.OW, p.Cout = H, W, Cout
    p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = 3, 3, 1, 1, 1, 1
    p.w_ld, p.Cout_pad = ld, cpad
    p.shift, p.act = shift.data_ptr(), 1
    p.out0, p.out0_dtype = y.data_ptr(), L.ODT_F16
    p.out0_img_stride, p.out0_pix_stride = (yh + 2 * oh) * (yw + 2 * oh) * old, old
    p.in_halo, p.out0_halo, p.out0_pool = ih, oh, pool
    L.check(lib.odt_conv2d_f16_tc(xd.data_ptr(), wd.data_ptr(), C.byref(p), torch.cuda.current_stream().cuda_stream),
            "conv")
    torch.cuda.synchronize()
    return y[:, oh:oh + yh, oh:oh + yw, :Cout]


@pytest.mark.parametrize("shape,kw", [
    ((2, 40, 40, 16, 7, 1, 1, 1), {"pre": True}),                                       # 1x1 reduce + consumer BN/ReLU
    ((2, 37, 41, 28, 7, 1, 1, 1), {"in_halo": 1, "out_halo": 1}),                       # halo both sides, ragged block
    ((2, 40, 40, 7, 28, 1, 1, 1), {"residual": True, "pre": True, "pre2": True, "no_out0": True, "aux_halo": 1}),
    ((2, 40, 40, 7, 28, 1, 1, 1), {"residual": True, "pre": True, "pre2": True, "out_halo": 1}),
    ((2, 33, 35, 14, 56, 1, 1, 1), {"residual": True, "pre": True, "pre2": True, "no_out0": True, "aux_halo": 1}),
    ((2, 25, 25, 28, 112, 1, 1, 1), {"residual": True, "pre": True, "pre2": True, "no_out0": True, "aux_halo": 1}),
    ((2, 13, 13, 56, 224, 1, 1, 1), {"residual": True, "pre": True, "aux_halo": 1}),
    ((2, 25, 25, 112, 28, 1, 1, 1), {"act": "leaky", "in_halo": 1}),
    ((2, 20, 20, 56, 14, 1, 1, 1), {"pre": True, "aux_halo": 1}),
])
def test_conv_pw_matches_reference(built, monkeypatch, shape, kw):
    """Staged pointwise kernel for RetinaNet's narrow 1x1 layers (csrc/conv_pw.cu) behind the tensor-core entry point:
    ODT_TC_PW=2 = wherever the layer qualifies (the default planner leaves 56->224 to the tensor cores)."""
    from odt_b200 import lib as L
    monkeypatch.setenv("ODT_TC_PW", "2")
    before = L.load().odt_debug_pw_launches()
    got, ref, g1, r1 = _conv_case(*shape, mode="tc", seed=sum(shape), **kw)
    assert L.load().odt_debug_pw_launches() == before + 1, "the layer did not take the pointwise path"
    tol = 2e-3 * max(np.abs(ref).max(), 1.0)
    if not kw.get("no_out0"):
        assert np.abs(got - ref).max() <= tol, shape
    if g1 is not None:
        assert np.abs(g1 - r1).max() <= 3 * tol


def test_conv_pw_is_bit_identical_to_the_tensor_core_path_on_exact_inputs(built, monkeypatch):
    """Small-integer activations and weights make every product and partial sum exact in fp16 / fp32, so the
    CUDA-core pointwise kernel and the wgmma kernel must agree bit for bit (same epilogue rounding chain)."""
    from odt_b200 import lib as L
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(3)
    B, H, W, Cin, Cout = 4, 50, 50, 28, 112
    ld, old = 64, 128
    x = torch.zeros((B, H, W, ld), dtype=torch.float16, device="cuda")
    x[..., :Cin] = torch.randint(-4, 5, (B, H, W, Cin), generator=g, device="cuda").half()
    w = torch.zeros((128, 1, 1, ld), dtype=torch.float16, device="cuda")
    w[:Cout, 0, 0, :Cin] = torch.randint(-3, 4, (Cout, Cin), generator=g, device="cuda").half() / 8
    res = torch.zeros((B, H, W, old), dtype=torch.float16, device="cuda")
    res[..., :Cout] = torch.randint(-8, 9, (B, H, W, Cout), generator=g, device="cuda").half()
    scale = torch.full((Cout,), 0.5, device="cuda")
    shift = torch.full((Cout,), 0.25, device="cuda")
    outs = []
    for mode in ("0", "2"):
        monkeypatch.setenv("ODT_TC_PW", mode)
        monkeypatch.setenv("ODT_TC_THIN", "0")
        y0 = torch.zeros((B, H, W, old), dtype=torch.float16, device="cuda")
        y1 = torch.zeros((B, H + 2, W + 2, old), dtype=torch.float16, device="cuda")
        p = L.ConvParams()
        p.B, p.H, p.W, p.Cin, p.in_ld = B, H, W, Cin, ld
        p.OH, p.OW, p.Cout = H, W, Cout
        p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = 1, 1, 1, 1, 0, 0
        p.w_ld, p.Cout_pad = ld, 128
        p.scale, p.shift, p.act = scale.data_ptr(), shift.data_ptr(), 0
        p.residual = res.data_ptr()
        p.out0, p.out0_dtype = y0.data_ptr(), L.ODT_F16
        p.out0_img_stride, p.out0_pix_stride = H * W * old, old
        p.scale2, p.shift2, p.act2 = shift.data_ptr(), scale.data_ptr(), 1
        p.out1, p.out1_img_stride, p.out1_pix_stride, p.out1_halo = y1.data_ptr(), (H + 2) * (W + 2) * old, old, 1
        before = lib.odt_debug_pw_launches()
        L.check(lib.odt_conv2d_f16_tc(x.data_ptr(), w.data_ptr(), C.byref(p), torch.cuda.current_stream().cuda_stream),
                "conv")
        torch.cuda.synchronize()
        assert lib.odt_debug_pw_launches() == before + (mode == "2")
        outs.append((y0, y1))
    assert float(outs[0][0].float().abs().max()) > 1.0
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("tapn", ["0", "2"])
def test_conv1_2_full_size_properties(built, monkeypatch, tapn):
    """SSD300's conv1_2 + fused pool at the BASELINE batch (64 x 300 x 300 x 64 -> 64): properties that need no
    oracle.  (a) scaling the input by 2 scales the output by 2 bit for bit (powers of two commute with every
    rounding of a normal number, with ReLU and with max); (b) an image computed alone equals its slice of the batch (tiles never mix images);
    (c) two runs agree bit for bit."""
    monkeypatch.setenv("ODT_TC_TAPN", tapn)
    g = torch.Generator(device="cuda").manual_seed(7)
    x = (torch.randn((64, 300, 300, 64), generator=g, device="cuda") * 0.5).half()
    w = (torch.randn((64, 3, 3, 64), generator=g, device="cuda") * (2.0 / 576) ** 0.5).half()
    y = _tc_raw(x, w, pool=2)
    assert y.shape == (64, 150, 150, 64) and float(y.float().abs().max()) > 0.1
    assert torch.equal(_tc_raw(x, w, pool=2), y)
    d = (_tc_raw(x * 2, w, pool=2).float() - 2 * y.float()).abs()
    assert float(d[y >= 1e-3].max()) == 0.0          # exact wherever the fp16 result is a normal number
    assert float(d.max()) <= 2.0 ** -22               # fp16 subnormals: the fixed 2^-24 grid breaks the commutation
    for b in (0, 37, 63):
        assert torch.equal(_tc_raw(x[b:b + 1], w, pool=2)[0], y[b])
    # pooling really happened: the un-pooled result, max-reduced on the device, is the same tensor
    full = _tc_raw(x[:2], w, pool=0)
    assert torch.equal(full.reshape(2, 150, 2, 150, 2, 64).amax(dim=(2, 4)), y[:2])


@pytest.mark.parametrize("shape,kw", [
    ((2, 40, 40, 7, 7, 3, 1, 1), {"in_halo": 1, "out_halo": 1}),                       # RetinaNet stage 1, 3x3
    ((2, 37, 41, 7, 7, 3, 1, 1), {}),                                                   # no halo: border checks
    ((2, 40, 40, 16, 7, 1, 1, 1), {"pre": True}),                                       # 1x1 reduce + consumer BN/ReLU
    ((2, 40, 40, 7, 28, 1, 1, 1), {"residual": True, "pre": True, "pre2": True}),       # 1x1 expand, residual, 2 extras
    ((2, 40, 40, 28, 14, 1, 1, 1), {"in_halo": 1, "act": "leaky"}),
    ((2, 41, 39, 14, 14, 3, 2, 1), {"in_halo": 1}),                                     # stride 2, odd sizes
    ((2, 40, 40, 14, 14, 3, 2, 1), {"out_halo": 1}),
    ((2, 20, 20, 32, 32, 1, 1, 1), {"no_out0": True, "pre": True}),                     # widest 1x1, out1 only
    # RetinaNet's 1x1 expand as the engine launches it: residual added, raw sum not stored, both consumers' BN+ReLU
    ((2, 40, 40, 7, 28, 1, 1, 1), {"residual": True, "pre": True, "pre2": True, "no_out0": True, "aux_halo": 1}),
])
def test_conv_thin_matches_reference(built, monkeypatch, shape, kw):
    """CUDA-core kernel for very thin layers (csrc/conv_thin.cu) behind the same entry point."""
    from odt_b200 import lib as L
    monkeypatch.setenv("ODT_TC_THIN", "2")
    monkeypatch.setenv("ODT_TC_PW", "0")  # the staged pointwise kernel would take the 1x1 cases first
    before = L.load().odt_debug_thin_launches()
    got, ref, g1, r1 = _conv_case(*shape, mode="tc", seed=sum(shape), **kw)
    assert L.load().odt_debug_thin_launches() == before + 1, "the layer did not take the thin path"
    tol = 2e-3 * max(np.abs(ref).max(), 1.0)
    if not kw.get("no_out0"):
        assert np.abs(got - ref).max() <= tol, shape
    if g1 is not None:
        assert np.abs(g1 - r1).max() <= 3 * tol
