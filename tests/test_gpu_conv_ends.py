"""The two ends of the convolution stack against float64 references with per-element forward-error bounds
(tests/conv_ends_ref.py derives the bound and each path's accumulation depth):

  a. the reference and its bound, on the host: the restatement against oracle/tfops.py, an honest fp32 computation
     inside the bound, and three perturbed references (a border column read one pixel off, a filter tap dropped, two
     output channels / regrouped head columns swapped) rejected by it;
  b. the Cin = 3 stems on every path -- the packed-RGBX tensor-core stem, the fp32-gather tensor-core stem (vec2
     interior, plain interior and border gathers), the CUDA-core fp32 stems and the generic direct stem in both dtypes --
     each case with the launched kernel named by a torch.profiler trace, its output inside a sentinel-filled buffer;
  c. the fp32 head scatter into candidate rows (channel regrouping, anchor count, level offset, ragged Cout over
     32-column slices and N tiles, every conv_tc N tile width) through conv_tc and conv_direct;
  d. every network's stem and head convolutions in situ at full size, and the candidate rows of pipeline slot 1.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import conv_ends_ref as R
import prior_count_ref as PR
from gpu_harness import Guarded, kernels_launched
from gpu_harness import interior as _interior
from gpu_harness import mask as _mask
from gpu_harness import model as _model

ERR_INVALID = -1


def _lib():
    from odt_b200 import lib as L
    return L, L.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------
# a. the reference and its bound (host)
# ---------------------------------------------------------------------------------------------------------------------
def _small_stem(seed=3, f16=True, B=2, H=9, W=12, Cout=8, k=7, stride=2):
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (B, H, W, 3), generator=g).float()
    x = R.stem_operand(img, f16)
    w = (torch.randn(Cout, k, k, 3, generator=g) * (2.0 / (k * k * 3)) ** 0.5 / 64)
    w = w.half() if f16 else w
    scale = torch.rand(Cout, generator=g) + 0.5
    shift = torch.randn(Cout, generator=g) * 0.2
    return x, w, scale, shift


def _fp32_conv(x, w, stride, scale, shift, act):
    """An honest fp32 computation of the same layer (any summation order stays within gamma_K)."""
    _, H, W, _ = x.shape
    _, KR, KS, _ = w.shape
    _, pt, pb = R.same_pad(H, KR, stride)
    _, pl, pr = R.same_pad(W, KS, stride)
    t = torch.nn.functional.pad(x.float().permute(0, 3, 1, 2), (pl, pr, pt, pb))
    y = torch.nn.functional.conv2d(t, w.float().permute(0, 3, 1, 2), stride=stride).permute(0, 2, 3, 1)
    y = y * scale + shift
    if act == "relu":
        y = y.clamp_min(0)
    elif act == "leaky":
        y = torch.maximum(y, R.LEAKY * y)
    return y


@pytest.mark.parametrize("k,stride,H,W", [(7, 2, 9, 12), (7, 2, 10, 11), (3, 1, 7, 8), (5, 1, 6, 9)])
def test_restatement_matches_oracle(k, stride, H, W):
    """conv64 (TF SAME pads from engine.same_pad, asymmetric for stride 2) against oracle/tfops.conv2d_same in fp32."""
    from oracle import tfops as T
    x, w, _, _ = _small_stem(f16=False, H=H, W=W, k=k, stride=stride)
    ref = R.conv64(x, w, stride)
    ora = torch.from_numpy(np.asarray(T.conv2d_same(x.numpy(), w.permute(1, 2, 3, 0).numpy(), None, stride)))
    mag = R.conv64(x.abs(), w.abs(), stride)
    assert ref.shape == ora.shape
    assert bool(((ora.double() - ref).abs() <= R.n_acc_cuda_core(k, k, 3) * R.U32 * mag + 1e-30).all())


@pytest.mark.parametrize("act", ["relu", "leaky", None])
@pytest.mark.parametrize("f16", [True, False])
def test_bound_admits_an_honest_fp32_computation(act, f16):
    x, w, scale, shift = _small_stem(f16=f16)
    ref, mag = R.reference(x, w, 2, scale, shift, act)
    y = _fp32_conv(x, w, 2, scale, shift, act)
    n = R.n_acc_cuda_core(7, 7, 3)
    r, _ = R.worst(y, ref, mag, n, False)
    assert r <= 1.0, r
    r16, _ = R.worst(y.half(), ref, mag, n, True)
    assert r16 <= 1.0, r16


@pytest.mark.parametrize("out16", [False, True])
def test_bound_rejects_perturbed_stems(out16):
    """The three bugs the kernel checks target, planted in a seeded reference: each lands outside the bound of the
    path with the loosest accumulation term (the packed tensor-core stem)."""
    x, w, scale, shift = _small_stem()
    ref, mag = R.reference(x, w, 2, scale, shift, "relu")
    n = R.n_acc_stem_tc(7, True)
    assert R.worst(ref.float(), ref, mag, n, out16)[0] <= 1.0
    xs = x.clone()
    xs[:, :, -1] = x[:, :, -2]  # the right border column read one pixel off
    tap = w.clone()
    tap[:, 3, 0] = 0  # one filter tap dropped
    swapped = ref.clone()
    swapped[..., [2, 5]] = ref[..., [5, 2]]
    bad = {"border shifted": R.reference(xs, w, 2, scale, shift, "relu")[0],
           "tap dropped": R.reference(x, tap, 2, scale, shift, "relu")[0],
           "channels swapped": swapped}
    for what, b in bad.items():
        r, at = R.worst(b.half() if out16 else b.float(), ref, mag, n, out16)
        assert r > 1.0, "%s passes the bound (%.3g of it)" % (what, r)
        print("%s: %.3g x the bound at %s" % (what, r, at))


def test_bound_rejects_swapped_head_columns():
    """RetinaNet-style class + box heads sharing rows: two regrouped columns exchanged in the rows are caught when the
    heads are read back through the scatter restatement."""
    g = torch.Generator().manual_seed(5)
    nc, A, row, OH, OW, Cin, k = 6, 3, 10, 4, 5, 16, 3
    x = torch.randn(2, OH, OW, Cin, generator=g).half()
    heads = [(nc * A, (7, 0, nc, row, A)), (4 * A, (7, nc, 4, row, A))]
    N = 7 + OH * OW * A + 3
    rows = torch.full((2, N, row), float("nan"), dtype=torch.float64)
    refs = []
    for cout, head in heads:
        w = (torch.randn(cout, k, k, Cin, generator=g) * 0.1).half()
        ref, mag = R.reference(x, w, 1, None, torch.randn(cout, generator=g), None)
        refs.append((ref, mag, cout, head))
        sub = R.head_scatter(ref, N, row, head)
        rows = torch.where(torch.isnan(sub), rows, sub)
    own = R.head_owners(N, row, [(OH, OW, c, h) for _, _, c, h in refs])
    assert bool((own[7:7 + OH * OW * A] == 1).all()) and int(own.sum()) == OH * OW * A * row
    n = R.n_acc_conv_tc(k, k, 64)
    for ref, mag, cout, head in refs:
        assert R.worst(R.head_gather(rows, OH, OW, cout, head), ref, mag, n, False)[0] <= 1.0
    bad = rows.clone()
    bad[:, :, [1, nc + 2]] = rows[:, :, [nc + 2, 1]]  # a class column and a box column exchanged
    worst = max(R.worst(R.head_gather(bad, OH, OW, c, h), ref, mag, n, False)[0] for ref, mag, c, h in refs)
    assert worst > 1.0, worst


# ---------------------------------------------------------------------------------------------------------------------
# b. stems
# ---------------------------------------------------------------------------------------------------------------------
KERNEL = {"rgbx": "conv_stem_tc_kernel<16,7,2,true>", "tc": "conv_stem_tc_kernel<%d,%d,%d,false>",
          "cc": "conv_stem_kernel<float,%d,%d,%d>", "direct16": "conv_direct_kernel<__half,true>",
          "direct32": "conv_direct_kernel<float,true>"}


def stem_path(p, f16, rgbx):
    """The host predicates of odt_conv2d_stem_rgbx / odt_conv2d_stem (conv_stem_tc.cu, conv_direct.cu): which kernel
    a stem launch runs.  The stem cases check this against the profiler; the in-situ checks use it for n_acc."""
    if rgbx:
        return "rgbx"
    plain = (p.out0 and not p.out1 and not p.out2 and not p.residual and p.out0_group == 0 and p.R == p.S and
             p.dil == 1 and p.in_ld == 3 and p.out0_pool == 0)
    variant = (p.R, p.stride, p.Cout) in ((3, 1, 64), (3, 1, 32), (7, 2, 16))
    if f16 and plain and variant and p.out0_dtype == 0 and p.out0 % 16 == 0 and p.out0_pix_stride % 8 == 0 and \
            p.out0_pix_stride >= p.Cout and p.out0_img_stride % 8 == 0:
        return "tc"
    esz = 2 if f16 else 4
    if plain and variant and p.out0_dtype == (0 if f16 else 1) and p.out0 % 16 == 0 and \
            (p.out0_pix_stride * esz) % 16 == 0 and (p.out0_img_stride * esz) % 16 == 0:
        return "cc16" if f16 else "cc"
    return "direct16" if f16 else "direct32"


def stem_n_acc(path, k):
    if path in ("rgbx", "tc"):
        return R.n_acc_stem_tc(k, path == "rgbx")
    return R.n_acc_cuda_core(k, k, 3)


def _stem_case(path, B, H, W, Cout, k, stride, out_halo, ld, img_off=0, act="relu", seed=0, pads=None, dtype=None):
    """Builds one stem launch; returns (launch, ctx).  pads = (pad_t, pad_l) overrides the SAME pads (refusals)."""
    L, lib = _lib()
    rgbx = path == "rgbx"
    f16 = path in ("rgbx", "tc", "direct16") if dtype is None else dtype == "f16"
    dt = torch.float16 if f16 else torch.float32
    OH, pt, _ = R.same_pad(H, k, stride)
    OW, pl, _ = R.same_pad(W, k, stride)
    if pads is not None:
        pt, pl = pads
    rng = np.random.default_rng(seed)
    n = B * H * W * 3
    ibuf = torch.zeros(n + 8, dtype=torch.float32, device="cuda")
    img = ibuf[img_off:img_off + n].view(B, H, W, 3)
    img.copy_(torch.from_numpy(rng.integers(0, 256, (B, H, W, 3)).astype(np.float32)))
    cpad = 16 if rgbx else Cout
    w = torch.zeros((cpad, k, k, 3), dtype=torch.float32)
    w[:Cout] = torch.from_numpy(rng.standard_normal((Cout, k, k, 3)) * np.sqrt(2.0 / (k * k * 3)) / 64)
    wd = w.to(dt).cuda()
    sc, sh = torch.zeros(cpad), torch.zeros(cpad)
    sc[:Cout] = torch.from_numpy(rng.uniform(0.5, 1.5, Cout))
    sh[:Cout] = torch.from_numpy(rng.standard_normal(Cout) * 0.2)
    sd, hd = sc.cuda(), sh.cuda()
    h = out_halo
    out = Guarded((B, OH + 2 * h, OW + 2 * h, ld), dt)
    p = L.ConvParams()
    p.B, p.H, p.W, p.Cin, p.in_ld = B, H, W, 3, 3
    p.OH, p.OW, p.Cout = OH, OW, Cout
    p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = k, k, stride, 1, pt, pl
    p.w_ld, p.Cout_pad = 3, cpad
    p.scale, p.shift, p.act = sd.data_ptr(), hd.data_ptr(), R.ACTS[act]
    p.out0, p.out0_dtype = out.ptr(), (L.ODT_F16 if f16 else L.ODT_F32)
    p.out0_img_stride, p.out0_pix_stride = (OH + 2 * h) * (OW + 2 * h) * ld, ld
    p.out0_halo = h
    mean = (C.c_float * 3)(*R.MEAN.tolist())
    packed = None
    if rgbx:
        P = 4
        packed = torch.zeros((B, H + 2 * P, W + 2 * P, 4), dtype=torch.float16, device="cuda")
        L.check(lib.odt_pack_input_rgbx(img.data_ptr(), packed.data_ptr(), B, H, W, P, mean, _st()), "pack")
        p.in_ld, p.in_halo = 4, P
        torch.cuda.synchronize()

    def launch():
        if rgbx:
            return lib.odt_conv2d_stem_rgbx(packed.data_ptr(), wd.data_ptr(), C.byref(p), _st())
        return lib.odt_conv2d_stem(img.data_ptr(), mean, wd.data_ptr(), L.ODT_F16 if f16 else L.ODT_F32,
                                   C.byref(p), _st())

    ctx = dict(img=img, packed=packed, w=wd, scale=sd, shift=hd, out=out, p=p, f16=f16, OH=OH, OW=OW, act=act,
               keep=(ibuf, mean))
    return launch, ctx


RGBX_CASES = [
    # B, H, W, Cout, out_halo, ld    (even W: pad_l = 2 and the last 8-pixel window ends on the padded image's edge)
    (1, 2, 4, 16, 0, 16),     # M = 2: far less than one tile
    (3, 6, 2, 16, 1, 16),     # W = 2, halo output
    (3, 7, 2, 7, 0, 24),      # W = 2, odd H (pad_t = 3), 7 outputs
    (2, 64, 96, 16, 1, 64),   # whole tiles, halo, ld > 16
    (2, 65, 98, 7, 0, 64),    # odd H, ragged last tile (M % 128 = 34)
    (1, 20, 26, 16, 0, 24),   # M = 130: a 2-pixel last tile
    (1, 4, 254, 7, 1, 16),    # M = 254: a 126-pixel last tile, halo
    (3, 7, 10, 7, 1, 24),     # odd H, small, halo
    (2, 33, 48, 16, 0, 16),   # odd H, W % 4 = 0
]
GATHER_CASES = [
    # B, H, W, Cout, k, stride, out_halo, ld, img_off
    (2, 33, 47, 16, 7, 2, 1, 64, 0),   # odd W (pad_l = 3): vec2 off, the packed stem refuses it
    (2, 40, 52, 16, 7, 2, 0, 16, 1),   # even W, image base one float off: vec2 off, still 4-byte aligned
    (1, 30, 40, 16, 7, 2, 0, 24, 0),   # even W, aligned: the vec2 interior gather
    (3, 37, 53, 64, 3, 1, 1, 64, 0),   # 3x3 / 64 (SSD conv1_1), halo, ragged last tile
    (2, 16, 17, 32, 3, 1, 0, 64, 0),   # 3x3 / 32 (YOLOv3), ld > Cout
    (1, 5, 7, 64, 3, 1, 0, 64, 0),     # M = 35
    (1, 9, 11, 32, 3, 1, 1, 40, 0),    # halo, ld = 40
]
CC_CASES = [
    # B, H, W, Cout, k, stride, ld       (fp32: the CUDA-core stems)
    (2, 37, 53, 64, 3, 1, 68),
    (2, 416, 416, 32, 3, 1, 32),       # M = 346 112 > 132 * 16 * 128: the grid-stride loop iterates
    (4, 600, 600, 16, 7, 2, 16),       # M = 360 000, the 7x7 / 2 variant likewise
    (1, 33, 47, 16, 7, 2, 20),         # odd W
    (1, 5, 7, 32, 3, 1, 36),           # M = 35
]
DIRECT_CASES = [
    # B, H, W, Cout, k, stride, ld       (no specialised variant: conv_direct_kernel<T, true>)
    (2, 33, 47, 7, 7, 2, 7),           # RetinaNet basic-block stem width at odd W
    (3, 9, 10, 7, 7, 2, 9),
    (1, 20, 21, 24, 5, 1, 32),         # 5x5
    (1, 30, 40, 16, 7, 2, 18),         # a variant shape whose output rows are not whole 16-byte sectors
]

STEM_PARAMS = ([pytest.param("rgbx", c[0], c[1], c[2], c[3], 7, 2, c[4], c[5], 0, id="rgbx-%dx%dx%d-c%d-h%d-ld%d" % c)
                for c in RGBX_CASES] +
               [pytest.param("tc", *c, id="tc-%dx%dx%d-c%d-k%d-s%d-h%d-ld%d-off%d" % c) for c in GATHER_CASES] +
               [pytest.param("cc", *c[:6], 0, c[6], 0, id="cc-%dx%dx%d-c%d-k%d-s%d-ld%d" % c) for c in CC_CASES] +
               [pytest.param(d, *c[:6], 0, c[6], 0, id="%s-%dx%dx%d-c%d-k%d-s%d-ld%d" % ((d,) + c))
                for d in ("direct16", "direct32") for c in DIRECT_CASES])


@pytest.mark.gpu
@pytest.mark.parametrize("path,B,H,W,Cout,k,stride,out_halo,ld,img_off", STEM_PARAMS)
def test_stem_paths(built, path, B, H, W, Cout, k, stride, out_halo, ld, img_off):
    launch, c = _stem_case(path, B, H, W, Cout, k, stride, out_halo, ld, img_off, act="relu", seed=B * H + W + Cout)
    p, out = c["p"], c["out"]
    rc, names = kernels_launched(launch)
    from odt_b200 import lib as L
    L.check(rc, "stem %s" % path)
    exp = KERNEL[path] if path in ("rgbx", "direct16", "direct32") else KERNEL[path] % (Cout, k, stride)
    convs = [n for n in names if "conv" in n]
    assert len(convs) == 1 and exp in convs[0], (exp, names)
    assert stem_path(p, c["f16"], path == "rgbx") == path
    if path == "tc":
        vec2 = W % 2 == 0 and p.pad_l % 2 == 0 and c["img"].data_ptr() % 8 == 0
        print("fp32-gather stem: vec2 interior gather %s" % ("on" if vec2 else "off"))
    if path == "rgbx":  # the packed operand is the reference operand, bit for bit, with a zero border and X lane
        P = 4
        pk = c["packed"]
        assert torch.equal(pk[:, P:P + H, P:P + W, :3], R.stem_operand(c["img"], True))
        assert not bool(pk[..., 3].ne(0).any())
        assert not bool(pk[:, :P].ne(0).any()) and not bool(pk[:, P + H:].ne(0).any())
        assert not bool(pk[:, :, :P].ne(0).any()) and not bool(pk[:, :, P + W:].ne(0).any())
    out.assert_outside_untouched()
    t = out.t
    stored = 16 if path == "rgbx" else Cout
    out.assert_untouched(_mask(t.shape, out_halo), "halo")
    if ld > stored:
        out.assert_untouched(_mask(t.shape, 0, stored), "channel >= %d" % stored)
    if path == "rgbx" and Cout < 16:
        assert not bool(_interior(t, out_halo)[..., Cout:16].ne(0).any()), "pad lanes [Cout, 16) must hold zeros"
    x = R.stem_operand(c["img"], path in ("rgbx", "tc"))
    got = _interior(t, out_halo)
    r, at = R.checked(lambda b0, b1: got[b0:b1, ..., :Cout], x, c["w"][:Cout], stride, c["scale"][:Cout],
                      c["shift"][:Cout], "relu", stem_n_acc(path, k), c["f16"], chunk=2)
    print("%s stem B=%d %dx%d Cout %d: worst error %.3g of the bound (at %s)" % (path, B, H, W, Cout, r, at))
    assert r <= 1.0, (r, at)


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["leaky", None])
@pytest.mark.parametrize("path", ["rgbx", "tc", "cc"])
def test_stem_activations(built, path, act):
    """The other two activations on the specialised stems (the networks use ReLU; the epilogue takes all three)."""
    k, s, Cout = (7, 2, 16) if path != "cc" else (3, 1, 32)
    launch, c = _stem_case(path, 2, 31, 44, Cout, k, s, 0, Cout if path != "rgbx" else 16, act=act, seed=11)
    from odt_b200 import lib as L
    L.check(launch(), "stem")
    torch.cuda.synchronize()
    x = R.stem_operand(c["img"], path != "cc")
    r, at = R.checked(lambda b0, b1: c["out"].t[b0:b1, ..., :Cout], x, c["w"][:Cout], s, c["scale"][:Cout],
                      c["shift"][:Cout], act, stem_n_acc(path, k), c["f16"])
    assert r <= 1.0, (r, at)


REFUSALS = {
    # name: (path, B, H, W, Cout, k, stride, out_halo, ld, pads)
    "rgbx-odd-W": ("rgbx", 1, 32, 47, 16, 7, 2, 0, 16, None),
    "rgbx-odd-pad_l": ("rgbx", 1, 32, 48, 16, 7, 2, 0, 16, (2, 3)),
    "rgbx-pad_t-5": ("rgbx", 1, 32, 48, 16, 7, 2, 0, 16, (5, 2)),
    "rgbx-pad_l-6": ("rgbx", 1, 32, 48, 16, 7, 2, 0, 16, (2, 6)),
    "rgbx-3x3": ("rgbx", 1, 32, 48, 16, 3, 1, 0, 16, None),
    "stem-f32-halo": ("cc", 1, 32, 48, 16, 7, 2, 1, 16, None),
    "stem-f32-halo-3x3": ("cc", 1, 20, 20, 64, 3, 1, 1, 64, None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFUSALS))
def test_stem_refusals(built, name):
    """Shapes the packed stem does not take return ODT_ERR_UNSUPPORTED, and odt_conv2d_stem rejects a halo output on
    the fp32 path; neither launches anything or touches the output."""
    from odt_b200 import lib as L
    path, B, H, W, Cout, k, s, h, ld, pads = REFUSALS[name]
    launch, c = _stem_case(path, B, H, W, Cout, k, s, h, ld, pads=pads)
    rc, names = kernels_launched(launch)
    assert rc == (L.ERR_UNSUPPORTED if path == "rgbx" else ERR_INVALID), rc
    assert not names, names
    out = c["out"]
    out.assert_outside_untouched()
    out.assert_untouched(torch.ones(out.t.shape, dtype=torch.bool, device="cuda"), "refused output")


# ---------------------------------------------------------------------------------------------------------------------
# c. head scatter, unit level
# ---------------------------------------------------------------------------------------------------------------------
# heads: (Cout, col, group, gstride) sharing the anchor count A and the row length; bn: conv_tc's N tile per head in
# im2col mode (odt_conv_tc_pick_bn), "flat" for the halo-flat mode (N tile = Cout_pad)
HEAD_CASES = {
    # RetinaNet's class + box pair at nc = 20: class group 20 / stride 24, box group 4 at column 20; 3 N tiles of 96
    # for the class head (the last one ragged), 2 of 32 for the box head
    "retina-pair": dict(B=4, H=40, W=40, Cin=64, k=3, A=9, row=24, lvl_off=0, n_after=0, in_halo=0, act=None,
                        heads=[(180, 0, 20, 24), (36, 20, 4, 24)], bn=[96, 32]),
    # the same pair fed by a halo'd pre-activation: the class head in im2col mode, the box head halo-flat; a later level
    "retina-pair-halo": dict(B=2, H=20, W=20, Cin=64, k=3, A=9, row=24, lvl_off=57, n_after=13, in_halo=1, act=None,
                             heads=[(180, 0, 20, 24), (36, 20, 4, 24)], bn=[32, "flat"]),
    # a group that does not divide 32 (and its partner of 2 columns)
    "group-7": dict(B=4, H=57, W=57, Cin=64, k=3, A=5, row=9, lvl_off=0, n_after=5, in_halo=0, act=None,
                    heads=[(35, 0, 7, 9), (10, 7, 2, 9)], bn=[64, 32]),
    # a group wider than one 32-column slice, leaky activation, 128-wide N tile
    "group-40": dict(B=4, H=57, W=57, Cin=64, k=3, A=3, row=45, lvl_off=11, n_after=0, in_halo=0, act="leaky",
                     heads=[(120, 0, 40, 45), (15, 40, 5, 45)], bn=[128, 32]),
    # YOLOv3 at 80 classes: a 255-channel 1x1 head with BN + leaky, Cout_pad 256 on the wide 128 x 256 tile, a later level
    "yolo80-wide": dict(B=32, H=13, W=13, Cin=128, k=1, A=3, row=85, lvl_off=300, n_after=40, in_halo=0, act="leaky",
                        heads=[(255, 0, 0, 0)], bn=[256]),
    # FCOS: class, centre-ness and box heads of one level (A = 1), halo-flat, a later level
    "fcos-triple": dict(B=2, H=24, W=24, Cin=64, k=3, A=1, row=25, lvl_off=37, n_after=11, in_halo=1, act=None,
                        heads=[(20, 0, 0, 0), (1, 20, 0, 0), (4, 21, 0, 0)], bn=["flat", "flat", "flat"]),
}


def _cout_pad(cout):
    return (cout + 31) // 32 * 32


def _tile_width(lib, case, cout):
    c = case
    M = c["B"] * c["H"] * c["W"]
    ld = (c["Cin"] + 63) // 64 * 64
    return lib.odt_conv_tc_pick_bn(_cout_pad(cout), M, c["k"] * c["k"] * ld // 64)


def test_head_cases_cover_every_tile_width(built):
    """The N tile each head case runs on conv_tc, from the library's own planner; together the cases take every width."""
    _, lib = _lib()
    seen = set()
    for name, c in HEAD_CASES.items():
        for (cout, _, _, _), bn in zip(c["heads"], c["bn"]):
            flat = c["in_halo"] and c["k"] == 3 and _cout_pad(cout) <= 128
            assert (bn == "flat") == bool(flat), (name, cout)
            if not flat:
                assert _tile_width(lib, c, cout) == bn, (name, cout, _tile_width(lib, c, cout))
            seen.add(_cout_pad(cout) if flat else bn)
    assert {32, 64, 96, 128, 256} <= seen, seen


def _head_run(mode, case, seed=0):
    """Runs the case's heads into one NaN-filled candidate-row buffer; returns (rows, x, per-head (w, scale, shift,
    cout, head), names of the kernels launched)."""
    L, lib = _lib()
    c = case
    B, H, W, Cin, k, A, row = c["B"], c["H"], c["W"], c["Cin"], c["k"], c["A"], c["row"]
    tc = mode == "tc"
    h = c["in_halo"] if tc else 0
    dt = torch.float32 if mode == "direct32" else torch.float16
    OH, pt, _ = R.same_pad(H, k, 1)
    OW, pl, _ = R.same_pad(W, k, 1)
    N = c["lvl_off"] + OH * OW * A + c["n_after"]
    rng = np.random.default_rng(seed)
    ld = (Cin + 63) // 64 * 64 if tc else Cin
    x = torch.zeros((B, H + 2 * h, W + 2 * h, ld), dtype=dt, device="cuda")
    x[:, h:h + H, h:h + W, :Cin] = torch.from_numpy(rng.standard_normal((B, H, W, Cin)).astype(np.float32)).cuda()
    rows = torch.full((B, N, row), float("nan"), dtype=torch.float32, device="cuda")
    heads, keep = [], []
    for cout, col, group, gstride in c["heads"]:
        cpad = _cout_pad(cout) if tc else cout
        w = torch.zeros((cpad, k, k, ld), dtype=torch.float32)
        w[:cout, :, :, :Cin] = torch.from_numpy(rng.standard_normal((cout, k, k, Cin)) * np.sqrt(2.0 / (k * k * Cin)))
        wd = w.to(dt).cuda()
        sd = torch.from_numpy(rng.uniform(0.5, 1.5, cout).astype(np.float32)).cuda()
        hd = torch.from_numpy((rng.standard_normal(cout) * 0.2).astype(np.float32)).cuda()
        head = (c["lvl_off"], col, group, gstride, A)
        p = L.ConvParams()
        p.B, p.H, p.W, p.Cin, p.in_ld = B, H, W, Cin, ld
        p.OH, p.OW, p.Cout = OH, OW, cout
        p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = k, k, 1, 1, pt, pl
        p.w_ld, p.Cout_pad = ld, cpad
        p.scale, p.shift, p.act = sd.data_ptr(), hd.data_ptr(), R.ACTS[c["act"]]
        p.out0 = rows.data_ptr() + 4 * (c["lvl_off"] * row + col)
        p.out0_dtype = L.ODT_F32
        p.out0_img_stride, p.out0_pix_stride = N * row, A * row
        p.out0_group, p.out0_group_stride = group, gstride
        p.in_halo = h
        keep.append(p)
        heads.append((wd, sd, hd, cout, head))
    names = []
    for p, (wd, _, _, _, _) in zip(keep, heads):
        if tc:
            rc, nm = kernels_launched(lambda: lib.odt_conv2d_f16_tc(x.data_ptr(), wd.data_ptr(), C.byref(p), _st()))
        else:
            code = L.ODT_F16 if dt == torch.float16 else L.ODT_F32
            rc, nm = kernels_launched(
                lambda: lib.odt_conv2d_direct(x.data_ptr(), wd.data_ptr(), code, C.byref(p), _st()))
        L.check(rc, "head conv")
        names.append(nm)
    torch.cuda.synchronize()
    return rows, _interior(x, h)[..., :Cin], heads, names, (OH, OW, N, row, tc, ld)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tc", "direct16", "direct32"])
@pytest.mark.parametrize("name", list(HEAD_CASES))
def test_head_scatter(built, mode, name):
    case = HEAD_CASES[name]
    rows, x, heads, names, (OH, OW, N, row, tc, ld) = _head_run(mode, case, seed=len(name))
    k = case["k"]
    for (wd, sd, hd, cout, head), nm, bn in zip(heads, names, case["bn"]):
        if tc:
            width = _cout_pad(cout) if bn == "flat" else bn
            exp = "conv_tc_kernel<%d,false>" % width
        else:
            exp = "conv_direct_kernel<%s,false>" % ("float" if mode == "direct32" else "__half")
        assert len(nm) == 1 and exp in nm[0], (exp, nm)
        n_acc = R.n_acc_conv_tc(k, k, ld) if tc else R.n_acc_cuda_core(k, k, case["Cin"])
        r, at = R.checked(lambda b0, b1: R.head_gather(rows, OH, OW, cout, head, b0, b1), x, wd[:cout, :, :, :x.shape[-1]],
                          1, sd, hd, case["act"], n_acc, False, chunk=8)
        print("%s %s head Cout %d group %d: worst error %.3g of the bound (at %s)" % (name, mode, cout, head[2], r, at))
        assert r <= 1.0, (cout, r, at)
    own = R.head_owners(N, row, [(OH, OW, h[3], h[4]) for h in heads], device="cuda")
    assert int(own.max()) == 1, "two heads write one element"
    nan = torch.isnan(rows)
    assert torch.equal(nan, (own == 0).expand_as(rows)), "a written element outside the heads, or a head element unwritten"
    lvl = slice(case["lvl_off"], case["lvl_off"] + OH * OW * case["A"])
    if name != "yolo80-wide":  # the case's heads share every row of their level
        assert bool((own[lvl] == 1).all()), "the heads do not fill every column of their rows exactly once"


# ---------------------------------------------------------------------------------------------------------------------
# d. in situ at full size
# ---------------------------------------------------------------------------------------------------------------------
def _op_operands(op, net):
    """(weights [Cout,R,S,Cin], scale or None, shift) the kernel multiplies, cut to the real channels."""
    cin = 3 if op.is_image else op.x.C
    w = op.wdev[:op.cout, :, :, :cin]
    sc = op.scale[:op.cout] if op.scale is not None else None
    return w, sc, op.shift[:op.cout]


def _insitu_stem(net, op):
    f16 = net.precision == "fp16"
    p = op.p
    path = stem_path(p, f16, bool(op.rgbx))
    if op.y is None or op.y.buf is None:
        return None
    x = R.stem_operand(net.image_buf, path in ("rgbx", "tc"))
    if op.rgbx:
        P = op.rgbx
        pk = net.image_rgbx
        assert torch.equal(pk[:, P:P + net.in_h, P:P + net.in_w, :3], x.half()), "packed image"
        assert not bool(pk[..., 3].ne(0).any()), "packed image X lane"
    w, sc, sh = _op_operands(op, net)
    y = op.y
    got = _interior(y.buf, y.halo)
    if y.halo:
        assert not bool(y.buf[_mask(y.buf.shape, 1)].ne(0).any()), "stem halo written"
    if y.ld > op.cout:
        assert not bool(got[..., op.cout:].ne(0).any()), "stem channels >= Cout written"
    r, at = R.checked(lambda b0, b1: got[b0:b1, ..., :op.cout], x, w, op.stride, sc, sh, op.act, stem_n_acc(path, op.k),
                      f16, chunk=8)
    return path, r, at


def _insitu_head(net, op):
    x = op.x
    xin = _interior(x.buf, x.halo)[..., :x.C]
    w, sc, sh = _op_operands(op, net)
    p = op.p
    n_acc = R.n_acc_conv_tc(op.k, op.k, x.ld) if op.use_tc else R.n_acc_cuda_core(op.k, op.k, x.C)
    r, at = R.checked(lambda b0, b1: R.head_gather(net.head_buf, p.OH, p.OW, op.cout, op.head, b0, b1), xin, w,
                      op.stride, sc, sh, op.act, n_acc, False, chunk=4, dil=op.dil)
    return ("conv_tc" if op.use_tc else "conv_direct"), r, at


INSITU = [("ssd300", "fp16", 64, {}), ("ssd512", "fp16", 8, {}),
          ("retinanet", "fp16", 16, {"data_shape": [800, 800, 3]}),
          ("retinanet", "fp16", 16, {"data_shape": [800, 800, 3], "is_bottleneck": False, "init_conv_filters": 7,
                                     "residual_block_list": [2, 2, 2, 2]}),
          ("yolov3", "fp16", 32, {"data_shape": [416, 416, 3], "num_classes": 20}),
          ("yolov3", "fp16", 32, {"data_shape": [416, 416, 3], "num_classes": 80}),
          ("fcos", "fp16", 4, {"data_shape": [1024, 1024, 3]}),
          ("fcos", "fp32", 4, {"data_shape": [1024, 1024, 3]}),
          ("retinanet", "fp32", 2, {"data_shape": [512, 512, 3]}),
          ("yolov2", "fp16", 64, {}), ("yolov2", "fp16", 8, {"size": 200}),
          # the widest head the code accepts (9 priors x 133 = 1197 channels) and the narrowest (6)
          ("yolov2", "fp16", 8, {"A": 9, "nc": 128}), ("yolov2", "fp16", 8, {"A": 1, "nc": 1}),
          ("yolov3", "fp16", 8, {"data_shape": [416, 416, 3], "num_classes": 128, "num_priors": 9,
                                 "priors": PR.priors_for(9)}),
          ("yolov3", "fp16", 8, {"data_shape": [416, 416, 3], "num_classes": 1, "num_priors": 1,
                                 "priors": PR.priors_for(1)})]
INSITU_IDS = ["ssd300-fp16-B64", "ssd512-fp16-B8", "retinanet800-fp16-B16", "retinanet800-basic-fp16-B16",
              "yolov3-416-nc20-fp16-B32", "yolov3-416-nc80-fp16-B32", "fcos1024-fp16-B4", "fcos1024-fp32-B4",
              "retinanet512-fp32-B2", "yolov2-480-fp16-B64", "yolov2-200-fp16-B8", "yolov2-480-A9-nc128-fp16-B8",
              "yolov2-480-A1-nc1-fp16-B8", "yolov3-416-A9-nc128-fp16-B8", "yolov3-416-A1-nc1-fp16-B8"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,precision,B,over", INSITU, ids=INSITU_IDS)
def test_conv_ends_in_situ(built, kind, precision, B, over):
    """The stem and every head convolution of the network at its full per-GPU geometry, checked on the actual buffers
    after one eager forward (every activation owns its buffer, so all of them are live), with the candidate rows
    NaN-filled beforehand: each head's columns against the float64 reference of its real input, and the heads' columns
    partition every row.  The float64 convolutions run a few images at a time."""
    from odt_b200 import engine as E
    m = _model(kind, precision, **over)
    net = m.engine(B, graph=False)
    img = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (B, net.in_h, net.in_w, 3)).astype(np.float32))
    net.image_buf.copy_(img)
    net.head_buf.fill_(float("nan"))
    net.forward(with_tail=False)
    torch.cuda.synchronize()
    stems = [op for op in net.ops if isinstance(op, E.ConvOp) and op.is_image]
    heads = [op for op in net.ops if isinstance(op, E.ConvOp) and op.head is not None]
    assert len(stems) == 1 and heads
    tag = "%s %s B=%d" % (kind, precision, B)
    res = _insitu_stem(net, stems[0])
    assert res is not None, "the stem output is not materialised"
    path, r, at = res
    print("%s stem (%s, Cout %d): worst error %.3g of the bound (at %s)" % (tag, path, stems[0].cout, r, at))
    assert r <= 1.0, ("stem", path, r, at)
    worst = 0.0
    for op in heads:
        path, r, at = _insitu_head(net, op)
        worst = max(worst, r)
        print("%s head %s (%s, Cout %d, head %s): worst error %.3g of the bound (at %s)" % (
            tag, op.kernel, path, op.cout, op.head, r, at))
        assert r <= 1.0, (op.kernel, r, at)
    row = net.tail.row
    own = R.head_owners(net.N, row, [(op.p.OH, op.p.OW, op.cout, op.head) for op in heads], device="cuda")
    assert bool((own == 1).all()), "the heads' columns do not partition the candidate rows"
    assert not bool(torch.isnan(net.head_buf).any()), "a candidate-row element left unwritten"
    print("%s: %d head convolutions, worst %.3g of the bound" % (tag, len(heads), worst))
    del net, m
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# e. pipeline slot 1
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind,over", [("retinanet", {}), ("fcos", {})])
def test_pipeline_slot1_head_params(built, kind, over):
    """After capture_pipelined(), each head's slot-1 parameter block equals slot 0's byte for byte except out0, which
    moves by the distance between the two candidate-row buffers; replaying slot 1's body on the same images fills
    head_buf1 bit-identically to slot 0's head_buf."""
    from odt_b200 import engine as E
    m = _model(kind, "fp16", **over)
    net = m.engine(2, graph=False)
    img = torch.from_numpy(np.random.default_rng(4).integers(0, 256, (2, net.in_h, net.in_w, 3)).astype(np.float32))
    net.image_buf.copy_(img)
    net.capture_pipelined()
    delta = net.head_buf1.data_ptr() - net.head_buf.data_ptr()
    heads = [op for op in net.ops if isinstance(op, E.ConvOp) and op.head is not None]
    assert heads
    n = C.sizeof(heads[0].p)
    for op in heads:
        assert op.p1.out0 - op.p.out0 == delta
        q = type(op.p)()
        C.memmove(C.byref(q), C.byref(op.p1), n)
        q.out0 = op.p.out0
        assert C.string_at(C.addressof(q), n) == C.string_at(C.addressof(op.p), n), op.kernel
        assert op.params(net) is op.p  # slot 0 outside the pipeline
    net.head_buf.fill_(float("nan"))
    net.head_buf1.fill_(float("nan"))
    torch.cuda.synchronize()
    net.body_graphs[0].replay()
    torch.cuda.synchronize()
    rows0 = net.head_buf.clone()
    assert not bool(torch.isnan(rows0).any())
    assert bool(torch.isnan(net.head_buf1).all()), "slot 0's body wrote slot 1's rows"
    net.body_graphs[1].replay()
    torch.cuda.synchronize()
    assert torch.equal(net.head_buf1, rows0), "slot 1's rows differ from slot 0's"
    assert torch.equal(net.head_buf, rows0), "slot 1's body wrote slot 0's rows"
    del net, m
    torch.cuda.empty_cache()
