"""The body convolutions -- every layer between the stem and the heads -- against float64 references with per-element
forward-error bounds (tests/conv_ends_ref.py derives them; tests/test_gpu_conv.py's _conv_case applies them together
with the write rules of a sentinel-guarded buffer):

  a. the bound on the host: an honest fp32 computation of a residual / pooled / out1 layer passes it, and five planted
     bugs are rejected by it (a pooling window one column off, a residual read one pixel off, the last 16 channels of
     the final K chunk dropped, a tile's pixel taken from the next image, taps-as-N's left and right partials swapped);
  b. dispatch coverage: a case table whose launches name every body-convolution kernel instantiation compiled into
     the library, each case at a named edge;
  c. out1 / out2 do not depend on whether out0 is stored, on every path that takes extra outputs;
  d. every body convolution of each network in situ at full size after one eager forward.  The float64 reference
     runs on images {0, B/2, B-1} of each layer, which keeps the file's run time to minutes at the full batches.
"""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_ends_ref as R
from gpu_harness import interior, last_conv_kernel, mask
from gpu_harness import model as _model


# ---------------------------------------------------------------------------------------------------------------------
# a. the bound (host)
# ---------------------------------------------------------------------------------------------------------------------
def _layer(seed=3, B=2, H=8, W=10, Cin=48, Cout=24, k=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g).half()
    w = (torch.randn(Cout, k, k, Cin, generator=g) * (2.0 / (k * k * Cin)) ** 0.5).half()
    scale = torch.rand(Cout, generator=g) + 0.5
    shift = torch.randn(Cout, generator=g) * 0.2
    res = torch.randn(B, H, W, Cout, generator=g).half()
    s2, h2 = torch.rand(Cout, generator=g) + 0.5, torch.randn(Cout, generator=g) * 0.2
    return x, w, scale, shift, res, s2, h2


def _fp32_conv(x, w, scale, shift, act):
    t = F.pad(x.float().permute(0, 3, 1, 2), (1, 1, 1, 1))
    y = F.conv2d(t, w.float().permute(0, 3, 1, 2)).permute(0, 2, 3, 1) * scale + shift
    return y.clamp_min(0) if act == "relu" else (torch.maximum(y, R.LEAKY * y) if act == "leaky" else y)


N_ACC = R.n_acc_conv_tc(3, 3, 64)


@pytest.mark.parametrize("act", ["relu", "leaky", None])
def test_body_bound_admits_an_honest_fp32_computation(act):
    x, w, scale, shift, res, s2, h2 = _layer()
    ref, mag = R.reference(x, w, 1, scale, shift, act)
    v = ref + res.double()
    b0 = R.bound(v, mag, N_ACC, True, res)
    v16 = (_fp32_conv(x, w, scale, shift, act) + res.float()).half()
    assert R.ratio(v16, v, b0)[0] <= 1.0
    assert R.ratio(R.pool2(v16), R.pool2(v), R.pool2(b0))[0] <= 1.0
    o1 = torch.relu(v16.float() * s2 + h2).half()
    t = R.consumer(v, s2, h2, "relu")
    assert R.ratio(o1, t, R.bound_through(t, b0, s2, True))[0] <= 1.0
    t_own = R.consumer(v16, s2, h2, "relu")
    assert R.ratio(o1, t_own, R.bound_own(t_own, True))[0] <= 1.0


def test_body_bound_rejects_planted_bugs():
    x, w, scale, shift, res, _, _ = _layer()
    B, H, W, Cout = res.shape
    ref, mag = R.reference(x, w, 1, scale, shift, "relu")
    v = ref + res.double()
    b0 = R.bound(v, mag, N_ACC, True, res)
    bad = {}
    # a pooling window one column off
    vs = torch.cat([v[:, :, 1:], v[:, :, -1:]], dim=2)
    bad["pool window one column off"] = (R.pool2(vs), R.pool2(v), R.pool2(b0))
    # the residual read one pixel off: its halo row length W + 2 taken as W
    rp = F.pad(res.float().permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1).reshape(B, -1, Cout)
    oy, ox = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    rbad = rp[:, ((oy + 1) * W + ox + 1).reshape(-1)].reshape(B, H, W, Cout)
    bad["residual row length W"] = (ref + rbad.double(), v, b0)
    # the last 16 channels of the final K chunk dropped (Cin = 48: klast = 3 k16 steps)
    wk = w.clone()
    wk[..., 32:48] = 0
    bad["klast step dropped"] = (R.reference(x, wk, 1, scale, shift, "relu")[0] + res.double(), v, b0)
    # a tile's pixel taken from the next image
    vt = v.clone()
    vt[0, -1, -1] = v[1, -1, -1]
    bad["pixel from the next image"] = (vt, v, b0)
    # taps-as-N: the left and right tap partials swapped
    wf = w.flip(2)
    bad["tap partials swapped"] = (R.reference(x, wf, 1, scale, shift, "relu")[0] + res.double(), v, b0)
    for what, (got, want, b) in bad.items():
        r, at = R.ratio(got.half(), want, b)
        print("%s: %.3g x the bound at %s" % (what, r, at))
        assert r > 1.0, "%s passes the bound (%.3g of it)" % (what, r)


def test_n_acc_per_path():
    assert R.n_acc_body("conv_tc_kernel<128,true>", 3, 3, 100, 128) == 3 * 9 * 128
    assert R.n_acc_body("conv_tc_swap_kernel", 3, 3, 64, 64) == 3 * 9 * 64
    assert R.n_acc_body("conv_tapn_kernel<32,1>", 3, 3, 16, 64) == 3 * 9 * 64
    for k in ("conv_pw_kernel<8>", "conv_thin_kernel<3,1,1>", "conv_direct_kernel<float,false>"):
        assert R.n_acc_body(k, 3, 3, 7, 64) == 9 * 7 + 1


# ---------------------------------------------------------------------------------------------------------------------
# b. dispatch coverage
# ---------------------------------------------------------------------------------------------------------------------
TC = "conv_tc_kernel<%d,%s>"
THIN = "conv_thin_kernel<%d,%d,%d>"
PIN_TC = {"ODT_TC_TAPN": "0", "ODT_TC_SWAP": "0"}
PIN_SWAP = {"ODT_TC_TAPN": "0", "ODT_TC_SWAP": "2"}
PIN_THIN = {"ODT_TC_THIN": "2", "ODT_TC_PW": "0"}
# id: ((B, H, W, Cin, Cout, k, stride, dil), _conv_case keywords, environment, launched kernel)
BODY_CASES = {
    # conv_tc im2col, TMA-store epilogue (fp16 out0 alone), each N tile width from the planner
    "tc32-tma-ragged-cout-in-slice": ((2, 19, 19, 64, 20, 3, 1, 1), {}, {}, TC % (32, "true")),
    "tc64-tma-odd-tile-count": ((8, 38, 38, 64, 64, 3, 1, 1), {"act": "leaky"}, {}, TC % (64, "true")),
    "tc96-tma-1x1": ((4, 38, 38, 256, 96, 1, 1, 1), {"act": None}, {}, TC % (96, "true")),
    "tc128-tma-ragged-cout-in-tile": ((8, 38, 38, 64, 100, 3, 1, 1), {}, {}, TC % (128, "true")),
    "tc256-tma-rounds": ((4, 38, 38, 64, 256, 3, 1, 1), {}, {}, TC % (256, "true")),
    # the staged epilogue: residual / extra outputs / output halo
    "tc32-staged-residual-klast1": ((2, 19, 19, 16, 20, 3, 1, 1), {"residual": True}, {}, TC % (32, "false")),
    "tc64-staged-flat-out-halo": ((8, 38, 38, 64, 64, 3, 1, 1), {"in_halo": 1, "out_halo": 1, "pre": True},
                                  {"ODT_TC_TAPN": "0"}, TC % (64, "false")),
    "tc96-staged-pre": ((4, 38, 38, 256, 96, 1, 1, 1), {"pre": True, "act": "leaky"}, {}, TC % (96, "false")),
    "tc128-staged-res-out1-out2": ((8, 38, 38, 64, 120, 3, 1, 1), {"residual": True, "pre": True, "pre2": True}, {},
                                   TC % (128, "false")),
    "tc256-staged-residual-klast3": ((4, 38, 38, 100, 256, 3, 1, 1), {"residual": True}, {}, TC % (256, "false")),
    # conv_tc edges
    "tc-stride2-odd": ((3, 37, 41, 128, 256, 3, 2, 1), {"act": "leaky"}, {}, None),
    "tc-conv6-dilation": ((2, 19, 19, 512, 1024, 3, 1, 2), {}, {}, None),
    "tc-1x1-stride2-shortcut": ((2, 38, 38, 256, 512, 1, 2, 1), {"act": None}, {}, None),
    "tc-im2col-in-halo": ((2, 19, 19, 256, 512, 3, 2, 1), {"in_halo": 1}, {}, None),
    "tc-im2col-out-halo": ((2, 26, 26, 128, 64, 1, 1, 1), {"in_halo": 1, "out_halo": 1}, {}, None),
    "tc-klast2-wraps-images": ((3, 75, 75, 40, 64, 3, 2, 1), {}, {}, None),
    "tc-flat-halo": ((3, 75, 75, 64, 128, 3, 1, 1), {"in_halo": 1, "out_halo": 1}, PIN_TC, None),
    "tc-flat-bres": ((1, 150, 150, 128, 128, 3, 1, 1), {"in_halo": 1, "out_halo": 1}, PIN_TC, None),
    "tc-rowblock-rp2": ((2, 300, 300, 64, 64, 3, 1, 1), {"in_halo": 1, "out_halo": 1, "pool": 2}, PIN_TC, None),
    "tc-rowblock-rp4": ((2, 150, 150, 128, 128, 3, 1, 1), {"in_halo": 1, "pool": 2}, PIN_TC, None),
    "tc-res-out1-out2-no-out0-halo": ((2, 26, 26, 512, 28, 1, 1, 1),
                                      {"residual": True, "pre": True, "pre2": True, "no_out0": True, "aux_halo": 1},
                                      {"ODT_TC_PW": "0", "ODT_TC_THIN": "0"}, None),
    # the generic fp16 column path: out0 one element off 16-byte alignment, or out1 alone misaligned
    "tc-generic-f16-out0-off": ((2, 19, 19, 128, 60, 3, 1, 1), {"residual": True, "pre": True, "off": 1}, {},
                                TC % (32, "false")),
    "tc-generic-f16-no-out0": ((2, 19, 19, 128, 60, 3, 1, 1), {"pre": True, "pre2": True, "no_out0": True,
                                                               "off": 1, "aux_halo": 1}, {}, TC % (32, "false")),
    # transposed tiles: halo-flat (resident and streamed filter bank) and row-block RP 8 / 4 / 2
    "swap-flat-resident": ((1, 16, 16, 64, 64, 3, 1, 1), {"in_halo": 1, "out_halo": 1}, PIN_SWAP,
                           "conv_tc_swap_kernel"),
    "swap-flat-streamed-second-half": ((3, 21, 23, 128, 100, 3, 1, 1), {"in_halo": 1, "out_halo": 1}, PIN_SWAP,
                                       "conv_tc_swap_kernel"),
    "swap-rp8": ((1, 8, 32, 64, 64, 3, 1, 1), {"in_halo": 1, "out_halo": 1, "pool": 2}, PIN_SWAP,
                 "conv_tc_swap_kernel"),
    "swap-rp4": ((1, 300, 300, 64, 64, 3, 1, 1), {"in_halo": 1, "pool": 2, "act": "leaky"}, PIN_SWAP,
                 "conv_tc_swap_kernel"),
    "swap-rp2": ((2, 2, 300, 64, 128, 3, 1, 1), {"in_halo": 1, "out_halo": 1, "pool": 2, "act": None}, PIN_SWAP,
                 "conv_tc_swap_kernel"),
    # taps as N
    "tapn32": ((2, 40, 40, 28, 28, 3, 1, 1), {"in_halo": 1, "residual": True, "pre": True, "pre2": True},
               {"ODT_TC_TAPN": "2"}, "conv_tapn_kernel<32,0>"),
    "tapn32-pool": ((2, 30, 46, 16, 28, 3, 1, 1), {"in_halo": 1, "pool": 2}, {"ODT_TC_TAPN": "2"},
                    "conv_tapn_kernel<32,1>"),
    "tapn64": ((2, 37, 61, 64, 64, 3, 1, 1), {"in_halo": 1, "out_halo": 1, "act": "leaky"}, {"ODT_TC_TAPN": "2"},
               "conv_tapn_kernel<64,0>"),
    "tapn64-pool": ((1, 8, 300, 64, 64, 3, 1, 1), {"in_halo": 1, "out_halo": 1, "pool": 2}, {"ODT_TC_TAPN": "2"},
                    "conv_tapn_kernel<64,1>"),
    # pointwise, each COT
    "pw8": ((2, 40, 40, 16, 7, 1, 1, 1), {"pre": True}, {"ODT_TC_PW": "2"}, "conv_pw_kernel<8>"),
    "pw16": ((2, 33, 35, 28, 14, 1, 1, 1), {"residual": True, "pre": True, "pre2": True, "no_out0": True,
                                            "aux_halo": 1}, {"ODT_TC_PW": "2"}, "conv_pw_kernel<16>"),
    "pw32": ((2, 25, 25, 28, 112, 1, 1, 1), {"residual": True, "pre": True, "act": None}, {"ODT_TC_PW": "2"},
             "conv_pw_kernel<32>"),
    # thin: every instantiation of ODT_THIN_DISPATCH
    "thin-1x1-8-8": ((2, 40, 40, 7, 7, 1, 1, 1), {"pre": True}, PIN_THIN, THIN % (1, 1, 1)),
    "thin-1x1-8-16": ((2, 41, 39, 8, 14, 1, 2, 1), {"act": "leaky"}, PIN_THIN, THIN % (1, 1, 2)),
    "thin-1x1-8-32": ((2, 40, 40, 7, 28, 1, 1, 1), {"residual": True, "pre": True, "pre2": True, "no_out0": True,
                                                    "aux_halo": 1}, PIN_THIN, THIN % (1, 1, 4)),
    "thin-1x1-16-8": ((2, 40, 40, 16, 7, 1, 1, 1), {"in_halo": 1, "out_halo": 1}, PIN_THIN, THIN % (1, 2, 1)),
    "thin-1x1-16-16": ((2, 20, 20, 14, 14, 1, 1, 1), {"act": None, "residual": True}, PIN_THIN, THIN % (1, 2, 2)),
    "thin-1x1-16-32": ((2, 20, 20, 14, 28, 1, 1, 1), {"pre": True, "aux_halo": 1}, PIN_THIN, THIN % (1, 2, 4)),
    "thin-1x1-32-8": ((2, 37, 41, 28, 7, 1, 1, 1), {"in_halo": 1, "out_halo": 1}, PIN_THIN, THIN % (1, 4, 1)),
    "thin-1x1-32-16": ((2, 40, 40, 28, 14, 1, 1, 1), {"in_halo": 1, "act": "leaky"}, PIN_THIN, THIN % (1, 4, 2)),
    "thin-1x1-32-32": ((2, 20, 20, 32, 32, 1, 1, 1), {"no_out0": True, "pre": True}, PIN_THIN, THIN % (1, 4, 4)),
    "thin-3x3-8-8": ((2, 40, 40, 7, 7, 3, 1, 1), {"in_halo": 1, "out_halo": 1}, PIN_THIN, THIN % (3, 1, 1)),
    "thin-3x3-8-16-s2": ((2, 41, 39, 7, 14, 3, 2, 1), {"in_halo": 1}, PIN_THIN, THIN % (3, 1, 2)),
    "thin-3x3-16-8": ((2, 37, 41, 14, 7, 3, 1, 1), {"act": None}, PIN_THIN, THIN % (3, 2, 1)),
    "thin-3x3-16-16-s2": ((2, 40, 40, 14, 14, 3, 2, 1), {"out_halo": 1, "residual": True}, PIN_THIN,
                          THIN % (3, 2, 2)),
    # CUDA-core fallback
    "direct16": ((2, 19, 19, 64, 96, 3, 1, 2), {"act": "leaky", "residual": True, "pre": True, "pre2": True},
                 {}, "conv_direct_kernel<__half,false>"),
    "direct32": ((1, 10, 10, 7, 28, 3, 2, 1), {"residual": True, "pre": True, "pre2": True}, {},
                 "conv_direct_kernel<float,false>"),
}


def _plan_bn(shape, kw):
    """The N tile conv_tc takes for an im2col-mode case, from the library's planner; None in the halo-flat modes."""
    from odt_b200 import lib as L
    B, H, W, Cin, Cout, k, stride, dil = shape
    if kw.get("in_halo") and k == 3 and stride == 1 and dil == 1 and (Cout + 31) // 32 * 32 <= 128:
        return None
    from odt_b200.engine import same_pad
    OH, OW = same_pad(H, k, stride, dil)[0], same_pad(W, k, stride, dil)[0]
    return L.load().odt_conv_tc_pick_bn((Cout + 31) // 32 * 32, B * OH * OW, k * k * ((Cin + 63) // 64))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BODY_CASES))
def test_body_dispatch(built, monkeypatch, name):
    from test_gpu_conv import _conv_case
    shape, kw, env, kern = BODY_CASES[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    mode = name if name.startswith("direct") else "tc"
    r = _conv_case(*shape, mode=mode, seed=sum(shape), **kw)
    if kern is not None:
        assert r.kernel == kern, (r.kernel, kern)
    if r.kernel.startswith("conv_tc_kernel<"):
        bn = _plan_bn(shape, kw)
        if bn is not None:
            assert r.kernel.startswith("conv_tc_kernel<%d," % bn), (r.kernel, bn)
    print("%s: %s, worst %.3g of the bound" % (name, r.kernel, r.worst))


def _compiled_body_kernels():
    """The body-convolution kernels compiled into the library (every conv kernel but the stems')."""
    import odt_b200
    import os
    so = os.path.join(os.path.dirname(odt_b200.__file__), "libodt_b200.so")
    out = subprocess.run(["nm", "-C", so], check=True, capture_output=True, text=True).stdout
    names = set()
    for line in out.splitlines():
        m = re.search(r" [tTwW] (?:void )?odt::(conv_\w+kernel(<[^(]*>)?)\(", line)
        if m:
            names.add(re.sub(r"\s+", "", m.group(1)))
    return {n for n in names if not n.startswith("conv_stem") and not re.match(r"conv_direct_kernel<\w+,true>", n)}


def test_body_cases_name_every_compiled_kernel(built):
    """The kernels the case table names are exactly the body-convolution kernels compiled into the library, so a new
    instantiation without a case fails here."""
    want = {k for _, _, _, k in BODY_CASES.values() if k is not None}
    compiled = _compiled_body_kernels()
    assert len(compiled) == 10 + 1 + 4 + 3 + 13 + 2, sorted(compiled)
    assert want == compiled, (sorted(compiled - want), sorted(want - compiled))


# ---------------------------------------------------------------------------------------------------------------------
# c. out1 / out2 do not depend on whether out0 is stored
# ---------------------------------------------------------------------------------------------------------------------
OUT0_CASES = {
    # id: (shape, keywords, environment, kernel family)
    "tc-vector": ((2, 26, 26, 128, 64, 3, 1, 1), {"residual": True}, PIN_TC, "conv_tc_kernel<"),
    "tc-generic": ((2, 19, 19, 128, 60, 3, 1, 1), {"residual": True, "off": 1}, {}, "conv_tc_kernel<"),
    "tc-wide": ((4, 38, 38, 64, 256, 3, 1, 1), {"residual": True}, {"ODT_TC_WIDE": "2"}, "conv_tc_kernel<256,"),
    "tapn": ((2, 40, 40, 28, 28, 3, 1, 1), {"in_halo": 1, "residual": True}, {"ODT_TC_TAPN": "2"}, "conv_tapn_kernel<"),
    "pw": ((2, 33, 35, 28, 14, 1, 1, 1), {"residual": True}, {"ODT_TC_PW": "2"}, "conv_pw_kernel<"),
    "thin": ((2, 40, 40, 7, 28, 1, 1, 1), {"residual": True}, PIN_THIN, "conv_thin_kernel<"),
    "direct16": ((2, 19, 19, 64, 40, 3, 1, 1), {"residual": True}, {}, "conv_direct_kernel<__half"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(OUT0_CASES))
def test_extra_outputs_independent_of_out0(built, monkeypatch, name):
    """The same layer with and without out0: out1 / out2 bit-identical (both take the fp16-rounded v)."""
    from test_gpu_conv import _conv_case
    shape, kw, env, fam = OUT0_CASES[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    mode = "direct16" if name == "direct16" else "tc"
    runs = [_conv_case(*shape, mode=mode, seed=7, act="leaky", pre=True, pre2=True, aux_halo=1, no_out0=n, **kw)
            for n in (False, True)]
    for r in runs:
        assert r.kernel.startswith(fam), (r.kernel, fam)
    a, b = runs
    np.testing.assert_array_equal(a.got1.view(np.uint32), b.got1.view(np.uint32))
    np.testing.assert_array_equal(a.got2.view(np.uint32), b.got2.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# d. in situ at full size
# ---------------------------------------------------------------------------------------------------------------------
def _family(kernel):
    return kernel.split("<")[0]


def _act_name(a):
    return {0: None, 1: "relu", 2: "leaky"}[a]


def _assert_layout(t, what):
    """The halo ring and the pad lanes [C, ld) of an activation hold zero."""
    if t.halo:
        assert not bool(t.buf[mask(t.buf.shape, 1)].ne(0).any()), "%s: halo written" % what
    if t.ld > t.C:
        assert not bool(t.buf[..., t.C:].ne(0).any()), "%s: pad lanes written" % what


def _insitu_op(net, op, imgs):
    """(kernel, worst ratio, where) of one body ConvOp, checked on images `imgs` of its real buffers."""
    from odt_b200 import lib as L
    p = op.p
    op.launch(net, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    kernel = last_conv_kernel()
    lib = net.lib
    if op.use_tc:
        rp, tiles, waste = C.c_int(-1), C.c_longlong(-1), C.c_int(-1)
        swap = lib.odt_conv_tc_swap_plan(C.byref(p), C.byref(rp), C.byref(tiles), C.byref(waste))
        assert (kernel == "conv_tc_swap_kernel") == bool(swap == 1), (op.kernel, kernel, swap)
        flat = p.in_halo == 1 and p.R == 3 and p.stride == 1 and p.dil == 1 and p.Cout_pad <= 128
        if kernel.startswith("conv_tc_kernel<") and not flat:
            bn = lib.odt_conv_tc_pick_bn(p.Cout_pad, p.B * p.OH * p.OW, p.R * p.S * p.in_ld // 64)
            assert kernel.startswith("conv_tc_kernel<%d," % bn), (op.kernel, kernel, bn)
    else:
        assert kernel.startswith("conv_direct_kernel<"), (op.kernel, kernel)
    f16 = net.precision == "fp16"
    x = op.x
    idx = torch.tensor(imgs, device="cuda")
    xin = interior(x.buf, x.halo)[..., :x.C].index_select(0, idx)
    w = op.wdev[:op.cout, :, :, :x.C]
    sc = op.scale[:op.cout] if op.scale is not None else None
    ref, mag = R.reference(xin, w, op.stride, sc, op.shift[:op.cout], _act_name(p.act), op.dil)
    res = None
    if op.residual is not None:
        res = interior(op.residual.buf, op.residual.halo)[..., :op.cout].index_select(0, idx)
    v = ref + res.double() if res is not None else ref
    b0 = R.bound(v, mag, R.n_acc_body(kernel, p.R, p.S, p.Cin, p.in_ld), f16, res)
    worst = [(0.0, None)]
    got0 = None
    if op.y is not None and op.y.needed:
        _assert_layout(op.y, op.kernel + " out0")
        got0 = interior(op.y.buf, op.y.halo)[..., :op.cout].index_select(0, idx)
        worst.append(R.ratio(got0, R.pool2(v), R.pool2(b0)) if op.pool else R.ratio(got0, v, b0))
    for pre, s2n, h2n, act2 in ((op.pre, "scale2", "shift2", p.act2), (op.pre2, "scale3", "shift3", p.act3)):
        if pre is None:
            continue
        t = pre[2]
        _assert_layout(t, op.kernel + " out1/out2")
        got = interior(t.buf, t.halo)[..., :op.cout].index_select(0, idx)
        s2 = getattr(op, s2n)[:op.cout] if pre[0] is not None else torch.ones(op.cout, device="cuda")
        h2 = getattr(op, h2n)[:op.cout] if pre[0] is not None else torch.zeros(op.cout, device="cuda")
        if got0 is not None:
            tt = R.consumer(got0, s2, h2, _act_name(act2))
            worst.append(R.ratio(got, tt, R.bound_own(tt, f16)))
        else:
            tt = R.consumer(v, s2, h2, _act_name(act2))
            worst.append(R.ratio(got, tt, R.bound_through(tt, b0, s2, f16)))
    r, at = max(worst, key=lambda q: q[0])
    if r > 1.0:  # what the failing element holds, for the report
        at = (at, "got0 %s ref %s mag %s x-nan %s" % (
            None if got0 is None else float(got0[at]), float(v[at]), float(mag[at]), bool(torch.isnan(xin).any())))
    return kernel, r, at


INSITU = [("ssd300", "fp16", 64, {}), ("ssd512", "fp16", 8, {}),
          ("retinanet", "fp16", 16, {"data_shape": [800, 800, 3]}),
          ("retinanet", "fp16", 16, {"data_shape": [800, 800, 3], "is_bottleneck": False, "init_conv_filters": 7,
                                     "residual_block_list": [2, 2, 2, 2]}),
          ("yolov3", "fp16", 32, {"data_shape": [416, 416, 3], "num_classes": 20}),
          ("fcos", "fp16", 4, {"data_shape": [1024, 1024, 3]}),
          ("fcos", "fp32", 4, {"data_shape": [1024, 1024, 3]}),
          ("retinanet", "fp32", 2, {"data_shape": [512, 512, 3]}),
          ("yolov2", "fp16", 64, {}), ("yolov2", "fp16", 8, {"size": 200}), ("yolov2", "fp32", 2, {})]
INSITU_IDS = ["ssd300-fp16-B64", "ssd512-fp16-B8", "retinanet800-fp16-B16", "retinanet800-basic-fp16-B16",
              "yolov3-416-fp16-B32", "fcos1024-fp16-B4", "fcos1024-fp32-B4", "retinanet512-fp32-B2",
              "yolov2-480-fp16-B64", "yolov2-200-fp16-B8", "yolov2-480-fp32-B2"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,precision,B,over", INSITU, ids=INSITU_IDS)
def test_body_convs_in_situ(built, kind, precision, B, over):
    """Every body convolution of the network at its full per-GPU geometry, on its real buffers after one eager
    forward: launched kernel (the library's record of the op's own launch, against the host planners), out0 (pooled
    or not), residual, out1 / out2 against the bound (a concat part's out1 read through its slice view), and zero
    halo rings and pad lanes.  A concat tensor is NaN-filled before the forward: its parts' slices must tile it."""
    from odt_b200 import engine as E
    m = _model(kind, precision, **over)
    net = m.engine(B, graph=False)
    img = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (B, net.in_h, net.in_w, 3)).astype(np.float32))
    net.image_buf.copy_(img)
    concats = [t for t in net.acts if t.parts]
    for y in concats:
        y.buf[..., :y.C] = float("nan")
    net.forward(with_tail=False)
    torch.cuda.synchronize()
    for y in concats:
        assert [(v.c0, v.c0 + v.C) for v in y.parts] == list(zip([0] + [v.c0 + v.C for v in y.parts[:-1]],
                                                                 [v.c0 + v.C for v in y.parts]))
        assert y.parts[-1].c0 + y.parts[-1].C == y.C
        for v in y.parts:
            assert v.buf.data_ptr() == y.buf.data_ptr() + v.c0 * y.buf.element_size() and v.buf.stride() == y.buf.stride()
        assert not bool(torch.isnan(y.buf).any()), "%s: a channel no slice covers" % y.name
        if y.ld > y.C:
            assert not bool(y.buf[..., y.C:].ne(0).any()), "%s: pad lanes written" % y.name
    # every activation owns its buffer (a concat's slices are views of it): re-launching one op cannot change another
    # op's input
    acts = {}
    for op in net.ops:
        extra = tuple(pr[2] for pr in (getattr(op, "pre", None), getattr(op, "pre2", None)) if pr is not None)
        for t in tuple(op.reads) + tuple(op.writes) + extra:
            if t is not None and t.buf is not None and t.base is None:
                acts[id(t)] = t
    spans = sorted((t.buf.data_ptr(), t.buf.data_ptr() + t.buf.numel() * t.buf.element_size(), t.name)
                   for t in acts.values())
    for a, b in zip(spans, spans[1:]):
        assert a[1] <= b[0], ("activation buffers overlap", a[2], b[2])
    body = [op for op in net.ops if isinstance(op, E.ConvOp) and not op.is_image and op.head is None]
    assert body
    imgs = sorted({0, B // 2, B - 1})
    tag = "%s %s B=%d" % (kind, precision, B)
    fam = {}
    for op in body:
        kernel, r, at = _insitu_op(net, op, imgs)
        f = _family(kernel)
        fam[f] = max(fam.get(f, 0.0), r)
        print("%s %-40s %-34s %.3g%s" % (tag, op.kernel, kernel, r,
                                         "" if (op.y is not None and op.y.needed) else "  (out0 not stored)"))
        assert r <= 1.0, (op.kernel, kernel, r, at)
    print("%s: %d body convolutions; worst per kernel family: %s" % (
        tag, len(body), ", ".join("%s %.3g" % kv for kv in sorted(fam.items()))))
    del net, m
    torch.cuda.empty_cache()
