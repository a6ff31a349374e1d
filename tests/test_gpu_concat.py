"""Net.concat's copy-free channel slices: each part's producer stores its slice [c0, c0 + C) of the concatenated tensor
as an extra epilogue output (out1 / out2) at the concat's pixel stride.

  a. the slice write rules (gpu_harness.assert_slice_writes) on the host: an honest slice passes, a zero written into
     the next slice's first lane and a slice written at the producer's own pixel stride are rejected;
  b. the refusals of Net.fuse() (engine._check_slice_producer) on the host: pools, upsample-adds and parts whose
     producer's store width (engine.slice_store_width) reaches the next part;
  c. every kernel family that takes an extra output writing it into a slice of a sentinel-filled wider tensor, at
     c0 = 0, 8, 20 (not 16-byte aligned) and 512, aligned and ragged Cout, out0 stored and not: the slice against the
     float64 reference and bound of tests/test_gpu_conv.py's _conv_case, every other channel and both guard bands
     untouched but for the +0 pad lanes the store width allows;
  d. small networks built with the Net API: the concat buffer against torch.cat of the same parts computed without a
     concat, and the eager forward against the lane-planned graph replay, bit for bit.
"""
import numpy as np
import pytest
import torch

import conv_ends_ref as R
from gpu_harness import SENT, Guarded, assert_slice_writes, last_conv_kernel


# ---------------------------------------------------------------------------------------------------------------------
# a. the slice write rules (host)
# ---------------------------------------------------------------------------------------------------------------------
def test_slice_check_rejects_planted_faults():
    B, H, W, ld, c0, C, end = 2, 3, 5, 96, 20, 20, 52
    was = torch.full((B, H, W, ld), SENT, dtype=torch.float16)
    vals = torch.randn(B, H, W, C).half()
    honest = was.clone()
    honest[..., c0:c0 + C] = vals
    honest[..., c0 + C:c0 + 32] = 0                  # pad lanes of a 32-channel chunk store: allowed, reported
    assert assert_slice_writes(honest, was, c0, C, end, "honest") == 12
    bad = {}
    t = honest.clone()
    t[..., end] = 0                                   # a zero in the next slice's first lane
    bad["zero in the next slice"] = t
    t = was.clone().reshape(-1)                       # the slice at the producer's own pixel stride (64)
    for pix in range(B * H * W):
        t[pix * 64 + c0:pix * 64 + c0 + C] = vals.reshape(-1, C)[pix]
    bad["producer's own stride"] = t.reshape(was.shape)
    for what, t in bad.items():
        with pytest.raises(AssertionError):
            assert_slice_writes(t, was, c0, C, end, what)


# ---------------------------------------------------------------------------------------------------------------------
# b. the refusals (host)
# ---------------------------------------------------------------------------------------------------------------------
def _graph(case, precision, B=2, size=32):
    """(net, concat tensor or None, parts) of one small network.  concat=False: the same graph with the parts left
    as tensors of their own (the reference of the concat)."""
    from odt_b200 import engine as E
    name, concat = case
    net = E.Net(B, size, size, precision)
    if name in ("image", "image-overflow"):
        s = net.conv(None, 20, 3, name="stem", bn=True, act="relu")
        b = net.conv(s, 32 if name == "image" else 40, 3, name="b", bn=True, act="leaky")
        parts = [s, b]
    else:
        x = net.conv(None, 32, 3, name="stem", bn=True, act="relu")
        a = net.conv(x, 64, 3, name="a", bn=True, act="leaky")
        b = net.conv(x, 128, 1, name="b", bn=True)
        r = net.conv(x, 20, 3, name="r", bn=True, act="relu")
        net.conv(a, 64, 1, name="reads_a", bn=True)   # a keeps its own output: out0 and the slice both stored
        parts = {"tc": [a, b], "tc-ragged-last": [a, b, r], "ragged-ahead": [r, a],
                 "cuda-core": [r, a, net.conv(x, 60, 1, name="c", bn=True), net.conv(x, 100, 3, name="d", bn=True)],
                 "pool": [net.maxpool(a, 3, 1), b],
                 "upsample": [net.upsample_add(net.conv(a, 64, 3, 2, name="top", bn=True), a), b]}[name]
    y = net.concat(parts) if concat else None
    return net, y, parts


HOST_CASES = [("tc", "fp16"), ("tc-ragged-last", "fp16"), ("cuda-core", "fp32"), ("image", "fp16"), ("image", "fp32"),
              ("image-overflow", "fp32"), ("ragged-ahead", "fp32"), ("pool", "fp16"), ("pool", "fp32"),
              ("upsample", "fp16"), ("upsample", "fp32"), ("ragged-ahead", "fp16"), ("image-overflow", "fp16")]


def _refused(name, precision):
    """Whether fuse() must refuse the case: pools and upsample-adds always; on the tensor cores (32-channel chunks) a
    20-channel part ahead of another, and a 40-channel part at c0 = 20 of a 64-channel row."""
    return name in ("pool", "upsample") or (name in ("ragged-ahead", "image-overflow") and precision == "fp16")


def _slice_producer(net, v):
    """Index in net.ops of the op that stores the slice v as an extra output."""
    return next(i for i, o in enumerate(net.ops) for pr in (getattr(o, "pre", None), getattr(o, "pre2", None))
                if pr is not None and pr[2] is v)


@pytest.mark.parametrize("name,precision", HOST_CASES)
def test_fuse_refuses_what_a_producer_cannot_store(name, precision):
    from odt_b200 import engine as E
    E.Net.spec_only = True
    try:
        net, y, parts = _graph((name, True), precision)
    finally:
        E.Net.spec_only = False
    if _refused(name, precision):
        with pytest.raises(ValueError, match="cannot store its channel slice"):
            net.fuse()
        return
    net.fuse()
    assert not any(isinstance(op, E.AffineActOp) for op in net.ops)
    for v, nxt in zip(y.parts, y.parts[1:] + (None,)):
        op = net.ops[_slice_producer(net, v)]
        assert isinstance(op, E.ConvOp)
        assert v.c0 + op.slice_channels(net) <= (nxt.c0 if nxt is not None else y.ld), (name, v.name)


def test_yolov2_concat_is_accepted():
    """YOLOv2's passthrough concat (512 + 1024 channels) is what the refusals must leave alone."""
    from odt_b200 import engine as E
    from odt_b200 import nets
    from test_gpu_yolov2 import _cfg
    E.Net.spec_only = True
    try:
        net, _ = nets.build_yolov2(2, _cfg(), "fp16", "cpu", True)
    finally:
        E.Net.spec_only = False
    net.fuse()
    y = next(t for t in net.acts if t.parts)
    assert [(v.c0, v.C) for v in y.parts] == [(0, 512), (512, 1024)] and y.ld == 1536


# ---------------------------------------------------------------------------------------------------------------------
# c. slice stores per kernel family
# ---------------------------------------------------------------------------------------------------------------------
PIN_TC = {"ODT_TC_TAPN": "0", "ODT_TC_SWAP": "0", "ODT_TC_PW": "0", "ODT_TC_THIN": "0"}
# family: (shape as a function of Cout, the Couts, mode, _conv_case keywords, environment, launched kernel)
FAMILIES = {
    "tc32": (lambda c: (2, 19, 19, 64, c, 3, 1, 1), (20, 32), "tc", {}, PIN_TC, "conv_tc_kernel<32,false>"),
    "tc64": (lambda c: (8, 38, 38, 64, c, 3, 1, 1), (60, 64), "tc", {}, PIN_TC, "conv_tc_kernel<64,false>"),
    "tc96": (lambda c: (4, 38, 38, 256, c, 1, 1, 1), (96,), "tc", {}, PIN_TC, "conv_tc_kernel<96,false>"),
    "tc128": (lambda c: (8, 38, 38, 64, c, 3, 1, 1), (100, 128), "tc", {}, PIN_TC, "conv_tc_kernel<128,false>"),
    "tc256-wide": (lambda c: (4, 38, 38, 64, c, 3, 1, 1), (256,), "tc", {"residual": True},
                   dict(PIN_TC, ODT_TC_WIDE="2"), "conv_tc_kernel<256,false>"),
    "tc-generic": (lambda c: (2, 19, 19, 128, c, 3, 1, 1), (20, 60, 100), "tc", {"off": 1}, PIN_TC,
                   "conv_tc_kernel<"),
    "tapn": (lambda c: (2, 40, 40, 64, c, 3, 1, 1), (20, 60, 64), "tc", {"in_halo": 1}, {"ODT_TC_TAPN": "2"},
             "conv_tapn_kernel<"),
    "pw": (lambda c: (2, 33, 35, 28, c, 1, 1, 1), (20, 60, 100), "tc", {}, {"ODT_TC_PW": "2"}, "conv_pw_kernel<"),
    "thin": (lambda c: (2, 40, 40, 7, c, 1, 1, 1), (20, 32), "tc", {}, {"ODT_TC_THIN": "2", "ODT_TC_PW": "0"},
             "conv_thin_kernel<"),
    "direct16": (lambda c: (2, 19, 19, 64, c, 3, 1, 2), (20, 60, 100), "direct16", {"act": "leaky"}, {},
                 "conv_direct_kernel<__half,false>"),
    "direct32": (lambda c: (1, 10, 10, 7, c, 3, 2, 1), (20, 60, 100), "direct32", {}, {},
                 "conv_direct_kernel<float,false>"),
}
C0S = (0, 8, 20, 512)


@pytest.mark.gpu
@pytest.mark.parametrize("family", list(FAMILIES))
def test_slice_stores(built, monkeypatch, family):
    """out1 and out2 into channel c0 of sentinel-filled tensors of pixel stride ld > Cout_pad.  A slice that does not
    start on a 16-byte boundary (fp16, c0 = 20) leaves the sector-store kernels (taps as N, pointwise, thin) for
    conv_tc's column path."""
    from test_gpu_conv import _conv_case
    shape_of, couts, mode, kw, env, kern = FAMILIES[family]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    worst, spills = 0.0, []
    for cout in couts:
        for c0 in C0S:
            for no_out0 in (False, True):
                shape = shape_of(cout)
                ld = (c0 + (cout + 31) // 32 * 32 + 63) // 64 * 64 + 64
                what = "%s Cout %d c0 %d ld %d%s" % (family, cout, c0, ld, " (out0 not stored)" if no_out0 else "")
                r = _conv_case(*shape, mode=mode, seed=sum(shape) + c0, pre=True, pre2=True, no_out0=no_out0,
                               slice_at=(c0, ld), **kw)
                want = kern
                if mode == "tc" and c0 % 8 and not kern.startswith("conv_tc_kernel<"):
                    want = "conv_tc_kernel<"
                assert r.kernel.startswith(want), (what, r.kernel, want)
                worst = max(worst, r.worst)
                if r.spill:
                    spills.append("Cout %d c0 %d: %d" % (cout, c0, r.spill))
                print("%s: %s, worst %.3g of the bound, %d +0 channels past the slice" % (what, r.kernel, r.worst,
                                                                                         r.spill))
    print("%s: worst %.3g of the bound; +0 channels stored past a slice: %s" % (family, worst,
                                                                               "; ".join(spills) or "none"))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["f16", "f32"])
def test_stem_slice_stores(built, dtype):
    """The image convolution with an extra output takes the CUDA-core stem (conv_direct_kernel<T,true>): its slice
    against the stem's own out0 through the consumer affine, exact store width, and bit-identical whether or not out0
    is stored."""
    from odt_b200 import lib as L
    from test_gpu_conv_ends import _stem_case
    f16 = dtype == "f16"
    tdt = torch.float16 if f16 else torch.float32
    worst = 0.0
    for cout in (20, 60):
        for c0 in C0S:
            firsts = None
            for no_out0 in (False, True):
                B, H, W = 2, 20, 21
                launch, c = _stem_case("direct16" if f16 else "direct32", B, H, W, cout, 3, 1, 0, cout,
                                       seed=cout + c0)
                p, OH, OW = c["p"], c["OH"], c["OW"]
                ld = (c0 + cout + 63) // 64 * 64 + 64
                g = torch.Generator(device="cpu").manual_seed(c0)
                outs = []
                for i, act in enumerate(("relu", "leaky")):
                    s = (torch.rand(cout, generator=g) + 0.5).cuda()
                    h = (torch.randn(cout, generator=g) * 0.2).cuda()
                    outs.append((Guarded((B, OH, OW, ld), tdt), s, h, act))
                (g1, s2, h2, a2), (g2, s3, h3, a3) = outs
                esz = 2 if f16 else 4
                p.scale2, p.shift2, p.act2 = s2.data_ptr(), h2.data_ptr(), R.ACTS[a2]
                p.out1, p.out1_img_stride, p.out1_pix_stride = g1.ptr() + c0 * esz, OH * OW * ld, ld
                p.scale3, p.shift3, p.act3 = s3.data_ptr(), h3.data_ptr(), R.ACTS[a3]
                p.out2, p.out2_img_stride, p.out2_pix_stride = g2.ptr() + c0 * esz, OH * OW * ld, ld
                if no_out0:
                    p.out0 = None
                L.check(launch(), "stem")
                torch.cuda.synchronize()
                assert last_conv_kernel() == "conv_direct_kernel<%s,true>" % ("__half" if f16 else "float")
                got0 = c["out"].t[..., :cout]
                if no_out0:
                    c["out"].assert_untouched(torch.ones(c["out"].t.shape, dtype=torch.bool, device="cuda"), "out0")
                else:
                    x = R.stem_operand(c["img"], False)
                    r, at = R.checked(lambda b0, b1: got0[b0:b1], x, c["w"][:cout], 1, c["scale"][:cout],
                                      c["shift"][:cout], "relu", R.n_acc_cuda_core(3, 3, 3), f16, chunk=2)
                    assert r <= 1.0, (cout, c0, "out0", r, at)
                    worst = max(worst, r)
                got = []
                for i, (gg, s, h, act) in enumerate(outs):
                    gg.assert_outside_untouched()
                    assert assert_slice_writes(gg.t, gg.initial(), c0, cout, c0 + cout, "out%d" % (i + 1)) == 0
                    t = gg.t[..., c0:c0 + cout]
                    if not no_out0:
                        tt = R.consumer(got0, s, h, act)
                        r, at = R.ratio(t, tt, R.bound_own(tt, f16))
                        assert r <= 1.0, (cout, c0, "out%d" % (i + 1), r, at)
                        worst = max(worst, r)
                    got.append(t.clone())
                if firsts is None:
                    firsts = got
                else:
                    for a, b in zip(firsts, got):
                        assert torch.equal(a, b), (cout, c0, "an extra output depends on out0")
    print("stem %s: worst %.3g of the bound" % (dtype, worst))


# ---------------------------------------------------------------------------------------------------------------------
# d. Net.concat end to end
# ---------------------------------------------------------------------------------------------------------------------
class _StubTail:
    row = 0

    def prepare(self, net, head_buf=None):
        pass

    def launch(self, net, stream):
        pass

    def num_launches(self):
        return 0


def _run(case, precision, weights=None, img=None):
    from odt_b200 import engine as E
    net, y, parts = _graph(case, precision)
    w = E.init_weights(net.vars, seed=3, bn_mode="trained") if weights is None else weights
    net.finalize(w, _StubTail())
    if img is None:
        img = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (net.batch, net.in_h, net.in_w, 3))
                               .astype(np.float32))
    net.image_buf.copy_(img)
    return net, y, parts, w, img


ENGINE_CASES = [("tc", "fp16"), ("tc-ragged-last", "fp16"), ("cuda-core", "fp32"), ("image", "fp16"),
                ("image", "fp32"), ("pool", "fp16"), ("pool", "fp32"), ("upsample", "fp16"), ("ragged-ahead", "fp16")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,precision", ENGINE_CASES)
def test_concat_in_a_network(built, name, precision):
    """The concat buffer of one eager forward against torch.cat of the parts of the same network built without the
    concat, bit for bit (the identity extra output stores the value out0 would hold); a part whose out0 is stored too against it bit for bit; the concat's pad lanes zero; the graph replay
    (parts on separate lanes where the plan puts them there) bit-identical to the eager forward.  The cases fuse()
    must refuse raise instead."""
    try:
        net, y, parts, w, img = _run((name, True), precision)
    except ValueError as e:
        assert _refused(name, precision), ("refused", name, precision, str(e))
        return
    lane_of, _, _ = net.plan_lanes()
    lanes = sorted({lane_of[_slice_producer(net, v)] for v in y.parts})
    net.forward(with_tail=False)
    torch.cuda.synchronize()
    eager = y.buf.clone()
    ref_net, _, ref_parts, _, _ = _run((name, False), precision, w, img)
    ref_net.forward(with_tail=False)
    torch.cuda.synchronize()
    want = torch.cat([t.buf[..., :t.C] for t in ref_parts], dim=-1)
    got = eager[..., :y.C]
    bad = got.ne(want)
    assert not bool(bad.any()), (name, precision, "concat differs from torch.cat of its parts at channel",
                                 int(bad.nonzero()[0][-1]), float((got.double() - want.double()).abs().max()))
    assert _refused(name, precision) is False, (name, precision, "computed, but fuse() must refuse it")
    if y.ld > y.C:
        assert not bool(eager[..., y.C:].ne(0).any()), "concat pad lanes written"
    for t, v in zip(parts, y.parts):
        if t.buf is not None:
            assert torch.equal(t.buf[..., :t.C], eager[..., v.c0:v.c0 + v.C]), (name, t.name, "slice != own out0")
    net.capture()
    y.buf[..., :y.C] = SENT
    net.graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(y.buf, eager), (name, precision, "graph replay differs from the eager forward")
    print("%s %s: parts %s on lanes %s" % (name, precision, [(v.c0, v.C) for v in y.parts], lanes))
    if name in ("tc", "cuda-core"):
        assert len(lanes) > 1, (name, "the parts' producers share one lane")
