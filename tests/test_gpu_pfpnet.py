"""PFPNet-R on the GPU: the three new glue kernels against float64 references, the transposed-convolution layers
against oracle/pfpnet.py in fp32 and fp16, the two-step decode / NMS tail on oracle rows (bit-exact class ids and keep
indices, a dense case past the 1 024-key window), the whole network at 128², 320² and 512² against the oracle forward,
the loss and gradient kernels (odt_pfpnet_loss_*) against the oracle and the restatement, the training step through
them, pipelined against single-graph streams, and the convolution dispatch."""
import numpy as np
import pytest
import torch

from helpers import BASE_CFG, assert_boxes_close

pytestmark = pytest.mark.gpu
F32 = np.float32


def _model(size=320, **over):
    import PFPNetR
    c = dict(BASE_CFG)
    c.update(input_size=size, bn_init="trained")
    c.update(over)
    return PFPNetR.PFPNetR(c, None)


def _img(b, s, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (b, s, s, 3)).astype(F32)


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda().to(dtype)


DT = {"fp32": (torch.float32, 1, 1e-6), "fp16": (torch.float16, 0, 2e-3)}  # (dtype, ODT_F32 / ODT_F16, tol)


# --------------------------------------------------------------------------------------------- glue kernels ----
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("C,res,act", [(85, False, 0), (85, True, 0), (256, True, 1), (256, False, 1)])
def test_pixel_shuffle(built, prec, C, res, act):
    from odt_b200 import lib
    L = lib.load()
    tdt, code, tol = DT[prec]
    rng = np.random.default_rng(C + res)
    B, h, w = 2, 5, 7
    in_ld, out_ld = 4 * C + 44, C + 43  # strides wider than the tensors, as a padded layout has
    x = rng.standard_normal((B, h, w, in_ld)).astype(F32)
    r = rng.standard_normal((B, 2 * h, 2 * w, C + 11)).astype(F32)
    xd, rd = _dev(x, tdt), _dev(r, tdt)
    out = torch.full((B, 2 * h, 2 * w, out_ld), 7.0, dtype=tdt, device="cuda")
    lib.check(L.odt_pixel_shuffle2x(xd.data_ptr(), out.data_ptr(), rd.data_ptr() if res else None, code, B, h, w, C,
                                    in_ld, out_ld, C + 11, act, torch.cuda.current_stream().cuda_stream))
    xq = xd.double().cpu().numpy()
    exp = np.zeros((B, 2 * h, 2 * w, C))
    for py in range(2):
        for px in range(2):
            p = 2 * py + px
            exp[:, py::2, px::2] = xq[..., p * C:(p + 1) * C]
    if res:
        exp += rd.double().cpu().numpy()[..., :C]
    if act == 1:
        exp = np.maximum(exp, 0)
    got = out.double().cpu().numpy()
    np.testing.assert_allclose(got[..., :C], exp, rtol=tol, atol=tol)
    assert np.all(got[..., C:] == 7.0), "stores past C"


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("H,W,OH,OW", [(40, 40, 20, 20), (40, 40, 5, 5), (9, 6, 1, 1), (7, 5, 4, 3), (4, 4, 9, 7)])
def test_resize_align_corners(built, prec, H, W, OH, OW):
    from odt_b200 import lib
    L = lib.load()
    tdt, code, tol = DT[prec]
    C, ld, ld2 = 85, 96, 800
    x = np.random.default_rng(H * OH).standard_normal((2, H, W, ld)).astype(F32)
    xd = _dev(x, tdt)
    out = torch.zeros((2, OH, OW, C), dtype=tdt, device="cuda")
    out2 = torch.full((2, OH, OW, ld2), 5.0, dtype=tdt, device="cuda")
    lib.check(L.odt_resize_bilinear_ac(xd.data_ptr(), out.data_ptr(), out2[..., 96:].data_ptr(), code, 2, H, W, C,
                                       ld, OH, OW, C, ld2, torch.cuda.current_stream().cuda_stream))
    xq = xd.double().cpu().numpy()[..., :C]

    def axis(n, m):
        s = (n - 1) / (m - 1) if m > 1 else 0.0
        src = np.arange(m) * s
        lo = np.floor(src).astype(int)
        return lo, np.minimum(lo + 1, n - 1), src - lo

    y0, y1, ly = axis(H, OH)
    x0, x1, lx = axis(W, OW)
    ly, lx = ly[None, :, None, None], lx[None, None, :, None]
    top = xq[:, y0][:, :, x0] * (1 - lx) + xq[:, y0][:, :, x1] * lx
    bot = xq[:, y1][:, :, x0] * (1 - lx) + xq[:, y1][:, :, x1] * lx
    exp = top * (1 - ly) + bot * ly
    # float64 positions and weights: the float32 scale and lerps of TF's arithmetic differ from them by ~1e-6
    bar = 1e-4 if prec == "fp32" else 8e-3
    np.testing.assert_allclose(out.double().cpu().numpy(), exp, rtol=bar, atol=bar)
    g2 = out2.double().cpu().numpy()
    assert np.array_equal(g2[..., 96:96 + C], out.double().cpu().numpy())
    assert np.all(g2[..., :96] == 5.0) and np.all(g2[..., 96 + C:] == 5.0)
    if prec == "fp32":  # the oracle's TF arithmetic, rounded op by op, bit for bit
        from oracle.pfpnet import resize_bilinear_ac
        assert np.array_equal(out.cpu().numpy(), resize_bilinear_ac(x[..., :C], OH, OW))


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("H,W", [(3, 3), (5, 8), (1, 7), (20, 20), (11, 9)])
def test_avgpool_same(built, prec, H, W):
    from odt_b200 import lib
    L = lib.load()
    tdt, code, tol = DT[prec]
    C, ld = 85, 128
    x = np.random.default_rng(H * W).standard_normal((2, H, W, ld)).astype(F32)
    xd = _dev(x, tdt)
    OH, OW = (H + 1) // 2, (W + 1) // 2
    out = torch.zeros((2, OH, OW, ld), dtype=tdt, device="cuda")
    lib.check(L.odt_avgpool2x2_same(xd.data_ptr(), out.data_ptr(), code, 2, H, W, C, ld, ld,
                                    torch.cuda.current_stream().cuda_stream))
    xq = xd.double().cpu().numpy()[..., :C]
    exp = np.zeros((2, OH, OW, C))
    for i in range(OH):
        for j in range(OW):
            exp[:, i, j] = xq[:, 2 * i:2 * i + 2, 2 * j:2 * j + 2].reshape(2, -1, C).mean(1)
    got = out.double().cpu().numpy()
    np.testing.assert_allclose(got[..., :C], exp, rtol=tol, atol=tol)
    assert not got[..., C:].any()
    if prec == "fp32":
        from oracle.pfpnet import avg_pool_same
        assert np.array_equal(out.cpu().numpy()[..., :C], avg_pool_same(x[..., :C]))


# ------------------------------------------------------------------------------------------------------- tail ----
def _rows(rng, N, dense=False):
    """Candidate rows [N, 31]: ODM logits with a background that wins, ties or loses, ARM logits either side of the
    0.99 cut, deltas that keep boxes in a sane range."""
    r = np.zeros((N, 31), F32)
    r[:, :21] = rng.standard_normal((N, 21)) * 2.0
    if dense:
        r[:, :20] += 4.0
    bg = rng.integers(0, 3, N)  # 0: as drawn, 1: background ties the best class, 2: background wins
    best = r[:, :20].max(1)
    r[bg == 1, 20] = best[bg == 1]
    r[bg == 2, 20] = best[bg == 2] + 0.5
    r[:, 21:25] = rng.standard_normal((N, 4)) * 0.3
    d = rng.choice([np.log(99.0), 0.0, -2.0, 3.0], N) + rng.choice([-1e-3, 1e-3], N)
    r[:, 25] = rng.standard_normal(N)
    r[:, 26] = (r[:, 25] + d).astype(F32)
    r[:, 27:31] = rng.standard_normal((N, 4)) * 0.3
    return r


@pytest.mark.parametrize("size,B,thr,dense", [(320, 3, 0.3, False), (512, 2, 0.05, False), (512, 1, 0.0, True)])
def test_tail_on_oracle_rows(built, size, B, thr, dense):
    from odt_b200.engine import RowsHarness
    from odt_b200 import nets
    from oracle.pfpnet import pfpnet_tail
    c = dict(BASE_CFG, input_size=size, nms_score_threshold=thr, nms_max_boxes=50 if dense else 20)
    tail = nets.pfpnet_tail(c)
    g = size // 8
    levels = [(g >> i, g >> i, 3) for i in range(4)]
    N = sum(h * w * a for h, w, a in levels)
    rng = np.random.default_rng(size + B)
    rows = np.stack([_rows(rng, N, dense) for _ in range(B)])
    h = RowsHarness(tail, levels, rows)
    res = h.run()
    keeps = h.keep_indices()
    if dense:
        assert int(tail.cand_count.cpu().numpy().max()) > 1024, "the dense case must exceed the shared-memory window"
    total = 0
    for b in range(B):
        s, bx, cid, k = pfpnet_tail(rows[b], [(hh, ww) for hh, ww, _ in levels], thr, c["nms_max_boxes"],
                                    c["nms_iou_threshold"])
        assert np.array_equal(res[b][2], cid), b
        assert np.array_equal(keeps[b], k), b
        np.testing.assert_allclose(res[b][0], s, rtol=1e-6, atol=1e-7)
        assert_boxes_close(res[b][1], bx)
        total += len(cid)
    assert total > 0


# ----------------------------------------------------------------------------------------------- network ----
@pytest.mark.parametrize("size,B,prec,tol", [(128, 2, "fp32", 2e-4), (128, 2, "fp16", 5e-3), (320, 1, "fp32", 2e-4),
                                             (320, 1, "fp16", 5e-3), (512, 1, "fp16", 5e-3)])
def test_full_network_vs_oracle(built, size, B, prec, tol):
    """Head rows within tol x max|ref| of the oracle forward; the tail on the GPU's own rows matches the oracle's tail
    bit for bit in class ids and keep indices."""
    from oracle.pfpnet import pfpnet_heads, pfpnet_rows, pfpnet_tail
    m = _model(size, precision=prec, nms_score_threshold=0.05)
    img = _img(B, size, seed=size)
    res = m.detect_batch(img)
    net = m.engine(B)
    rows = net.head_buf.cpu().numpy()
    heads = pfpnet_heads(m.get_weights(), img)
    ref = pfpnet_rows(heads)
    assert rows.shape == ref.shape == (B, 3 * sum((size // s) ** 2 for s in (8, 16, 32, 64)), 31)
    scale = float(np.abs(ref).max())
    err = float(np.abs(rows - ref).max())
    assert err <= tol * scale, (err, scale)
    shapes = [(a.shape[1], a.shape[2]) for a, _, _, _ in heads]
    for b in range(B):
        s, bx, cid, k = pfpnet_tail(rows[b], shapes, 0.05, m.nms_max_boxes, m.nms_iou_threshold)
        assert np.array_equal(res[b][2], cid)
        assert_boxes_close(res[b][1], bx)


def _dense(t):
    """An activation's values [B, H, W, C] as float32, without its halo border (Act.halo) and channel padding."""
    h = t.halo
    return t.buf.float().cpu().numpy()[:, h:h + t.H, h:h + t.W, :t.C]


def test_transposed_convolution_layers_in_situ(built):
    """Every PhaseConvOp + PixelShuffleOp pair of the 320² network, fed its own input from the GPU, against the oracle's
    scatter-definition conv2d_transpose -> BN (+ residual, ReLU): fp32 to 1e-4 and fp16 to 5e-3 of max|ref|."""
    from odt_b200 import engine as E
    from oracle import tfops as T
    from oracle.pfpnet import conv2d_transpose_same
    for prec, tol in (("fp32", 1e-4), ("fp16", 5e-3)):
        m = _model(320, precision=prec)
        m.detect_batch(_img(1, 320, seed=4))
        net = m.engine(1)
        w = m.get_weights()
        ops = net.ops
        n = 0
        for i, op in enumerate(ops):
            if not isinstance(op, E.PhaseConvOp):
                continue
            sh = next(o for o in ops[i + 1:] if isinstance(o, E.PixelShuffleOp) and o.x is op.y)
            x = _dense(op.x)
            y = T.batch_norm_inference(conv2d_transpose_same(x, w[op.kernel], w[op.bias]),
                                       *(w[op.bn + k] for k in ("/gamma", "/beta", "/moving_mean",
                                                                  "/moving_variance")))
            if sh.residual is not None:
                y = y + _dense(sh.residual)
            if sh.act == "relu":
                y = np.maximum(y, 0)
            got = _dense(sh.y)
            assert np.abs(got - y).max() <= tol * np.abs(y).max(), (prec, op.kernel)
            n += 1
        assert n == 9


def test_pipelined_and_single_graph_streams_agree(built, monkeypatch):
    m = _model(128, precision="fp16", nms_score_threshold=0.05)
    batches = [_img(2, 128, seed=s) for s in range(31, 35)]
    ref = [m.detect_batch(b) for b in batches]
    assert sum(len(r[2]) for rr in ref for r in rr) > 0
    pinned = [torch.from_numpy(b).pin_memory() for b in batches]
    for mode in ("1", "0"):
        monkeypatch.setenv("ODT_PIPELINE", mode)
        got = list(m.detect_stream(pinned))
        assert len(got) == len(ref)
        for g, r in zip(got, ref):
            for gi, ri in zip(g, r):
                for a, b in zip(gi, ri):
                    np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("size", [320, 512])
def test_dispatch_audit(built, size):
    """Every fp16 convolution runs a hand-written tensor-core kernel -- the image convolution on a stem kernel, every
    other one, the 85-channel 1x1 layers and the phase convolutions included, on odt_conv2d_f16_tc -- none on
    conv_direct.  The concats have no op of their own: conv4_3, the 1x1 layers and the resizes store their slices."""
    from odt_b200 import engine as E
    m = _model(size, precision="fp16")
    assert len(m.detect_batch(_img(1, size, seed=2))) == 1
    net = m.engine(1)
    convs = [op for op in net.ops if isinstance(op, E.ConvOp)]
    direct = [op.kernel for op in convs if not (op.is_image or op.use_tc)]
    assert not direct, direct
    phase = [op for op in convs if isinstance(op, E.PhaseConvOp)]
    assert sorted(op.p.Cout for op in phase) == [340] * 6 + [1024] * 3
    assert all(op.p.Cin == 85 and op.p.in_ld == 128 for op in phase if op.p.Cout == 340)
    kinds = {type(op).__name__ for op in net.ops}
    assert kinds == {"ConvOp", "PhaseConvOp", "PixelShuffleOp", "PoolOp", "ResizeOp", "AvgPoolOp", "L2NormOp"}
    resizes = [op for op in net.ops if isinstance(op, E.ResizeOp)]
    assert len(resizes) == 3 and all(op.out2 is not None for op in resizes)
    sliced = [op for op in convs if op.pre is not None and op.pre[2].base is not None]
    assert len(sliced) == 13  # conv4_3 + 12 of the 85-channel 1x1 layers
    assert np.isfinite(net.head_buf.cpu().numpy()).all()


# ------------------------------------------------------------------------------------------------ loss kernels ----
def _loss_harness(levels, rows):
    from odt_b200.engine import RowsHarness
    from odt_b200 import nets
    return RowsHarness(nets.pfpnet_tail(dict(BASE_CFG, input_size=320)), levels, rows)


L320 = [(40, 40, 3), (20, 20, 3), (10, 10, 3), (5, 5, 3)]


@pytest.mark.parametrize("G", [1, 128])
def test_loss_forward_vs_oracle(built, G):
    """odt_pfpnet_loss_fwd at 320² against oracle/pfpnet.py's loss within 2e-5, G = 1 and a full 128-row GT block,
    plus the three empty cases on the rows the CPU tests use."""
    import test_pfpnet as TP
    from oracle.pfpnet import pfpnet_image_loss
    rng = np.random.default_rng(G)
    B = 3
    rows = np.stack([TP.loss_rows(6375, 40 + b) for b in range(B)])
    gt = np.full((B, G, 5), -1.0, F32)
    for b, n in enumerate((G if G == 1 else 127, 0, G if G == 1 else 40)):
        gt[b] = TP.loss_gt(rng, 320, n, G)
    h = _loss_harness(L320, rows)
    got = h.loss("pfpnet", gt)
    for b in range(B):
        want, _ = pfpnet_image_loss(rows[b], [(a, c) for a, c, _ in L320], gt[b])
        assert abs(got[b] - want) <= 2e-5 * max(abs(want), 1.0), (b, got[b], want)
    for levels, r, g, what in TP.empty_cases():
        want, _ = pfpnet_image_loss(r, [(a, c) for a, c, _ in levels], g)
        got = _loss_harness(levels, r[None]).loss("pfpnet", g[None])
        assert abs(got[0] - want) <= 2e-5 * max(abs(want), 1.0), (what, got[0], want)


def test_loss_gradient_vs_restatement(built):
    """odt_pfpnet_loss_grad at B = 65 against autograd of train.pfpnet_image_loss: every element written (a NaN
    sentinel is overwritten), within 1e-5 of each image's max |gradient|; the loss agrees with the forward entry."""
    import test_pfpnet as TP
    from odt_b200.train import GraphTrainer
    B = 65
    rng = np.random.default_rng(9)
    rows = np.stack([TP.loss_rows(6375, 100 + b) for b in range(B)])
    gt = np.stack([TP.loss_gt(rng, 320, int(n), 16) for n in rng.integers(0, 17, B)])
    h = _loss_harness(L320, rows)
    sentinel = torch.full(h.head_buf.shape, float("nan"), device="cuda")
    loss, grad = h.loss_grad("pfpnet", gt, grad_out=sentinel)
    assert np.isfinite(grad).all()
    assert np.array_equal(loss, h.loss("pfpnet", gt))
    tr = _model(320, mode="test").trainer()
    tr._loss_kernels = None
    for b in range(0, B, 8):
        r = torch.from_numpy(rows[b]).cuda().requires_grad_(True)
        ref = tr.image_loss(r, gt[b])
        ref.backward()
        want = r.grad.cpu().numpy()
        assert abs(float(ref) - loss[b]) <= 2e-5 * max(abs(float(ref)), 1.0), b
        scale = max(np.abs(want).max(), 1e-12)
        assert np.abs(grad[b] - want).max() <= 1e-5 * scale, (b, np.abs(grad[b] - want).max(), scale)


def test_training_step_through_kernels_matches_restatement(built):
    """The CUDA trainer's data term is the kernels' (LossKernels); its autograd loss and parameter gradients agree with
    the restatement path on the same batch.  The row gradients agree to 1e-5 (test_loss_gradient_vs_restatement); the
    parameter gradients go back through PyTorch's fp32 convolutions, whose TF32 tensor-core backward rounds inputs
    to 10 mantissa bits, hence 2e-3 of the largest component."""
    import test_pfpnet as TP
    m = _model(128, mode="test")
    tr = m.trainer()
    assert tr._loss_kernels is not None
    rng = np.random.default_rng(3)
    img = _img(2, 128, seed=8)
    gt = np.stack([TP.loss_gt(rng, 128, 4), TP.loss_gt(rng, 128, 2)])
    rows = tr.forward_rows(img, True, [])
    loss_k, data_k = tr.total_loss(rows, gt)
    keep = tr._loss_kernels
    tr._loss_kernels = None
    loss_r, data_r = tr.total_loss(rows, gt)
    tr._loss_kernels = keep
    assert abs(float(data_k.detach()) - float(data_r.detach())) <= 2e-5 * max(abs(float(data_r)), 1.0)
    # a conv bias ahead of a training-mode BN has a gradient of zero up to rounding: not compared
    names = [k for k in tr.params if ("ODM/odm1" in k or "ARM/arm1" in k) and not k.endswith("/bias")]
    gk = torch.autograd.grad(data_k, [tr.params[k] for k in names], retain_graph=True, allow_unused=True)
    gr = torch.autograd.grad(data_r, [tr.params[k] for k in names], allow_unused=True)
    for k, a, b in zip(names, gk, gr):
        if b is None:
            continue
        assert float((a - b).abs().max()) <= 2e-3 * float(b.abs().max()) + 1e-9, k
    before = float(tr.params["ODM/odm1/conv2d_5/bias"][0])
    tr.step(img, gt, 1e-3)
    assert float(tr.params["ODM/odm1/conv2d_5/bias"][0]) != before and tr.global_step == 1
