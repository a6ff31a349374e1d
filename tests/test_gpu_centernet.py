"""CenterNet on the GPU: the DLA join kernel against float64, the peak + top-k tail bit for bit on oracle rows, the
network against oracle/centernet.py in fp32 and fp16, the loss and gradient kernels against the oracle and the
restatement, the training step through them, pipelined against single-graph streams, and the convolution dispatch."""
import numpy as np
import pytest
import torch

import test_centernet as TC

pytestmark = pytest.mark.gpu
F32 = np.float32


def _model(size=384, **over):
    c = TC.cfg(input_size=size, device="cuda")
    c.update(over)
    import CenterNet
    return CenterNet.CenterNet(c, None)


def _img(b, s, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (b, s, s, 3)).astype(F32)


# ---------------------------------------------------------------------------------------------- DLA join ----
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("H,W,pooled", [(12, 12, 1), (7, 5, 1), (1, 3, 1), (9, 6, 0)])
def test_dla_join(built, prec, H, W, pooled):
    from odt_b200 import lib
    L = lib.load()
    tdt, code, tol = {"fp32": (torch.float32, 1, 1e-6), "fp16": (torch.float16, 0, 2e-3)}[prec]
    C, ld = 72, 128
    rng = np.random.default_rng(H * W + pooled)
    a = torch.from_numpy(rng.standard_normal((2, H, W, ld)).astype(F32)).cuda().to(tdt)
    b = torch.from_numpy(rng.standard_normal((2, H, W, 96)).astype(F32)).cuda().to(tdt)
    OH, OW = ((H + 1) // 2, (W + 1) // 2) if pooled else (H, W)
    out = torch.full((2, OH, OW, ld), 3.0, dtype=tdt, device="cuda")
    lib.check(L.odt_dla_join(a.data_ptr(), b.data_ptr(), out.data_ptr(), code, 2, H, W, C, ld, 96, ld, pooled,
                             torch.cuda.current_stream().cuda_stream))
    aq, bq = a.double().cpu().numpy()[..., :C], b.double().cpu().numpy()[..., :C]
    if pooled:
        exp = np.zeros((2, OH, OW, C))
        for i in range(OH):
            for j in range(OW):
                exp[:, i, j] = (aq[:, 2 * i:2 * i + 2, 2 * j:2 * j + 2].reshape(2, -1, C).max(1)
                                + bq[:, 2 * i:2 * i + 2, 2 * j:2 * j + 2].reshape(2, -1, C).mean(1))
    else:
        exp = aq + bq
    got = out.double().cpu().numpy()
    np.testing.assert_allclose(got[..., :C], exp, rtol=tol, atol=tol)
    assert np.all(got[..., C:] == 3.0), "stores past C"


# --------------------------------------------------------------------------------------------------- tail ----
def _tail_rows(rng, h, w, nc, kind):
    """Rows [h*w, nc + 4]: 'sparse' a few hundred peaks, 'plateau' saturated logits in blocks (every cell a peak) and
    exact ties, 'none' nothing above the threshold."""
    r = np.zeros((h * w, nc + 4), F32)
    r[:, :nc] = rng.standard_normal((h * w, nc)) * 1.5 - 3.0
    if kind == "plateau":
        cells = rng.choice(h * w, h * w // 6, replace=False)
        r[cells, rng.integers(0, nc, len(cells))] = 60.0
        tie = rng.choice(h * w, 40, replace=False)
        r[tie, :] = -30.0
        r[tie, 0] = 0.5
    if kind == "none":
        r[:, :nc] = -20.0
    r[:, nc:nc + 2] = rng.uniform(0, 1, (h * w, 2))
    r[:, nc + 2:] = rng.uniform(0, 40, (h * w, 2))
    return r


@pytest.mark.parametrize("size,B,nc,K,thr,kind", [
    (384, 1, 20, 100, 0.1, "sparse"), (384, 15, 20, 100, 0.1, "plateau"), (384, 15, 80, 1024, 0.05, "sparse"),
    (512, 1, 128, 100, 0.1, "plateau"), (512, 2, 1, 1024, 0.01, "plateau"), (384, 3, 20, 7, 0.3, "sparse"),
    (384, 2, 20, 100, 0.1, "none")])
def test_tail_on_oracle_rows(built, size, B, nc, K, thr, kind):
    from odt_b200.engine import RowsHarness
    from odt_b200.nets import centernet_tail
    from oracle.centernet import centernet_tail as ref_tail
    h = size // 4
    rng = np.random.default_rng(size + B + nc)
    rows = np.stack([_tail_rows(rng, h, h, nc, kind) for _ in range(B)])
    tail = centernet_tail(TC.cfg(num_classes=nc, score_threshold=thr, top_k_results_output=K))
    hr = RowsHarness(tail, [(h, h, 1)], rows)
    res = hr.run()
    keeps = hr.keep_indices()
    more = 0
    for b in range(B):
        s, bx, cid, k = ref_tail(rows[b], h, h, thr, K)
        assert np.array_equal(keeps[b], k), b
        assert np.array_equal(res[b][0], s) and np.array_equal(res[b][1], bx) and np.array_equal(res[b][2], cid), b
        more += len(k) == K
    if kind == "none":
        assert all(len(r[0]) == 0 for r in res)
    elif K < 1000:
        assert more > 0, "the case must have more peaks than K"


# ------------------------------------------------------------------------------------------------ network ----
@pytest.mark.parametrize("size,prec,tol", [(384, "fp32", 2e-4), (384, "fp16", 2e-2), (512, "fp16", 2e-2)])
def test_full_network_vs_oracle(built, size, prec, tol):
    """Head rows within tol x max|ref| of the oracle forward; the GPU tail on the GPU's own rows equals the oracle tail
    on them bit for bit."""
    from oracle.centernet import centernet_heads, centernet_rows, centernet_tail
    m = _model(size, precision=prec, score_threshold=0.05)
    img = _img(1, size, seed=size)
    res = m.detect_batch(img)
    net = m.engine(1)
    rows = net.head_buf.cpu().numpy()
    ref = centernet_rows(centernet_heads(m.get_weights(), img))
    assert rows.shape == ref.shape == (1, (size // 4) ** 2, 24)
    scale = float(np.abs(ref).max())
    err = float(np.abs(rows - ref).max())
    print("%d %s rows max|err| %.4g of max|ref| %.4g" % (size, prec, err, scale))
    assert err <= tol * scale, (err, scale)
    s, bx, cid, k = centernet_tail(rows[0], size // 4, size // 4, 0.05, 100)
    assert np.array_equal(res[0][0], s) and np.array_equal(res[0][1], bx) and np.array_equal(res[0][2], cid)
    assert len(s) > 0


def test_pipelined_and_single_graph_streams_agree(built, monkeypatch):
    m = _model(128, precision="fp16", score_threshold=0.05)
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


@pytest.mark.parametrize("size", [384, 512])
def test_dispatch_audit(built, size):
    """No 3x3 convolution with 32 or more input channels runs on conv_direct: every fp16 layer but the 7x7 image stem
    is on odt_conv2d_f16_tc, the transposed convolutions as phase convolutions with ReLU in the epilogue."""
    from odt_b200 import engine as E
    m = _model(size, precision="fp16")
    m.detect_batch(_img(1, size, seed=2))
    net = m.engine(1)
    convs = [op for op in net.ops if isinstance(op, E.ConvOp)]
    direct = [op.kernel for op in convs if not (op.is_image or op.use_tc)]
    assert not direct, direct
    assert [op.kernel for op in convs if op.is_image] == ["backone/conv2d/kernel"]
    phase = [op for op in convs if isinstance(op, E.PhaseConvOp)]
    assert len(phase) == 6 and all(op.p.Cout == 1024 and op.act == "relu" for op in phase)
    kinds = {type(op).__name__ for op in net.ops}
    assert kinds == {"ConvOp", "PhaseConvOp", "PixelShuffleOp", "PoolOp", "DlaJoinOp"}
    assert sum(isinstance(op, E.DlaJoinOp) for op in net.ops) == 6 + 3
    assert np.isfinite(net.head_buf.cpu().numpy()).all()


# ------------------------------------------------------------------------------------------------ loss kernels ----
def _harness(rows, h):
    from odt_b200.engine import RowsHarness
    from odt_b200.nets import centernet_tail
    return RowsHarness(centernet_tail(TC.cfg(num_classes=rows.shape[2] - 4)), [(h, h, 1)], rows)


@pytest.mark.parametrize("G", [1, 128])
def test_loss_forward_vs_oracle(built, G):
    """odt_centernet_loss_fwd at 384² against the float64 oracle, G = 1 and a full 128-row block, plus the CPU edge
    cases (no boxes, two GTs on one cell, a box smaller than a cell, one class only)."""
    from oracle.centernet import centernet_image_loss
    rng = np.random.default_rng(G)
    h, B = 96, 3
    rows = np.stack([TC.loss_rows(h * h, 20, 40 + b) for b in range(B)])
    gt = np.stack([TC.loss_gt(rng, 384, n, G) for n in (G if G == 1 else 127, 0, G)])
    got = _harness(rows, h).loss("centernet", gt)
    for b in range(B):
        want, _ = centernet_image_loss(rows[b], h, h, gt[b])
        assert abs(got[b] - want) <= 1e-5 * max(abs(want), 1.0), (b, got[b], want)
    for name, r, g in TC.loss_cases():
        want, _ = centernet_image_loss(r, 24, 24, g)
        got = _harness(r[None], 24).loss("centernet", g[None])
        assert abs(got[0] - want) <= 1e-5 * max(abs(want), 1.0), (name, got[0], want)


def test_loss_gradient_vs_restatement(built):
    """odt_centernet_loss_grad at B = 15 against autograd of the restatement: every element written (a NaN sentinel is
    overwritten), within 1e-5 of each image's max |gradient|; bit-identical run to run and image by image alone."""
    B, h = 15, 96
    rng = np.random.default_rng(9)
    rows = np.stack([TC.loss_rows(h * h, 20, 100 + b) for b in range(B)])
    gt = np.stack([TC.loss_gt(rng, 384, int(n), 16) for n in rng.integers(0, 17, B)])
    gt[3, :2] = [[40.0, 40.0, 30.0, 20.0, 5], [41.0, 42.0, 10.0, 12.0, 5]]  # two GTs on one cell
    hr = _harness(rows, h)
    sentinel = torch.full(hr.head_buf.shape, float("nan"), device="cuda")
    loss, grad = hr.loss_grad("centernet", gt, grad_out=sentinel)
    assert np.isfinite(grad).all()
    loss2, grad2 = hr.loss_grad("centernet", gt, grad_out=torch.zeros_like(sentinel))
    assert np.array_equal(loss, loss2) and np.array_equal(grad, grad2)
    assert np.array_equal(loss, hr.loss("centernet", gt))
    for b in (0, 3, 14):
        l1, g1 = _harness(rows[b:b + 1], h).loss_grad("centernet", gt[b:b + 1])
        assert np.array_equal(l1[0], loss[b]) and np.array_equal(g1[0], grad[b]), b
    tr = _model(384).trainer()
    tr._loss_kernels = None
    for b in range(0, B, 4):
        r = torch.from_numpy(rows[b]).cuda().requires_grad_(True)
        ref = tr.image_loss(r, gt[b])
        ref.backward()
        want = r.grad.cpu().numpy()
        assert abs(float(ref) - loss[b]) <= 2e-5 * max(abs(float(ref)), 1.0), b
        scale = max(np.abs(want).max(), 1e-12)
        assert np.abs(grad[b] - want).max() <= 1e-5 * scale, (b, np.abs(grad[b] - want).max(), scale)


def test_training_step_through_kernels_matches_restatement(built):
    m = _model(128, mode="test")
    tr = m.trainer()
    assert tr._loss_kernels is not None
    rng = np.random.default_rng(3)
    img = _img(2, 128, seed=8)
    gt = np.stack([TC.loss_gt(rng, 128, 4, 5), TC.loss_gt(rng, 128, 2, 5)])
    rows = tr.forward_rows(img, True, [])
    _, data_k = tr.total_loss(rows, gt)
    keep = tr._loss_kernels
    tr._loss_kernels = None
    _, data_r = tr.total_loss(rows, gt)
    tr._loss_kernels = keep
    assert abs(float(data_k.detach()) - float(data_r.detach())) <= 2e-5 * max(abs(float(data_r)), 1.0)
    before = float(tr.params["center_detector/conv2d/bias"][0])
    tr.step(img, gt, 1e-3)
    assert float(tr.params["center_detector/conv2d/bias"][0]) != before and tr.global_step == 1
