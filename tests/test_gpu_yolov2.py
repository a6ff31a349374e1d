"""YOLOv2 on the GPU: the decode / NMS tail on oracle rows, the whole network at 480² and at a size that is not a
multiple of 32 against the oracle forward, the loss forward and gradient kernels (odt_yolo2_loss_*) at their matching
edges, the training step through the kernels, the pipelined stream and the convolution dispatch.  The oracle is
oracle/yolov2.py."""
import functools
from unittest import mock

import numpy as np
import pytest

import margins as MG
from helpers import BASE_CFG, assert_boxes_close

pytestmark = pytest.mark.gpu
F32 = np.float32
PRIORS = [[1.08, 1.19], [3.42, 4.41], [6.63, 11.38], [9.42, 5.11], [16.62, 10.52]]  # testYOLOv2.py:44
SCALES = dict(coord_scale=2.0, noobj_scale=0.5, obj_scale=5.0, class_scale=1.5)


def _priors(A):
    return (PRIORS + [[2.0, 2.5], [5.0, 3.0], [12.0, 14.0], [0.6, 0.7]])[:A]


def _cfg(A=5, nc=20, size=480, **over):
    c = dict(BASE_CFG)
    c.update(data_shape=[size, size, 3], coord_scale=1, noobj_scale=1, obj_scale=5., class_scale=1.,
             rescore_confidence=False, priors=_priors(A), num_classes=nc, nms_max_boxes=10)
    c.update(over)
    return c


def _model(A=5, nc=20, size=480, **over):
    import YOLOv2
    return YOLOv2.YOLOv2(_cfg(A, nc, size, **over), None)


def _img(b, h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (b, h, w, 3)).astype(F32)


def _rows(h, w, A, nc, B, seed, obj_mean=-1.0):
    rng = np.random.default_rng(seed)
    N = h * w * A
    r = (rng.standard_normal((B, N, nc + 5)) * 1.5).astype(F32)
    r[..., nc:] = (rng.standard_normal((B, N, 5)) * 0.5).astype(F32)
    r[..., nc + 4] = (rng.standard_normal((B, N)) * 2.0 + obj_mean).astype(F32)
    return r


def _as_pred(rows, h, w):
    return rows.reshape(rows.shape[0], h, w, -1)


# ------------------------------------------------------------------------------------------------------ tail ----
@pytest.mark.parametrize("A", [1, 5, 9])
@pytest.mark.parametrize("nc", [1, 20, 80, 128])
def test_tail_on_oracle_rows(built, A, nc):
    """YOLOv3's decode on one level with out_mul 32 and the priors in grid cells, then per-class NMS over every class:
    class ids and keep indices bit for bit against oracle/yolov2.py."""
    from odt_b200 import nets
    from odt_b200.engine import RowsHarness
    from oracle import yolov2 as OY
    h, w, B, thr, mb, iou = 15, 15, 3, 0.2, 10, 0.45
    rows = _rows(h, w, A, nc, B, seed=10 * A + nc)
    cfg = _cfg(A, nc, nms_score_threshold=thr, nms_max_boxes=mb, nms_iou_threshold=iou)
    hr = RowsHarness(nets.yolo2_tail(cfg), [(h, w, A)], rows)
    res, keep = hr.run(), hr.keep_indices()
    total = 0
    for b in range(B):
        s, bx, cid, kp = OY.yolo2_detect(_as_pred(rows, h, w), cfg["priors"], thr, mb, iou, image=b, num_classes=nc)
        np.testing.assert_array_equal(res[b][2], cid, err_msg="class ids")
        np.testing.assert_array_equal(keep[b], kp, err_msg="NMS keep indices")
        np.testing.assert_allclose(res[b][0], s, rtol=1e-6, atol=0)
        assert_boxes_close(res[b][1], bx)
        total += len(cid)
    assert total > 0
    if A > 1:
        assert any(np.any(k % A == A - 1) for k in keep)


# ------------------------------------------------------------------------------------------------------ loss ----
def _edge_gt(nc, G=8):
    """Image 0: a GT on a cell border, two GTs in one cell on one row, a GT past the grid (clamped), one matched to the
    last prior; image 1: no boxes."""
    gt = np.full((2, G, 5), -1.0, F32)
    gt[0, :6] = [[64.0, 96.0, 40.0, 30.0, 0], [70.0, 70.0, 20.0, 60.0, nc - 1], [71.0, 69.0, 22.0, 58.0, 0],
                 [480.0, 10.0, 50.0, 50.0, 2 % nc], [200.0, 300.0, 520.0, 340.0, 1 % nc],
                 [75.0, 72.0, 300.0, 250.0, 0]]
    return gt


def _full_gt(nc):
    """G = 128 rows: image 0 has no padding row, so its count is the index of the first minimum of column 0, put on
    the last row (127 boxes); image 1 holds 40 boxes."""
    rng = np.random.default_rng(nc)
    gt = np.full((2, 128, 5), -1.0, F32)
    for b, n in ((0, 128), (1, 40)):
        gt[b, :n, 0:2] = rng.uniform(1.0, 479.0, (n, 2))
        gt[b, :n, 2:4] = rng.uniform(8.0, 500.0, (n, 2))
        gt[b, :n, 4] = rng.integers(0, nc, n)
    gt[0, 127, 0] = 0.0
    return gt


def _oracle_loss(rows, gt, A, nc, b):
    from oracle import yolov2 as OY
    return OY.yolo2_image_loss(_as_pred(rows, 15, 15), _priors(A), gt[b], image=b, num_classes=nc, **SCALES)


@pytest.mark.parametrize("A,nc", [(5, 20), (1, 1), (9, 128)])
@pytest.mark.parametrize("which", ["edges", "full"])
def test_loss_forward_vs_oracle(built, A, nc, which):
    from odt_b200 import nets
    from odt_b200.engine import RowsHarness
    rows = _rows(15, 15, A, nc, 2, seed=A + nc)
    gt = _edge_gt(nc) if which == "edges" else _full_gt(nc)
    hr = RowsHarness(nets.yolo2_tail(_cfg(A, nc)), [(15, 15, A)], rows)
    got = hr.loss("yolo2", gt, **SCALES)
    for b in range(2):
        ref = _oracle_loss(rows, gt, A, nc, b)
        print("%s A=%d nc=%d image %d: loss gpu %.6f oracle %.6f" % (which, A, nc, b, got[b], ref))
        assert np.isfinite(got[b]) and abs(got[b] - ref) <= 2e-5 * max(abs(ref), 1.0)
    assert np.array_equal(hr.loss("yolo2", gt, **SCALES), got), "run-to-run deterministic"


@pytest.mark.parametrize("A,nc", [(5, 20), (1, 1), (9, 128)])
@pytest.mark.parametrize("which", ["edges", "full"])
def test_loss_gradient_vs_autograd(built, A, nc, which):
    """odt_yolo2_loss_grad: loss bit-identical to _fwd, the gradient within 1e-5 of the image's max |gradient| of the
    autograd restatement (train.yolo2_image_loss), bit-identical from run to run."""
    import torch
    from odt_b200 import nets
    from odt_b200.engine import RowsHarness
    from odt_b200.train import GraphTrainer
    rows = _rows(15, 15, A, nc, 2, seed=A + nc)
    gt = _edge_gt(nc) if which == "edges" else _full_gt(nc)
    hr = RowsHarness(nets.yolo2_tail(_cfg(A, nc)), [(15, 15, A)], rows)
    fwd = hr.loss("yolo2", gt, **SCALES)
    loss, grad = hr.loss_grad("yolo2", gt, **SCALES)
    assert np.array_equal(loss, fwd)
    loss2, grad2 = hr.loss_grad("yolo2", gt, **SCALES)
    assert np.array_equal(grad, grad2) and np.array_equal(loss, loss2)
    tr = GraphTrainer(_model(A, nc, **SCALES), "cpu")
    for b in range(2):
        r = torch.from_numpy(rows[b].copy()).requires_grad_(True)
        tr.image_loss(r, gt[b]).backward()
        want = r.grad.numpy()
        err, scale = float(np.abs(grad[b] - want).max()), float(np.abs(want).max())
        print("%s A=%d nc=%d image %d: grad max|err| %.3g of max %.3g" % (which, A, nc, b, err, scale))
        assert err <= 1e-5 * scale
    # the image without boxes: only objectness columns carry a gradient, on every row
    if which == "edges":
        nz = np.nonzero(grad[1])
        assert set(nz[1]) == {nc + 4} and len(nz[0]) == 15 * 15 * A


# ------------------------------------------------------------------------------------------------ full size ----
@functools.lru_cache(maxsize=None)
def _oracle_rows(size, A, nc):
    from oracle import yolov2 as OY
    probe = _model(A, nc, size, bn_init="trained")
    img = _img(1, size, size, seed=11)
    return img, OY.yolo2_rows(OY.yolov2_heads(probe.get_weights(), img), nc)


def _per_row(rows, geom, nc):
    from oracle import yolov2 as OY
    h, w = geom["grid"]
    conf, boxes = OY.yolo2_scores_boxes(_as_pred(np.asarray(rows, F32)[None], h, w), geom["priors"], num_classes=nc)
    return conf, boxes, np.ones(conf.shape[0], bool), None


@pytest.mark.parametrize("precision,row_tol,ds_tol", [("fp32", 2e-4, 1e-4), ("fp16", 5e-3, 3.5e-2)])
@pytest.mark.parametrize("size", [480, 200])
def test_full_network_decisions(built, size, precision, row_tol, ds_tol):
    """The whole network (the copy-free concat included) against the oracle forward, then margin-aware decision parity
    of the detections at a dense threshold (about 1 % of the candidates per class)."""
    A, nc = 5, 20
    img, ref = _oracle_rows(size, A, nc)
    g = -(-size // 32)
    geom = {"grid": (g, g), "priors": _priors(A)}
    vals = _per_row(ref[0], geom, nc)[0].reshape(-1)
    k = int(min(max(0.01 * ref.shape[1] * nc, 40), vals.size - 1))
    thr = float(np.partition(vals, vals.size - k)[vals.size - k])
    m = _model(A, nc, size, nms_score_threshold=thr, bn_init="trained", precision=precision)
    res = m.detect_batch(img)
    net = m.engine(1)
    rows = net.head_buf.cpu().numpy()
    assert rows.shape == ref.shape == (1, g * g * A, nc + 5) and np.isfinite(rows).all()
    scale, err = float(np.abs(ref).max()), float(np.abs(rows - ref).max())
    print("%d² %s: rows max|err| %.3g of max|ref| %.3g (%.2e rel), threshold %.4f"
          % (size, precision, err, scale, err / scale, thr))
    assert err <= row_tol * scale
    keep = net.tail.det_anchor.cpu().numpy()
    mb, iou = m.config["nms_max_boxes"], m.config["nms_iou_threshold"]
    with mock.patch.object(MG, "per_row", lambda kind, r, gm: _per_row(r, gm, nc)):
        rep = MG.compare_image("yolo", rows[0], ref[0], geom, res[0][2], keep[0, :len(res[0][2])], res[0][1], thr,
                               mb, iou, nc)
    tot = MG.summarize([rep])
    print("%d² %s: classes clean %d ambiguous %d identical %d; keeps oracle %d gpu %d common %d; ds %.3g"
          % (size, precision, tot["clean"], tot["ambiguous"], tot["identical"], tot["kept_oracle"], tot["kept_gpu"],
             tot["same_keeps"], tot["ds"]))
    assert tot["ds"] <= ds_tol, tot
    assert tot["kept_gpu"] > 0 and tot["same_keeps"] >= 0.5 * tot["kept_oracle"], tot


# ------------------------------------------------------------------------------------------------- training ----
def test_training_step_through_kernels_matches_restatement(built):
    """Two trainers from the same weights, one with the CUDA loss-and-gradient kernels (the default on CUDA), one on
    the autograd restatement: the same loss and BN moving statistics, and parameters within 5e-3 of the largest update
    (the bound and the measure of tests/test_gpu_loss_grad.py's training-step test)."""
    import torch
    from odt_b200.train import GraphTrainer
    size, B = 160, 2
    m = _model(5, 20, size, bn_init="trained", **SCALES)
    rng = np.random.default_rng(4)
    img = _img(B, size, size, seed=9)
    gt = np.full((B, 8, 5), -1.0, F32)
    gt[0, :5, 0:2] = rng.uniform(10, 150, (5, 2))
    gt[0, :5, 2:4] = rng.uniform(10, 200, (5, 2))
    gt[0, :5, 4] = rng.integers(0, 20, 5)
    kern, rest = GraphTrainer(m, "cuda"), GraphTrainer(m, "cuda")
    assert kern._loss_kernels is not None
    rest._loss_kernels = None
    p0 = {k: v.detach().clone() for k, v in kern.params.items()}
    lk, lr_ = kern.step(img, gt, 1e-3), rest.step(img, gt, 1e-3)
    assert np.isfinite(lk) and abs(lk - lr_) <= 1e-5 * abs(lr_), (lk, lr_)
    for k in kern.buffers:
        assert torch.equal(kern.buffers[k], rest.buffers[k]), k
    upd = max(float((rest.params[k] - p0[k]).abs().max()) for k in p0)
    diff = max(float((kern.params[k] - rest.params[k]).abs().max()) for k in p0)
    print("step loss: kernels %.7f restatement %.7f; max param difference %.3g = %.3g of the largest update"
          % (lk, lr_, diff, diff / upd))
    assert diff <= 5e-3 * upd


def test_train_one_epoch_and_checkpoint(built, tmp_path):
    """The driver's loop on synthetic batches: train_one_epoch, save_weight, load_weight, test_one_image."""
    import YOLOv2
    size = 160
    img = _img(2, size, size, seed=8)
    gt = _edge_gt(20)
    gt[..., :4] *= size / 480.0

    class It:
        def get_next(self):
            return img, gt
    provider = {"data_shape": [size, size, 3], "num_train": 4, "num_val": 0,
                "train_generator": ((lambda: None), It()), "val_generator": None}
    m = YOLOv2.YOLOv2(_cfg(5, 20, size, mode="train", batch_size=2, bn_init="trained"), provider)
    loss = m.train_one_epoch(1e-3)
    assert np.isfinite(loss) and m.global_step == 2
    path = m.save_weight("latest", str(tmp_path / "yolo2" / "test"))
    t = YOLOv2.YOLOv2(_cfg(5, 20, size, mode="test"), None)
    t.load_weight(path)
    assert t.global_step == 2
    res = t.test_one_image(img[:1])
    assert len(res) == 3 and res[1].shape[1:] == (4,)


# ------------------------------------------------------------------------------------------------ pipelines ----
def test_pipelined_and_single_graph_streams_agree(built, monkeypatch):
    import torch
    m = _model(5, 20, 160, precision="fp16", nms_score_threshold=0.05)
    batches = [_img(2, 160, 160, seed=s) for s in range(51, 56)]
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


# ------------------------------------------------------------------------------------------- dispatch audit ----
@pytest.mark.parametrize("A,nc", [(5, 20), (1, 1), (9, 128)])
def test_dispatch_audit(built, A, nc):
    """Every fp16 convolution of YOLOv2 480² runs a hand-written kernel: the image convolution on a stem kernel, every
    other one on odt_conv2d_f16_tc -- none on conv_direct; the concat has no op of its own: conv17 and the head's conv5
    store its two channel slices, and predictions reads all 1536 channels."""
    from odt_b200 import engine as E
    m = _model(A, nc, precision="fp16", bn_init="trained")
    assert len(m.detect_batch(_img(1, 480, 480, seed=2))) == 1
    net = m.engine(1)
    convs = [op for op in net.ops if isinstance(op, E.ConvOp)]
    direct = [op.kernel for op in convs if not (op.is_image or op.use_tc)]
    assert not direct, direct
    assert not [op for op in net.ops if not isinstance(op, (E.ConvOp, E.PoolOp))]
    pred = [op for op in convs if op.head is not None]
    assert len(pred) == 1 and pred[0].p.Cin == 1536 and pred[0].p.in_ld == 1536 and pred[0].p.Cout == (nc + 5) * A
    byname = {op.kernel: op for op in convs}
    assert byname["backone/conv17/kernel"].pre[2].c0 == 0 and byname["head/conv5/kernel"].pre[2].c0 == 512
    assert byname["head/conv5/kernel"].p.out0 is None
    assert np.isfinite(net.head_buf.cpu().numpy()).all()
