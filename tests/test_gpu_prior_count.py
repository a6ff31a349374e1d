"""YOLOv3 with 1 to 9 priors per level on the GPU: the decode / NMS tail and the loss forward on restated rows, whole
networks at 416² against the oracle forward, the training step, the pipelined stream and the convolution dispatch.
The restatement is tests/prior_count_ref.py (equal to the oracle at 3 priors, tests/test_prior_count.py)."""
import functools

import numpy as np
import pytest

import class_count_rows as CR
import margins as MG
import prior_count_ref as PR
from helpers import assert_boxes_close, model_cfg

pytestmark = pytest.mark.gpu
F32 = np.float32


def _img(b, h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (b, h, w, 3)).astype(F32)


def _cfg(A, nc, **over):
    return model_cfg("yolov3", num_classes=nc, num_priors=A, priors=PR.priors_for(A), **over)


def _model(A, nc, **over):
    import YOLOv3
    return YOLOv3.YOLOv3(_cfg(A, nc, **over), None)


def _rows(levels, nc, B, seed, obj_mean=-1.0):
    """Random candidate rows [B, N, nc + 5]: class logits around 0, box columns small, objectness mostly low."""
    rng = np.random.default_rng(seed)
    N = sum(h * w * a for h, w, a in levels)
    r = (rng.standard_normal((B, N, nc + 5)) * 1.5).astype(F32)
    r[..., nc:] = (rng.standard_normal((B, N, 5)) * 0.5).astype(F32)
    r[..., nc + 4] = (rng.standard_normal((B, N)) * 2.0 + obj_mean).astype(F32)
    return r


GRID = [(A, nc) for A in (1, 2, 5, 9) for nc in (1, 20, 80)]


@pytest.mark.parametrize("A,nc", GRID)
def test_tail_on_restated_rows(built, A, nc):
    """Decode + NMS at A priors against the restatement: class ids and keep indices bit for bit.  The small levels
    do not end on 32-row boundaries, so warps straddle levels and images."""
    from odt_b200 import nets
    from odt_b200.engine import RowsHarness
    levels, B, thr, mb, iou = [(5, 5, A), (3, 3, A), (2, 2, A)], 5, 0.2, 10, 0.45
    rows = _rows(levels, nc, B, seed=10 * A + nc)
    cfg = _cfg(A, nc, nms_score_threshold=thr, nms_max_boxes=mb, nms_iou_threshold=iou)
    h = RowsHarness(nets.yolo_tail(cfg), levels, rows)
    res, keep = h.run(), h.keep_indices()
    preds = CR.rows_to_levels(rows, levels, "yolo", nc)
    total = 0
    for b in range(B):
        s, bx, cid, kp = PR.yolo_detect(preds, cfg["priors"], thr, mb, iou, image=b, num_classes=nc)
        np.testing.assert_array_equal(res[b][2], cid, err_msg="class ids")
        np.testing.assert_array_equal(keep[b], kp, err_msg="NMS keep indices")
        np.testing.assert_allclose(res[b][0], s, rtol=1e-6, atol=0)
        assert_boxes_close(res[b][1], bx)
        total += len(cid)
    assert total > 0
    if A > 1:  # boxes of the last prior of a cell are decoded and kept
        assert any(np.any(k % A == A - 1) for k in keep)


def _loss_gt(rng, size, nc, B=2, G=14):
    """GT boxes from a few pixels to three times the image: at each A of GRID the last prior of some level is a best
    match (tests/test_prior_count.py::test_ground_truth_reaches_every_prior checks the same sets)."""
    gt = np.full((B, G, 5), -1.0, F32)
    for b in range(B):
        n = 12 - 2 * b  # padded: the GT count is the index of the first -1 row
        gt[b, :n, 0:2] = rng.uniform(0.15 * size, 0.85 * size, (n, 2))
        gt[b, :n, 2:4] = np.geomspace(0.04 * size, 3.0 * size, n)[:, None] * rng.uniform(0.7, 1.4, (n, 2))
        gt[b, :n, 4] = rng.integers(0, nc, n)
    gt[0, 0, 4] = nc - 1
    return gt


@pytest.mark.parametrize("A,nc", GRID)
def test_loss_forward_vs_restatement(built, A, nc):
    from odt_b200 import nets
    from odt_b200.engine import RowsHarness
    size = 160
    levels = [(5, 5, A), (10, 10, A), (20, 20, A)]
    rng = np.random.default_rng(A)
    rows = _rows(levels, nc, 2, seed=7 + A + nc)
    gt = _loss_gt(rng, size, nc)
    priors = PR.priors_for(A)
    assert A - 1 in {p for b in range(2) for _, p in PR.assignment(priors, gt[b])}
    h = RowsHarness(nets.yolo_tail(_cfg(A, nc)), levels, rows)
    kw = dict(coord_scale=2, noobj_scale=0.5, obj_scale=5, class_scale=1.5)
    got = h.loss("yolo", gt, **kw)
    for b in range(2):
        ref = PR.yolo_image_loss(CR.rows_to_levels(rows, levels, "yolo", nc), priors, gt[b], image=b, num_classes=nc,
                                 **kw)
        print("A=%d nc=%d image %d: loss gpu %.6f restatement %.6f" % (A, nc, b, got[b], ref))
        assert abs(got[b] - ref) <= 2e-5 * max(abs(ref), 1.0)
    assert np.array_equal(h.loss("yolo", gt, **kw), got), "run-to-run deterministic"


# ------------------------------------------------------------------------------- full size --
@functools.lru_cache(maxsize=None)
def _oracle_rows(A, nc, B):
    """The oracle network's rows at 416² (seeded weights of the A-prior, nc-class model), shared by both precisions."""
    from oracle import nets as ON
    from oracle import tails as OT
    probe = _model(A, nc, bn_init="trained", data_shape=[416, 416, 3])
    img = _img(B, 416, 416, seed=11)
    ref = OT.yolo_rows(ON.yolov3_heads(probe.get_weights(), img, num_classes=nc, num_priors=A), num_classes=nc)
    return img, ref, list(probe._build_spec().levels), probe.config["priors"]


@pytest.mark.parametrize("precision,row_tol,ds_tol", [("fp32", 2e-4, 1e-4), ("fp16", 5e-3, 3.5e-2)])
@pytest.mark.parametrize("A,nc", [(5, 20), (5, 80), (9, 20), (9, 80)])
def test_full_size_end_to_end_decisions(built, A, nc, precision, row_tol, ds_tol):
    """The pattern of test_gpu_class_count.py::test_full_size_80_classes_end_to_end_decisions at 5 and 9 priors: rows
    against the oracle forward within the class-count bounds, then margin-aware decision parity at a dense threshold
    (about 1 % of the candidates per class)."""
    B = 1
    img, ref, levels, priors = _oracle_rows(A, nc, B)
    geom = {"levels": levels, "priors": priors}
    vals = np.concatenate([PR.per_row(r, geom, nc)[0].reshape(-1) for r in ref])
    k = int(min(max(0.01 * ref.shape[1] * B * nc, 40), vals.size - 1))
    thr = float(np.partition(vals, vals.size - k)[vals.size - k])
    m = _model(A, nc, nms_score_threshold=thr, bn_init="trained", precision=precision, data_shape=[416, 416, 3])
    res = m.detect_batch(img)
    net = m.engine(B)
    rows = net.head_buf.cpu().numpy()
    assert rows.shape == ref.shape == (B, (13 * 13 + 26 * 26 + 52 * 52) * A, nc + 5) and np.isfinite(rows).all()
    scale, err = float(np.abs(ref).max()), float(np.abs(rows - ref).max())
    print("A=%d nc=%d %s: rows max|err| %.3g of max|ref| %.3g (%.2e rel), threshold %.4f"
          % (A, nc, precision, err, scale, err / scale, thr))
    assert err <= row_tol * scale
    keep_all = net.tail.det_anchor.cpu().numpy()
    mb, iou = m.config["nms_max_boxes"], m.config["nms_iou_threshold"]
    reps = [PR.compare_image(rows[b], ref[b], geom, res[b][2], keep_all[b, :len(res[b][2])], res[b][1], thr, mb, iou,
                             nc) for b in range(B)]
    tot = MG.summarize(reps)
    cc = net.tail.cand_count.cpu().numpy()
    print("A=%d nc=%d %s: candidates/class mean %.0f max %d; classes clean %d ambiguous %d (reasons %s) identical %d "
          "of %d; keeps oracle %d gpu %d common %d; ds %.3g di %.3g; common-keep box err %.3g px"
          % (A, nc, precision, cc.mean(), cc.max(), tot["clean"], tot["ambiguous"], tot["reasons"], tot["identical"],
             nc * B, tot["kept_oracle"], tot["kept_gpu"], tot["same_keeps"], tot["ds"], tot["di"], tot["box_err"]))
    assert cc.mean() >= 10
    assert tot["ds"] <= ds_tol, tot
    assert tot["kept_gpu"] > 0 and tot["same_keeps"] >= 0.5 * tot["kept_oracle"], tot


# -------------------------------------------------------------------------------- training --
def test_training_step_on_gpu_5_priors(built):
    """At A = 5: the autograd loss agrees with the CUDA loss forward on the same rows, the step moves the variables,
    the inference engine runs on the updated weights."""
    import torch
    import YOLOv3
    from odt_b200 import nets
    from odt_b200.engine import RowsHarness
    A, nc, size = 5, 20, 160
    rng = np.random.default_rng(3)
    img = _img(2, size, size, seed=8)
    gt = _loss_gt(rng, size, nc)

    class It:
        def get_next(self):
            return img, gt
    provider = {"num_train": 2, "num_val": 0, "train_generator": ((lambda: None), It()), "val_generator": None}
    m = YOLOv3.YOLOv3(_cfg(A, nc, mode="train", batch_size=2, bn_init="trained", data_shape=[size, size, 3]),
                      provider)
    tr = m.trainer()
    assert tr.device.type == "cuda" and tr.row == nc + 5
    rows = tr.forward_rows(img)
    per = [float(tr.image_loss(rows[b], gt[b])) for b in range(2)]
    hrn = RowsHarness(nets.yolo_tail(m.config), list(tr.net.levels), rows.detach().cpu().numpy())
    kw = {k: m.config[k] for k in ("coord_scale", "noobj_scale", "obj_scale", "class_scale")}
    got = hrn.loss("yolo", gt, **kw)
    for b in range(2):
        print("A=5 image %d: autograd %.6f, CUDA %.6f" % (b, per[b], got[b]))
        assert abs(per[b] - got[b]) <= 1e-4 * max(abs(per[b]), 1.0)
    w0 = {k: v.detach().clone() for k, v in tr.params.items()}
    loss = m.train_one_epoch(1e-3)
    assert np.isfinite(loss) and m.global_step == 1
    changed = sum(int(not torch.equal(w0[k], tr.params[k].detach())) for k in w0)
    assert changed >= 0.95 * len(w0)
    assert len(m.detect_batch(img[:1])) == 1


# ------------------------------------------------------------------------------- pipelines --
@pytest.mark.parametrize("A,nc", [(5, 20), (9, 80)])
def test_pipelined_and_single_graph_streams_agree(built, monkeypatch, A, nc):
    """The two-stage pipeline against the one-graph-per-step stream and the synchronous call at 5 and 9 priors."""
    import torch
    m = _model(A, nc, precision="fp16", data_shape=[160, 160, 3], nms_score_threshold=0.05)
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


# -------------------------------------------------------------------------- dispatch audit --
@pytest.mark.parametrize("A", [1, 2, 5, 9])
@pytest.mark.parametrize("nc", [1, 20, 80, 128])
def test_dispatch_audit(built, A, nc):
    """Every fp16 convolution of YOLOv3 416² at A priors and nc classes runs a hand-written kernel: the image
    convolution on a stem kernel, every other one on odt_conv2d_f16_tc -- none on conv_direct.  The prediction convs
    range from 6 (A = 1, one class) to 1 197 channels (A = 9, 128 classes)."""
    from odt_b200 import engine as E
    m = _model(A, nc, precision="fp16", bn_init="trained", data_shape=[416, 416, 3])
    res = m.detect_batch(_img(1, 416, 416, seed=2))
    assert len(res) == 1
    net = m.engine(1)
    convs = [op for op in net.ops if isinstance(op, E.ConvOp)]
    direct = [op.kernel for op in convs if not (op.is_image or op.use_tc)]
    assert not direct, direct
    assert {op.p.Cout for op in convs if op.head is not None} == {(nc + 5) * A}
    assert np.isfinite(net.head_buf.cpu().numpy()).all()
