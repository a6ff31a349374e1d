"""YOLOv3 and FCOS at class counts other than 20 on the GPU: the decode / NMS tail on oracle rows of num_classes + 5
floats (mask-word boundaries 31 / 32 / 33, 80, 128, FCOS with one class), whole networks at 80 classes against the
oracle forward, the loss forwards, the training step, the pipelined stream and the convolution dispatch."""
import numpy as np
import pytest

import class_count_rows as CR
import margins as MG
from helpers import YOLO_PRIORS, assert_boxes_close, model_cfg

pytestmark = pytest.mark.gpu
F32 = np.float32


def _img(b, h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (b, h, w, 3)).astype(F32)


def _model(family, nc, **over):
    import FCOS
    import YOLOv3
    if family == "yolov3":
        return YOLOv3.YOLOv3(model_cfg("yolov3", num_classes=nc, **over), None)
    return FCOS.FCOS(model_cfg("fcos", num_classes=nc, **over), None)


def _rows(levels, nc, B, seed, obj_mean=-1.0):
    """Random candidate rows [B, N, nc + 5]: class logits around 0, box columns small, the objectness / centre-ness
    column (index nc + 4 for YOLO, nc for FCOS: both set) mostly low, so the early-out and the class loop both run."""
    rng = np.random.default_rng(seed)
    N = sum(h * w * a for h, w, a in levels)
    r = (rng.standard_normal((B, N, nc + 5)) * 1.5).astype(F32)
    r[..., nc:] = (rng.standard_normal((B, N, 5)) * 0.5).astype(F32)
    r[..., nc] = (rng.standard_normal((B, N)) * 2.0 + obj_mean).astype(F32)
    r[..., nc + 4] = (rng.standard_normal((B, N)) * 2.0 + obj_mean).astype(F32)
    return r


def _tail(family, nc, thr, mb, iou):
    from odt_b200 import nets
    cfg = model_cfg(family, num_classes=nc, nms_score_threshold=thr, nms_max_boxes=mb, nms_iou_threshold=iou)
    return nets.yolo_tail(cfg) if family == "yolov3" else nets.fcos_tail(cfg)


def _oracle(family, rows, levels, nc, thr, mb, iou, image):
    from oracle import tails as OT
    if family == "yolov3":
        preds = CR.rows_to_levels(rows, levels, "yolo", nc)
        return OT.yolo_detect(preds, YOLO_PRIORS, thr, mb, iou, image=image, num_classes=nc)
    heads = CR.rows_to_levels(rows, levels, "fcos", nc)
    return OT.fcos_detect(heads, thr, mb, iou, image=image, num_classes=nc)


def _check(res, keep, exp):
    s, bx, cid, kp = exp
    np.testing.assert_array_equal(res[2], cid, err_msg="class ids")
    np.testing.assert_array_equal(keep, kp, err_msg="NMS keep indices")
    np.testing.assert_allclose(res[0], s, rtol=1e-6, atol=0)
    assert_boxes_close(res[1], bx)


# small geometries whose images do not end on a 32-row boundary: warps straddle images
LEVELS = {"yolov3": [(5, 5, 3), (3, 3, 3), (2, 2, 3)],
          "fcos": [(9, 9, 1), (5, 5, 1), (3, 3, 1), (2, 2, 1), (1, 1, 1)]}


@pytest.mark.parametrize("nc", [1, 31, 32, 33, 80, 128])
@pytest.mark.parametrize("family", ["yolov3", "fcos"])
def test_tail_on_oracle_rows(built, family, nc):
    from odt_b200.engine import RowsHarness
    if family == "fcos" and nc == 1:
        pytest.skip("FCOS with one class visits no class: test_fcos_one_class_returns_empty_records")
    levels, B, thr, mb, iou = LEVELS[family], 5, 0.2, 10, 0.45
    rows = _rows(levels, nc, B, seed=nc)
    h = RowsHarness(_tail(family, nc, thr, mb, iou), levels, rows)
    res, keep = h.run(), h.keep_indices()
    total = 0
    for b in range(B):
        _check(res[b], keep[b], _oracle(family, rows, levels, nc, thr, mb, iou, b))
        total += len(res[b][2])
    assert total > 0
    if (nc - 1 if family == "fcos" else nc) > 32:  # classes of the upper mask words are decoded and kept
        assert any(np.any(r[2] >= 32) for r in res)
    res2 = h.run()
    for b in range(B):
        for a, c in zip(res[b], res2[b]):
            np.testing.assert_array_equal(a, c)


@pytest.mark.parametrize("nc", [33, 80, 128])
@pytest.mark.parametrize("family", ["yolov3", "fcos"])
def test_tail_dense_lists_longer_than_smem(built, family, nc):
    """Every row passes for every class (threshold 0): 1 728 (YOLO) / 1 600 (FCOS) candidates per class, more than the
    1 024-key shared-memory window, so the NMS runs its prefilter / full-list paths in every class."""
    from odt_b200.engine import RowsHarness
    levels = [(24, 24, 3)] if family == "yolov3" else [(40, 40, 1)] + [(1, 1, 1)] * 4
    B, thr, mb, iou = 2, 0.0, 25, 0.6
    rows = _rows(levels, nc, B, seed=100 + nc, obj_mean=1.0)
    h = RowsHarness(_tail(family, nc, thr, mb, iou), levels, rows)
    res, keep = h.run(), h.keep_indices()
    N = rows.shape[1]
    assert np.all(h.tail.cand_count.cpu().numpy() == N) and N > 1024
    for b in range(B):
        _check(res[b], keep[b], _oracle(family, rows, levels, nc, thr, mb, iou, b))


def test_fcos_one_class_returns_empty_records(built):
    """num_classes = 1: the reference's NMS loop visits range(0) classes, so every image has no detection; the packed
    record is [B, 2] = (count 0, overflow 0)."""
    from odt_b200.engine import RowsHarness
    levels = LEVELS["fcos"]
    rows = _rows(levels, 1, 3, seed=5, obj_mean=2.0)
    h = RowsHarness(_tail("fcos", 1, 0.0, 10, 0.5), levels, rows)
    h.tail.rec.fill_(7.0)
    res = h.run()
    assert h.tail.D == 0 and tuple(h.tail.rec.shape) == (3, 2)
    np.testing.assert_array_equal(h.tail.rec.cpu().numpy(), np.zeros((3, 2), F32))
    assert np.all(h.tail.det_count.cpu().numpy() == 0) and int(h.tail.status.item()) == 0
    assert int(h.tail.cand_count.sum().item()) > 0  # the one class still decodes; no class is visited by NMS
    for r in res:
        assert r[0].shape == (0,) and r[1].shape == (0, 4) and r[2].shape == (0,)


# ------------------------------------------------------------------ full size, 80 classes --
FULL = {"yolov3": (416, 2), "fcos": (1024, 1)}


def _oracle_rows(family, weights, img, nc):
    from oracle import nets as ON
    from oracle import tails as OT
    if family == "yolov3":
        return OT.yolo_rows(ON.yolov3_heads(weights, img, num_classes=nc), num_classes=nc)
    return OT.fcos_rows(ON.fcos_heads(weights, img, num_classes=nc))


@pytest.mark.parametrize("precision,row_tol,ds_tol", [("fp32", 2e-4, 1e-4), ("fp16", 5e-3, 3.5e-2)])
@pytest.mark.parametrize("family", ["yolov3", "fcos"])
def test_full_size_80_classes_end_to_end_decisions(built, family, precision, row_tol, ds_tol):
    """The pattern of test_gpu_models.py::test_full_size_end_to_end_decisions at 80 classes: rows against the oracle
    forward, then margin-aware decision parity at a dense threshold (about 1 % of the candidates per class)."""
    nc = 80
    size, B = FULL[family]
    if family == "fcos" and precision == "fp16":
        row_tol = 1.5e-2  # as at 20 classes: GroupNorm re-normalises fp16-stored activations in every layer
    # The ds bounds are those of 20 classes.  Measured on an H100 80GB HBM3 (700 W), seed 11: ds 2.54e-2 (YOLOv3 fp16),
    # 2.3e-4 (FCOS fp16), 4.7e-5 / 1.2e-7 in fp32; rows 1.7e-3 / 1.1e-2 of max|ref| in fp16.
    over = dict(bn_init="trained", precision=precision, data_shape=[size, size, 3])
    img = _img(B, size, size, seed=11)
    probe = _model(family, nc, **over)
    ref = _oracle_rows(family, probe.get_weights(), img, nc)
    spec = probe._build_spec()
    mkind = "yolo" if family == "yolov3" else "fcos"
    geom = {"levels": list(spec.levels)}
    if family == "yolov3":
        geom["priors"] = probe.config["priors"]
    vals = np.concatenate([CR.per_row(mkind, r, geom, nc)[0].reshape(-1) for r in ref])
    k = int(min(max(0.01 * ref.shape[1] * B * nc, 40), vals.size - 1))
    thr = float(np.partition(vals, vals.size - k)[vals.size - k])
    m = _model(family, nc, nms_score_threshold=thr, **over)
    res = m.detect_batch(img)
    net = m.engine(B)
    rows = net.head_buf.cpu().numpy()
    assert rows.shape == ref.shape == (B, ref.shape[1], nc + 5) and np.isfinite(rows).all()
    scale, err = float(np.abs(ref).max()), float(np.abs(rows - ref).max())
    print("%s %s 80 classes: rows max|err| %.3g of max|ref| %.3g (%.2e rel), threshold %.4f"
          % (family, precision, err, scale, err / scale, thr))
    assert err <= row_tol * scale
    keep_all = net.tail.det_anchor.cpu().numpy()
    ncls = nc - 1 if family == "fcos" else nc
    mb, iou = m.config["nms_max_boxes"], m.config["nms_iou_threshold"]
    reps = [CR.compare_image(mkind, rows[b], ref[b], geom, res[b][2], keep_all[b, :len(res[b][2])], res[b][1], thr, mb,
                             iou, ncls, nc) for b in range(B)]
    tot = MG.summarize(reps)
    cc = net.tail.cand_count.cpu().numpy()
    print("%s %s: candidates/class mean %.0f max %d; classes clean %d ambiguous %d (reasons %s) identical %d of %d; "
          "keeps oracle %d gpu %d common %d; ds %.3g di %.3g; common-keep box err %.3g px"
          % (family, precision, cc.mean(), cc.max(), tot["clean"], tot["ambiguous"], tot["reasons"], tot["identical"],
             ncls * B, tot["kept_oracle"], tot["kept_gpu"], tot["same_keeps"], tot["ds"], tot["di"], tot["box_err"]))
    assert cc.mean() >= 10
    assert tot["ds"] <= ds_tol, tot
    assert tot["kept_gpu"] > 0 and tot["same_keeps"] >= 0.5 * tot["kept_oracle"], tot


# ------------------------------------------------------------------------------- losses --
def _loss_gt(rng, size, nc, B=2, G=10):
    gt = np.full((B, G, 5), -1.0, F32)
    for b in range(B):
        n = 3 + 3 * b
        gt[b, :n, 0:2] = rng.uniform(0.15 * size, 0.85 * size, (n, 2))
        gt[b, :n, 2:4] = rng.uniform(0.05 * size, 0.7 * size, (n, 2))
        gt[b, :n, 4] = rng.integers(0, nc, n)
    gt[0, 0, 4] = nc - 1
    return gt


@pytest.mark.parametrize("nc", [1, 80, 128])
@pytest.mark.parametrize("family", ["yolov3", "fcos"])
def test_loss_forward_vs_oracle(built, family, nc):
    from oracle import loss as OL
    from oracle import tails as OT
    from odt_b200.engine import RowsHarness
    size = 160 if family == "yolov3" else 256
    levels = ([(5, 5, 3), (10, 10, 3), (20, 20, 3)] if family == "yolov3"
              else [(32, 32, 1), (16, 16, 1), (8, 8, 1), (4, 4, 1), (2, 2, 1)])
    rng = np.random.default_rng(nc)
    rows = _rows(levels, nc, 2, seed=7 + nc)
    if family == "fcos":
        rows[..., nc + 1:] += F32(1.0)  # distances of a few stride units
    gt = _loss_gt(rng, size, nc)
    h = RowsHarness(_tail(family, nc, 0.5, 10, 0.5), levels, rows)
    kw = dict(coord_scale=2, noobj_scale=0.5, obj_scale=5, class_scale=1.5) if family == "yolov3" else {}
    got = h.loss("yolo" if family == "yolov3" else "fcos", gt, **kw)
    for b in range(2):
        if family == "yolov3":
            ref = OL.yolo_image_loss(CR.rows_to_levels(rows, levels, "yolo", nc), YOLO_PRIORS, gt[b], image=b,
                                     num_classes=nc, **kw)
        else:
            ref = OL.fcos_image_loss(CR.rows_to_levels(rows, levels, "fcos", nc), gt[b], image=b)
        print("%s nc=%d image %d: loss gpu %.6f oracle %.6f" % (family, nc, b, got[b], ref))
        assert abs(got[b] - ref) <= 2e-5 * max(abs(ref), 1.0)


@pytest.mark.parametrize("family,size", [("yolov3", 160), ("fcos", 256)])
def test_training_step_on_gpu_80_classes(built, family, size):
    """test_gpu_models.py::test_training_step_on_gpu at 80 classes: the autograd loss agrees with the CUDA loss
    forward on the same rows, the step moves the variables, the inference engine runs on the updated weights."""
    import torch
    from odt_b200.engine import RowsHarness
    nc = 80
    rng = np.random.default_rng(3)
    img = _img(2, size, size, seed=8)
    gt = _loss_gt(rng, size, nc)

    class It:
        def get_next(self):
            return img, gt
    provider = {"num_train": 2, "num_val": 0, "train_generator": ((lambda: None), It()), "val_generator": None}
    import FCOS
    import YOLOv3
    cls, ckind = (YOLOv3.YOLOv3, "yolov3") if family == "yolov3" else (FCOS.FCOS, "fcos")
    m = cls(model_cfg(ckind, num_classes=nc, mode="train", batch_size=2, bn_init="trained",
                      data_shape=[size, size, 3]), provider)
    tr = m.trainer()
    assert tr.device.type == "cuda" and tr.row == nc + 5
    rows = tr.forward_rows(img)
    per = [float(tr.image_loss(rows[b], gt[b])) for b in range(2)]
    hrn = RowsHarness(_tail(family, nc, 0.5, 10, 0.5), list(tr.net.levels), rows.detach().cpu().numpy())
    kw = {}
    if family == "yolov3":
        kw = dict(coord_scale=m.config["coord_scale"], noobj_scale=m.config["noobj_scale"],
                  obj_scale=m.config["obj_scale"], class_scale=m.config["class_scale"])
    got = hrn.loss("yolo" if family == "yolov3" else "fcos", gt, **kw)
    for b in range(2):
        print("%s 80 classes image %d: autograd %.6f, CUDA %.6f" % (family, b, per[b], got[b]))
        assert abs(per[b] - got[b]) <= 1e-4 * max(abs(per[b]), 1.0)
    w0 = {k: v.detach().clone() for k, v in tr.params.items()}
    loss = m.train_one_epoch(1e-3)
    assert np.isfinite(loss) and m.global_step == 1
    changed = sum(int(not torch.equal(w0[k], tr.params[k].detach())) for k in w0)
    assert changed >= 0.95 * len(w0)
    res = m.detect_batch(img[:1])
    assert len(res) == 1


# ---------------------------------------------------------------------------- pipelines --
@pytest.mark.parametrize("family,nc,hw,thr", [("yolov3", 80, 160, 0.05), ("fcos", 1, 256, 0.0),
                                              ("fcos", 128, 256, 5e-5)])
def test_pipelined_and_single_graph_streams_agree(built, monkeypatch, family, nc, hw, thr):
    """The two-stage pipeline against the one-graph-per-step stream and the synchronous call, for 80 and 128 classes and
    for FCOS's empty records (one class).  Random-init FCOS scores are about sigmoid(-4.6)^2 = 1e-4, hence its low
    thresholds."""
    import torch
    m = _model(family, nc, precision="fp16", data_shape=[hw, hw, 3], nms_score_threshold=thr)
    batches = [_img(2, hw, hw, seed=s) for s in range(51, 56)]
    ref = [m.detect_batch(b) for b in batches]
    if nc > 1:
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


# ------------------------------------------------------------------------- dispatch audit --
@pytest.mark.parametrize("family", ["yolov3", "fcos"])
def test_dispatch_audit_80_classes(built, family):
    """Every fp16 convolution of the 80-class networks runs a hand-written kernel: the image convolution on a stem
    kernel, every other one (the 255- and 80-channel heads included) on odt_conv2d_f16_tc -- none on conv_direct."""
    from odt_b200 import engine as E
    size = FULL[family][0]
    m = _model(family, 80, precision="fp16", bn_init="trained", data_shape=[size, size, 3])
    m.detect_batch(_img(1, size, size, seed=2))
    net = m.engine(1)
    convs = [op for op in net.ops if isinstance(op, E.ConvOp)]
    direct = [op.kernel for op in convs if not (op.is_image or op.use_tc)]
    assert not direct, direct
    heads = {op.p.Cout for op in convs if op.head is not None}
    assert (255 in heads) if family == "yolov3" else (80 in heads), heads
