"""The loss-gradient kernels (csrc/loss.cu, odt_<family>_loss_grad) on the GPU against the gradient of the training
step's loss restatement (odt_b200/train.py image_loss, run in float64 with autograd on the same rows): small geometries
with their matching edges, G = 128, class and prior counts, full-size rows of the networks, determinism, and the
training step on the kernel path against the same step with the data term built from image_loss.

Bar: every element within 1e-5 of the image's max |gradient|, exact zeros where the reference is exactly zero, and
loss_out equal bit for bit to the loss forward (RowsHarness.loss).

The reference is the restatement in float64 wherever float64 makes the matching decisions the float32 kernels make,
i.e. where its loss equals the float32 restatement's to 1e-6.  Where it does not -- a best IoU within float32 rounding
of 0.4 / 0.5, the float32 ties of the YOLO edge cases, SSD's mining, which orders near-equal negative losses
differently in float64 and selects another set -- the reference is the float32 restatement, whose decisions are the
kernels' (and the oracle's)."""
import numpy as np
import pytest
import torch

import loss_grad_ref as LR
import test_gpu_loss as GL
from helpers import YOLO_PRIORS, model_cfg

pytestmark = pytest.mark.gpu
F32 = np.float32
YOLO_SCALES = dict(coord_scale=2.0, noobj_scale=0.5, obj_scale=5.0, class_scale=1.5)


def _kw(kind, cfg):
    from odt_b200.engine import Tail
    return {k: float(cfg[k]) for k, _ in Tail.LOSS_SCALARS[kind]}


def reference(kind, levels, cfg, size, nc, row, gt):
    """(loss, gradient, dtype) of the restatement: float64 where its decisions are float32's (see above)."""
    with np.errstate(all="ignore"):
        l32, g32 = LR.grad(LR.restatement(kind, levels, cfg, size, nc, dtype=torch.float32), row, gt)
        l64, g64 = LR.grad(LR.restatement(kind, levels, cfg, size, nc), row, gt)
    if abs(l64 - l32) <= 1e-6 * max(abs(l32), 1.0):
        return l64, g64, "float64"
    return l32, g32, "float32"


def check(kind, levels, size, cfg, rows, gt, nc=20, images=None):
    """Kernel loss and gradient of every image against the restatement; returns (loss, grad)."""
    from odt_b200.engine import RowsHarness
    h = RowsHarness(LR.tail(kind, size, cfg), levels, rows)
    kw = _kw(kind, cfg)
    loss, grad = h.loss_grad(kind, gt, **kw)
    fwd = h.loss(kind, gt, **kw)
    assert np.array_equal(loss.view(np.uint32), fwd.view(np.uint32)), (loss, fwd)
    assert grad.shape == rows.shape and grad.dtype == np.float32
    for b in (range(rows.shape[0]) if images is None else images):
        ref_loss, ref, dt = reference(kind, levels, cfg, size, nc, rows[b], gt[b])
        scale = float(np.abs(ref).max())
        err = float(np.abs(grad[b] - ref).max())
        print("%s image %d: loss %.6f (%s restatement %.6f), grad max|err| %.3g of max|ref| %.3g, %d zero rows"
              % (kind, b, loss[b], dt, ref_loss, err, scale, int((np.abs(ref).max(-1) == 0).sum())))
        assert abs(loss[b] - ref_loss) <= 2e-5 * max(abs(ref_loss), 1.0)
        assert np.isfinite(grad[b]).all() and err <= 1e-5 * scale
        assert np.all(grad[b][ref == 0] == 0), "exact zeros where the restatement has no gradient"
    return loss, grad


# ------------------------------------------------------------------------------ small geometries --
def _dup(g, i, j, cls):
    """GT row j := GT row i with another class: both choose the same best anchor / YOLO cell and prior."""
    g[j] = g[i]
    g[j, 4] = cls


def test_retina_small(built):
    geo, size = GL.RET_SMALL, 64
    rng = np.random.default_rng(1)
    gt = np.stack([LR.gt(rng, 3, size, 8, lo=0.3, hi=0.7), LR.gt(rng, 5, size, 8, lo=0.2, hi=0.6)])
    _dup(gt[0], 0, 3, 11)
    rows = LR.rows("retina", geo.N, B=2, seed=2)
    # negatives whose background probability is far under 1e-8: the clamp stops their gradient
    iou = GL.match_iou(geo, gt[0]).max(0)
    low = np.flatnonzero(iou < 0.2)[:40]
    rows[0, low, 20] = -40.0
    loss, grad = check("retina", geo.levels, size, LR.config("retina", size), rows, gt)
    assert np.all(grad[0, low] == 0)
    best = set(np.argmax(GL.match_iou(geo, gt[0]), axis=1).tolist())
    ignored = [n for n in np.flatnonzero((iou >= 0.4) & (iou <= 0.5)) if n not in best]
    assert len(ignored) and np.all(grad[0, ignored] == 0)


def test_ssd_small_both_sides_of_three_negatives_per_positive(built):
    from odt_b200.engine import RowsHarness
    rng = np.random.default_rng(3)
    for geo, n in ((GL.SSD_FINE, 4), (GL.SSD_TINY, 12)):
        size = 300
        gt = np.stack([LR.gt(rng, n, size, 14, lo=0.15, hi=0.5), LR.gt(rng, n, size, 14, lo=0.15, hi=0.5)])
        _dup(gt[1], 0, n - 1, 7)
        rows = LR.rows("ssd", geo.N, B=2, seed=n)
        cfg = LR.config("ssd", size)
        check("ssd", geo.levels, size, cfg, rows, gt)
        _, info = RowsHarness(LR.tail("ssd", size, cfg), geo.levels, rows).loss("ssd", gt, return_info=True)
        npos, nneg = info[:, 0], info[:, 1]
        print("SSD N=%d: #pos %s #neg %s #mined %s" % (geo.N, npos, nneg, info[:, 2]))
        assert np.all(nneg > 3 * npos) if geo is GL.SSD_FINE else np.all(nneg <= 3 * npos)


@pytest.mark.parametrize("nc", [1, 20, 80, 128])
def test_fcos_small(built, nc):
    levels, size = GL.FCOS_SMALL.levels, 128
    gt = np.full((2, 8, 5), -1.0, F32)
    # sizes exactly 64 / 128 (two levels each), one level without GT in image 1, two GTs on the same cells
    gt[0, :4] = [[40, 50, 30, 40, 0], [60, 60, 64, 64, nc - 1], [64, 64, 128, 128, nc // 2], [64, 64, 128, 128, 0]]
    gt[1, :2] = [[50, 70, 90, 70, nc - 1], [70, 60, 256, 256, nc // 3]]
    rows = LR.rows("fcos", GL.FCOS_SMALL.N, nc=nc, B=2, seed=nc)
    check("fcos", levels, size, LR.config("fcos", size, nc=nc), rows, gt, nc=nc)


@pytest.mark.parametrize("A", [1, 3, 9])
@pytest.mark.parametrize("nc", [1, 20, 80, 128])
def test_yolo_small(built, A, nc):
    levels, size = [(5, 5, A), (10, 10, A), (20, 20, A)], 160
    rng = np.random.default_rng(10 * A + nc)
    gt = np.stack([LR.gt(rng, 6, size, 10, nc=nc), LR.gt(rng, 9, size, 10, nc=nc, lo=0.03, hi=0.9)])
    _dup(gt[0], 1, 6, nc - 1)  # same cell and prior on every level: the contributions add up
    cfg = LR.config("yolo", size, nc=nc, A=A, **YOLO_SCALES)
    rows = LR.rows("yolo", sum(h * w * a for h, w, a in levels), nc=nc, B=2, seed=A + nc)
    check("yolo", levels, size, cfg, rows, gt, nc=nc)


@pytest.mark.parametrize("name", sorted(GL.EDGE_CASES))
def test_matching_edges(built, name):
    """The forward kernels' edge cases (tests/test_gpu_loss.py): IoU exactly 0.5 / 0.4, tied best anchors, mining
    ties and mining that runs dry, FCOS boxes on grid lines and sizes exactly 64 / 128 / 256 / 512, tied areas, YOLO
    no-object IoU 0.5, centres on cell boundaries, level and prior ties."""
    c = GL.EDGE_CASES[name]()
    geo = c["geo"]
    cfg = LR.config(geo.kind, geo.size, priors=YOLO_PRIORS) if geo.kind == "yolo" else LR.config(geo.kind, geo.size)
    check(geo.kind, geo.levels, geo.size, cfg, c["rows"][None], c["gt"][None])


@pytest.mark.parametrize("kind", ["retina", "ssd", "fcos", "yolo"])
def test_full_gt_capacity(built, kind):
    """G = 128: padded in the last row only, unpadded, and with tied minima of column 0."""
    geo = GL.TAIL_GEOS[kind]
    gt = GL.capacity_gt(kind, seed=40)
    rows = LR.rows(kind, geo.N, B=3, seed=41)
    cfg = LR.config(kind, geo.size, priors=YOLO_PRIORS) if kind == "yolo" else LR.config(kind, geo.size)
    check(kind, geo.levels, geo.size, cfg, rows, gt)


@pytest.mark.parametrize("kind", ["retina", "ssd", "fcos", "yolo"])
def test_image_without_boxes(built, kind):
    """No GT: the kernels compute what the loss's formulas give.  FCOS has no level with GT: loss 0, zero gradient,
    as the restatement.  The other three divide by zero positives / GTs: the loss is not finite.  RetinaNet's and
    YOLOv3's gradients divide by it too; SSD selects nothing, so its gradient is zero.  The restatement itself raises
    on such an image (a maximum over zero GTs), so there is no gradient to compare."""
    from odt_b200.engine import RowsHarness
    geo = {"retina": GL.RET_SMALL, "ssd": GL.SSD_TINY, "fcos": GL.FCOS_SMALL, "yolo": GL.YOLO_SMALL}[kind]
    cfg = LR.config(kind, geo.size, priors=YOLO_PRIORS) if kind == "yolo" else LR.config(kind, geo.size)
    rng = np.random.default_rng(5)
    gt = np.stack([np.full((4, 5), -1.0, F32), LR.gt(rng, 3, geo.size, 4, lo=0.2)])
    rows = LR.rows(kind, geo.N, B=2, seed=6)
    h = RowsHarness(LR.tail(kind, geo.size, cfg), geo.levels, rows)
    loss, grad = h.loss_grad(kind, gt, **_kw(kind, cfg))
    tr = LR.restatement(kind, geo.levels, cfg, geo.size)
    if kind == "fcos":
        assert loss[0] == 0 and np.all(grad[0] == 0)
        assert LR.grad(tr, rows[0], gt[0])[0] == 0
    else:
        assert not np.isfinite(loss[0])
        assert np.all(grad[0] == 0) if kind == "ssd" else not np.isfinite(grad[0]).all()
        with pytest.raises(IndexError):
            LR.grad(tr, rows[0], gt[0])
    # the other image of the batch is unaffected
    check(kind, geo.levels, geo.size, cfg, rows, gt, images=[1])


# ------------------------------------------------------------------------------------ full size --
FULL = {"ssd300": ("SSD300", "ssd", "ssd", 300, {}), "ssd512": ("SSD512", "ssd", "ssd", 512, {}),
        "retinanet800": ("RetinaNet", "retinanet", "retina", 800, {}),
        "retinanet800_basic": ("RetinaNet", "retinanet", "retina", 800,
                               dict(is_bottleneck=False, init_conv_filters=7, residual_block_list=[2, 2, 2, 2])),
        "yolov3_416": ("YOLOv3", "yolov3", "yolo", 416, YOLO_SCALES), "fcos1024": ("FCOS", "fcos", "fcos", 1024, {})}


@pytest.mark.parametrize("name", sorted(FULL))
def test_full_size_network_rows(built, name):
    """B = 2 rows of the trained-BN network (fp32 engine), realistic GT padded to 60 rows."""
    import importlib
    mod, cfg_kind, kind, size, over = FULL[name]
    cfg = model_cfg(cfg_kind, data_shape=[size, size, 3], bn_init="trained", precision="fp32", **over)
    m = getattr(importlib.import_module(mod), mod)(cfg, None)
    img = np.random.default_rng(7).integers(0, 256, (2, size, size, 3)).astype(F32)
    m.detect_batch(img)
    net = m.engine(2)
    rows = net.head_buf.cpu().numpy()
    rng = np.random.default_rng(8)
    gt = np.stack([LR.gt(rng, n, size, 60, lo=0.05 if kind != "fcos" else 0.06, hi=0.6) for n in (12, 40)])
    check(kind, list(net.levels), size, m.config, rows, gt)


# ---------------------------------------------------------------------------------- determinism --
@pytest.mark.parametrize("kind", ["retina", "ssd", "fcos", "yolo"])
def test_deterministic_and_batch_independent(built, kind):
    from odt_b200.engine import RowsHarness
    geo = GL.TAIL_GEOS[kind]
    cfg = LR.config(kind, geo.size, priors=YOLO_PRIORS) if kind == "yolo" else LR.config(kind, geo.size)
    rng = np.random.default_rng(9)
    gt = np.stack([LR.gt(rng, n, geo.size, 20, lo=0.1) for n in (3, 19, 8, 1)])
    _dup(gt[2], 0, 7, 5)
    rows = LR.rows(kind, geo.N, B=4, seed=10)
    h = RowsHarness(LR.tail(kind, geo.size, cfg), geo.levels, rows)
    kw = _kw(kind, cfg)
    l1, g1 = h.loss_grad(kind, gt, **kw)
    l2, g2 = h.loss_grad(kind, gt, **kw)
    assert np.array_equal(l1, l2) and np.array_equal(g1.view(np.uint32), g2.view(np.uint32))
    for b in range(4):
        hb = RowsHarness(LR.tail(kind, geo.size, cfg), geo.levels, rows[b:b + 1])
        lb, gb = hb.loss_grad(kind, gt[b:b + 1], **kw)
        assert lb[0] == l1[b] and np.array_equal(gb[0].view(np.uint32), g1[b].view(np.uint32)), b


# -------------------------------------------------------------------------------- training step --
STEP = {"ssd300": ("SSD300", "ssd", 300, {}), "retinanet": ("RetinaNet", "retinanet", 128, {}),
        "yolov3": ("YOLOv3", "yolov3", 160, YOLO_SCALES), "fcos": ("FCOS", "fcos", 256, {})}
# max |p_kernel - p_restatement| over the largest update max |p_restatement - p_0| of any variable.  Measured on an
# H100 at 1.1e-3 to 1.9e-3 for the four families (the backward of the training-mode BN network amplifies the float32
# differences of the row gradient); per variable the ratio means little: a convolution bias in front of BN has no data
# gradient, its update is weight decay alone.
STEP_PARAM_BOUND = 5e-3


@pytest.mark.parametrize("name", sorted(STEP))
def test_training_step_kernel_path_against_restatement(built, name):
    """One tr.step on the kernel path and one with the data term built from image_loss, same GPU, same weights and
    images: identical BN moving statistics, parameters within STEP_PARAM_BOUND of the update; then train_one_epoch
    on the kernel path returns a finite loss and moves >= 95 % of the variables."""
    import importlib
    from odt_b200.train import GraphTrainer
    mod, cfg_kind, size, over = STEP[name]
    rng = np.random.default_rng(11)
    img = rng.integers(0, 256, (2, size, size, 3)).astype(F32)
    gt = np.stack([LR.gt(rng, n, size, 60, lo=0.1, hi=0.6) for n in (3, 6)])

    class It:
        def get_next(self):
            return img, gt
    provider = {"num_train": 2, "num_val": 0, "train_generator": ((lambda: None), It()), "val_generator": None}
    cfg = model_cfg(cfg_kind, data_shape=[size, size, 3], bn_init="trained", mode="train", batch_size=2, **over)
    m = getattr(importlib.import_module(mod), mod)(cfg, provider)
    ker, ref, ref2 = GraphTrainer(m, "cuda"), GraphTrainer(m, "cuda"), GraphTrainer(m, "cuda")
    assert ker._loss_kernels is not None
    ref._loss_kernels = ref2._loss_kernels = None  # the data term from image_loss
    p0 = {k: v.detach().clone() for k, v in ker.params.items()}
    lk = ker.step(img, gt, 1e-3)
    lr_ = ref.step(img, gt, 1e-3)
    ref2.step(img, gt, 1e-3)
    noise = max(float((ref2.params[k] - ref.params[k]).abs().max()) for k in p0)  # restatement path against itself
    assert np.isfinite(lk) and abs(lk - lr_) <= 1e-4 * max(abs(lr_), 1.0), (lk, lr_)
    for k in ker.buffers:
        assert torch.equal(ker.buffers[k], ref.buffers[k]), k
    upd = max(float((ref.params[k] - p0[k]).abs().max()) for k in p0)
    diff = max(float((ker.params[k] - ref.params[k]).abs().max()) for k in p0)
    rel = max(float((ker.params[k] - ref.params[k]).abs().max()) / max(float(ref.params[k].abs().max()), 1e-30)
              for k in p0)
    print("%s: loss kernel %.6f restatement %.6f; max param difference %.3g = %.3g of the largest update "
          "(restatement run twice: %.3g); max relative param difference %.3g" % (name, lk, lr_, diff, diff / upd,
                                                                               noise / upd, rel))
    assert diff <= STEP_PARAM_BOUND * upd
    tr = m.trainer()
    assert tr._loss_kernels is not None
    w0 = {k: v.detach().clone() for k, v in tr.params.items()}
    loss = m.train_one_epoch(1e-3)
    assert np.isfinite(loss) and m.global_step == 1
    changed = sum(int(not torch.equal(w0[k], tr.params[k].detach())) for k in w0)
    assert changed >= 0.95 * len(w0)
