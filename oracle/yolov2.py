"""YOLOv2 restated on the CPU in numpy fp32 (test oracle): the Darknet-19 graph with its passthrough concat
(YOLOv2.py:75-100,255-303), the decode / per-class NMS tail (:183-210,230-244) and the per-image training loss
(:105-173), built from the oracle's existing pieces.  Not product code -- see oracle/__init__.py."""
import numpy as np

from . import tfops as T
from .loss import _sig_xent
from .nets import Ctx
from .tails import _per_class_nms

F32 = np.float32

# (name, filters, kernel) of conv1 .. conv18, "pool" for a 2x2/2 SAME max-pool (:255-303)
DARKNET19 = [("conv1", 32, 3), "pool", ("conv2", 64, 3), "pool",
             ("conv3", 128, 3), ("conv4", 64, 1), ("conv5", 128, 3), "pool",
             ("conv6", 256, 3), ("conv7", 128, 1), ("conv8", 256, 3), "pool",
             ("conv9", 512, 3), ("conv10", 256, 1), ("conv11", 512, 3), ("conv12", 256, 1), ("conv13", 512, 3),
             "pool",
             ("conv14", 1024, 3), ("conv15", 512, 1), ("conv16", 1024, 3), ("conv17", 512, 1), ("conv18", 1024, 3)]
HEAD = ["conv1", "conv2", "conv3", "conv4", "conv5"]


def yolov2_heads(weights, images):
    """images [B,H,W,3] RGB 0..255 -> the `predictions` tensor [B,H/32,W/32,A*(num_classes+5)] (inference BN)."""
    c = Ctx(weights)
    x = (np.asarray(images, F32) - np.array([123.68, 116.779, 103.979], F32)).astype(F32)

    def cl(x, name, act=True):  # _conv_layer: conv + bias -> BN, then the caller's leaky_relu(0.1)
        y = c.bn(c.conv(x, 1, 1, name=name))
        return T.leaky_relu(y) if act else y

    with c.n.scope("backone"):
        for item in DARKNET19:
            if item == "pool":
                x = T.max_pool_same(x, 2, 2)
                continue
            x = cl(x, item[0])
            if item[0] == "conv17":
                passthrough = x
    with c.n.scope("head"):
        for name in HEAD:
            x = cl(x, name)
        x = np.concatenate([passthrough, x], axis=-1)      # same grid, no reorg (:90)
        return cl(x, "predictions", act=False)


def yolo2_rows(pred, num_classes):
    """[B,H,W,A*(nc+5)] -> candidate rows [B, H*W*A, nc+5] (cell after cell, the A priors of a cell consecutive)."""
    return pred.reshape(pred.shape[0], -1, num_classes + 5).astype(F32)


def yolo2_scores_boxes(pred, priors, image=0, num_classes=20):
    """Per-row confidences [N,nc] and boxes [N,4] of one image (:183-192): sigmoid(class) * sigmoid(obj), centre =
    cell + 0.5 + sigmoid, size = prior + exp (additive), corners x 32; priors in grid cells as given."""
    _, h, w, _ = pred.shape
    pri = np.asarray(priors, F32)
    A = len(pri)
    r = pred[image].reshape(h, w, A, num_classes + 5).astype(F32)
    ayx = np.zeros((h, w, A, 2), F32)
    ayx[..., 0] = (np.arange(h, dtype=F32) + F32(0.5)).reshape(h, 1, 1)
    ayx[..., 1] = (np.arange(w, dtype=F32) + F32(0.5)).reshape(1, w, 1)
    conf = (T.sigmoid(r[..., :num_classes]) * T.sigmoid(r[..., num_classes + 4:])).astype(F32)
    byx = (ayx + T.sigmoid(r[..., num_classes:num_classes + 2])).astype(F32)
    bhw = (pri.reshape(1, 1, A, 2) + np.exp(r[..., num_classes + 2:num_classes + 4]).astype(F32)).astype(F32)
    box = (np.concatenate([byx - bhw / F32(2.0), byx + bhw / F32(2.0)], axis=-1) * F32(32.0)).astype(F32)
    return conf.reshape(-1, num_classes), box.reshape(-1, 4)


def yolo2_detect(pred, priors, score_thr, max_boxes, iou_thr, image=0, num_classes=20):
    """:193-210 for one image: per-class NMS over every class.  Returns scores, boxes, class ids, keep indices."""
    conf, box = yolo2_scores_boxes(pred, priors, image, num_classes)
    idx = np.arange(conf.shape[0], dtype=np.int32)
    return _per_class_nms(conf, box, idx, num_classes, score_thr, max_boxes, iou_thr)


def yolo2_image_loss(pred, priors, gt, coord_scale=1.0, noobj_scale=1.0, obj_scale=5.0, class_scale=1.0, image=0,
                     num_classes=20, noobj_iou=0.6):
    """The per-image loss of :105-173, forward only.  The GT (y, x, h, w, id, padded with -1) is divided by 32; its cell
    is clamped to the grid; the best prior at that cell by UNCLAMPED IoU, first maximum; sigmoid-CE centre, squared
    log-size (x 0.5), sigmoid-CE class and objectness; the no-object term on every (cell, prior) of a cell without GT
    whose best IoU with the GTs is <= 0.6, the prior box re-used in corner form (:148-151).  Not divided by the GT
    count: an image without boxes is the no-object term of every row."""
    nc = num_classes
    gt = np.asarray(gt, F32)
    cnt = int(np.argmin(gt, axis=0)[0])
    g = gt[:cnt]
    _, h, w, _ = pred.shape
    pri = np.asarray(priors, F32)
    A = len(pri)
    r = pred[image].reshape(h, w, A, nc + 5).astype(F32)
    gn = (g / np.array([32.0] * 4 + [1.0], F32).reshape(1, 5)).astype(F32)
    gyx, ghw, lab = gn[:, :2], gn[:, 2:4], gn[:, 4].astype(np.int32)
    fl = np.floor(gyx).astype(np.int64)
    fl[:, 0] = np.clip(fl[:, 0], 0, h - 1)
    fl[:, 1] = np.clip(fl[:, 1], 0, w - 1)
    g1 = (gyx - ghw / F32(2.0)).astype(F32)
    g2 = (gyx + ghw / F32(2.0)).astype(F32)
    coord = cls_l = obj_l = 0.0
    for gi in range(cnt):
        y, x = fl[gi]
        ayx = np.array([y, x], F32) + F32(0.5)
        a1, a2 = (ayx - pri / F32(2)).astype(F32), (ayx + pri / F32(2)).astype(F32)
        inter = np.prod(np.minimum(g2[gi], a2) - np.maximum(g1[gi], a1), axis=-1).astype(F32)
        iou = (inter / (np.prod(pri, axis=-1) + np.prod(g2[gi] - g1[gi]) - inter)).astype(F32)
        a = int(np.argmax(iou))
        row = r[y, x, a]
        tyx = (gyx[gi] - np.floor(gyx[gi])).astype(F32)
        thw = np.log((ghw[gi] / pri[a]).astype(F32)).astype(F32)
        coord += float(_sig_xent(tyx, row[nc:nc + 2]).sum(dtype=np.float64))
        coord += 0.5 * float(np.square(row[nc + 2:nc + 4] - thw).astype(F32).sum(dtype=np.float64))
        onehot = np.zeros(nc, F32)
        onehot[lab[gi]] = 1.0
        cls_l += float(_sig_xent(onehot, row[:nc]).sum(dtype=np.float64))
        obj_l += float(_sig_xent(np.ones(1, F32), row[nc + 4:nc + 5]).sum(dtype=np.float64))
    occ = np.zeros((h, w), bool)
    occ[fl[:, 0], fl[:, 1]] = True
    ayx = np.zeros((h, w, A, 2), F32)
    ayx[..., 0] = (np.arange(h, dtype=F32) + F32(0.5)).reshape(h, 1, 1)
    ayx[..., 1] = (np.arange(w, dtype=F32) + F32(0.5)).reshape(1, w, 1)
    c_nb = (ayx - pri.reshape(1, 1, A, 2) / F32(2.0)).astype(F32)       # y1x1 re-used as a centre
    s_nb = (ayx + pri.reshape(1, 1, A, 2) / F32(2.0)).astype(F32)       # y2x2 re-used as a size
    b1 = (c_nb - s_nb / F32(2.0)).astype(F32)[..., None, :]
    b2 = (c_nb + s_nb / F32(2.0)).astype(F32)[..., None, :]
    if cnt:
        inter = np.prod(np.minimum(g2, b2) - np.maximum(g1, b1), axis=-1).astype(F32)
        union = np.prod(b2 - b1, axis=-1) + np.prod(g2 - g1, axis=-1) - inter
        best = (inter / union).astype(F32).max(axis=-1)
    else:
        best = np.full((h, w, A), -np.inf, F32)
    mask = (best <= F32(noobj_iou)) & (~occ)[..., None]
    noobj = float((_sig_xent(np.zeros_like(r[..., nc + 4]), r[..., nc + 4]) * mask).sum(dtype=np.float64))
    return coord_scale * coord + class_scale * cls_l + obj_scale * obj_l + noobj_scale * noobj
