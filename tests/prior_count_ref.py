"""Test restatement of the YOLOv3 tail and loss at any number of priors per level (num_priors = A, 1 to 9).

oracle/tails.py::yolo_scores_boxes and oracle/loss.py::yolo_image_loss reshape every level to 3 priors.  The functions
here are the same operations, in the same order and on the oracle's own pieces (tfops.sigmoid, loss._sig_xent, the
per-class NMS loop), with A read from the priors; at A = 3 they equal the oracle bit for bit
(tests/test_prior_count.py).  Rows go to levels with class_count_rows.rows_to_levels, which already takes (H, W, A)."""
from unittest import mock

import numpy as np

import class_count_rows as CR
import margins as MG
from oracle import loss as OL
from oracle import tails as OT
from oracle import tfops as T

F32 = np.float32


def priors_for(A):
    """A config's `priors` with A (h, w) pairs per level: sizes growing 1.3x from prior to prior, aspect ratios
    cycling through tall / square / wide, levels around 12, 40 and 120 pixels like the COCO anchors."""
    aspect = [(1.0, 1.4), (1.2, 1.2), (1.4, 1.0)]
    return [[[round(b * 1.3 ** i * aspect[i % 3][0], 2), round(b * 1.3 ** i * aspect[i % 3][1], 2)] for i in range(A)]
            for b in (12.0, 40.0, 120.0)]


def yolo_scores_boxes(preds, priors, image=0, num_classes=20):
    """Per-row confidences [N, nc] and boxes [N, 4] of YOLOv3.py:320-351 for one image; level k holds
    len(priors[k]) priors per cell."""
    stride = [8.0, 16.0, 32.0]
    mult = [stride[-1], stride[-1], stride[-2]]
    confs, boxes = [], []
    for k, p in enumerate(preds):
        _, h, w, _ = p.shape
        a = len(priors[k])
        r = p[image].reshape(h, w, a, num_classes + 5).astype(F32)
        pri = (np.array(priors[k], dtype=F32) / F32(stride[k])).astype(F32).reshape(1, 1, a, 2)
        cy = (np.arange(h, dtype=F32) + F32(0.5)).reshape(h, 1, 1)
        cx = (np.arange(w, dtype=F32) + F32(0.5)).reshape(1, w, 1)
        ayx = np.zeros((h, w, a, 2), dtype=F32)
        ayx[..., 0] = cy
        ayx[..., 1] = cx
        cls = T.sigmoid(r[..., :num_classes])
        obj = T.sigmoid(r[..., num_classes + 4:])
        byx = (ayx + T.sigmoid(r[..., num_classes:num_classes + 2])).astype(F32)
        bhw = (pri + np.exp(r[..., num_classes + 2:num_classes + 4]).astype(F32)).astype(F32)
        box = np.concatenate([byx - bhw / F32(2.0), byx + bhw / F32(2.0)], axis=-1).astype(F32)
        boxes.append((box * F32(mult[k])).astype(F32).reshape(-1, 4))
        confs.append((cls * obj).astype(F32).reshape(-1, num_classes))
    return np.concatenate(confs, axis=0), np.concatenate(boxes, axis=0)


def yolo_detect(preds, priors, score_thr, max_boxes, iou_thr, image=0, num_classes=20):
    """YOLOv3.py:320-368 for one image: (scores, boxes, class ids, keep indices)."""
    conf, box = yolo_scores_boxes(preds, priors, image, num_classes)
    idx = np.arange(conf.shape[0], dtype=np.int32)
    return OT._per_class_nms(conf, box, idx, num_classes, score_thr, max_boxes, iou_thr)


def _level_ious(priors, g, k):
    """GT rows g against the priors of level k at each GT's own cell (YOLOv3.py:161-194): the level's normalised GT
    and the unclamped IoU [G, A]."""
    norm = [32.0, 16.0, 8.0]
    pstride = [8.0, 16.0, 32.0]
    pri = (np.array(priors[k], dtype=F32) / F32(pstride[k])).astype(F32)      # [A,2] (h,w)
    gn = (g / np.array([norm[k]] * 4 + [1.0], F32).reshape(1, 5)).astype(F32)
    gyx, ghw, lab = gn[:, :2], gn[:, 2:4], gn[:, 4].astype(np.int32)
    fl = np.floor(gyx).astype(np.int64)
    ayx = (fl.astype(F32) + F32(0.5))[:, None, :]
    a1 = (ayx - pri[None] / F32(2)).astype(F32)                                    # [G,A,2]
    a2 = (ayx + pri[None] / F32(2)).astype(F32)
    g1 = (gyx - ghw / F32(2.0)).astype(F32)[:, None, :]
    g2 = (gyx + ghw / F32(2.0)).astype(F32)[:, None, :]
    inter = np.prod(np.minimum(g2, a2) - np.maximum(g1, a1), axis=-1).astype(F32)  # no clamp (:171-173)
    garea = np.prod(g2 - g1, axis=-1).astype(F32)
    aarea = np.prod(pri, axis=-1).astype(F32)[None]
    iou = (inter / (aarea + garea - inter)).astype(F32)                            # [G,A]
    return dict(pri=pri, gyx=gyx, ghw=ghw, lab=lab, fl=fl, g1=g1[:, 0], g2=g2[:, 0], idx=np.argmax(iou, axis=-1),
                mx=iou.max(axis=-1))


def _level_masks(lv):
    m1 = (lv[0]["mx"] > lv[1]["mx"]) & (lv[0]["mx"] > lv[2]["mx"])
    m2 = (lv[1]["mx"] > lv[0]["mx"]) & (lv[1]["mx"] > lv[2]["mx"])
    return m1, m2, ~(m1 | m2)


def assignment(priors, gt):
    """(level, prior) of every valid GT row of one image: where its positive terms are read."""
    gt = np.asarray(gt, F32)
    g = gt[:int(np.argmin(gt, axis=0)[0])]
    lv = [_level_ious(priors, g, k) for k in range(3)]
    out = [None] * len(g)
    for k, m in enumerate(_level_masks(lv)):
        for gi in np.nonzero(m)[0]:
            out[gi] = (k, int(lv[k]["idx"][gi]))
    return out


def yolo_image_loss(preds, priors, gt, coord_scale=1.0, noobj_scale=1.0, obj_scale=5.0, class_scale=1.0,
                    image=0, num_classes=20):
    """oracle/loss.py::yolo_image_loss with len(priors[k]) priors on level k: the prior arg-max runs over all of them
    (first maximum wins), the no-object term over every (cell, prior)."""
    nc = num_classes
    gt = np.asarray(gt, F32)
    cnt = int(np.argmin(gt, axis=0)[0])
    g = gt[:cnt]
    lv = []
    for k, p in enumerate(preds):
        _, h, w, _ = p.shape
        a = len(priors[k])
        L_ = _level_ious(priors, g, k)
        L_.update(r=p[image].reshape(h, w, a, nc + 5).astype(F32), h=h, w=w, a=a)
        lv.append(L_)
    coord = cls_l = obj_l = noobj = 0.0
    for L_, m in zip(lv, _level_masks(lv)):
        r, pri, a = L_["r"], L_["pri"], L_["a"]
        for gi in np.nonzero(m)[0]:
            y, x = L_["fl"][gi]
            ai = L_["idx"][gi]
            row = r[y, x, ai]
            tyx = (L_["gyx"][gi] - np.floor(L_["gyx"][gi])).astype(F32)
            thw = np.log((L_["ghw"][gi] / pri[ai]).astype(F32)).astype(F32)
            coord += float(OL._sig_xent(tyx, row[nc:nc + 2]).sum(dtype=np.float64))
            coord += 0.5 * float(np.square(row[nc + 2:nc + 4] - thw).astype(F32).sum(dtype=np.float64))
            onehot = np.zeros(nc, F32)
            onehot[L_["lab"][gi]] = 1.0
            cls_l += float(OL._sig_xent(onehot, row[:nc]).sum(dtype=np.float64))
            obj_l += float(OL._sig_xent(np.ones(1, F32), row[nc + 4:nc + 5]).sum(dtype=np.float64))
        h, w = L_["h"], L_["w"]
        occ = np.zeros((h, w), bool)
        occ[L_["fl"][:, 0], L_["fl"][:, 1]] = True
        cy = (np.arange(h, dtype=F32) + F32(0.5)).reshape(h, 1, 1, 1)
        cx = (np.arange(w, dtype=F32) + F32(0.5)).reshape(1, w, 1, 1)
        ayx = np.concatenate([cy + np.zeros((1, w, a, 1), F32), cx + np.zeros((h, 1, a, 1), F32)], -1).astype(F32)
        yx_nb = (ayx - pri.reshape(1, 1, a, 2) / F32(2.0)).astype(F32)      # really y1x1
        hw_nb = (ayx + pri.reshape(1, 1, a, 2) / F32(2.0)).astype(F32)      # really y2x2
        b1 = (yx_nb - hw_nb / F32(2.0)).astype(F32)[..., None, :]             # [h,w,A,1,2]
        b2 = (yx_nb + hw_nb / F32(2.0)).astype(F32)[..., None, :]
        gg1, gg2 = L_["g1"].reshape(1, 1, 1, -1, 2), L_["g2"].reshape(1, 1, 1, -1, 2)
        inter = np.prod(np.minimum(gg2, b2) - np.maximum(gg1, b1), axis=-1).astype(F32)
        aarea = np.prod(b2 - b1, axis=-1).astype(F32)
        garea = np.prod(gg2 - gg1, axis=-1).astype(F32)
        iou = (inter / (aarea + garea - inter)).astype(F32).max(axis=-1)       # [h,w,A]
        mask = (iou <= F32(0.5)) & (~occ)[..., None]
        noobj += float((OL._sig_xent(np.zeros_like(r[..., nc + 4]), r[..., nc + 4]) * mask).sum(dtype=np.float64))
    ng = float(cnt)
    return (coord_scale * coord + class_scale * cls_l + obj_scale * obj_l) / ng + noobj_scale * noobj / ng


def per_row(rows, geom, num_classes):
    """rows [N, nc + 5] of ONE image -> (scores, boxes, valid, None), tests/margins.py's per_row for YOLOv3 rows of
    any prior count (geom: levels, priors)."""
    rows = np.asarray(rows, np.float32)
    preds = CR.rows_to_levels(rows[None], geom["levels"], "yolo", num_classes)
    conf, boxes = yolo_scores_boxes(preds, geom["priors"], num_classes=num_classes)
    return conf, boxes, np.ones(conf.shape[0], bool), None


def compare_image(rows_gpu, rows_ref, geom, gpu_ids, gpu_keep, gpu_boxes, thr, max_boxes, iou_thr, num_classes):
    """margins.compare_image on YOLOv3 rows of any prior count: the checker's own decision logic, with its
    row -> (scores, boxes) restatement taken from per_row above."""
    with mock.patch.object(MG, "per_row", lambda k, r, g: per_row(r, g, num_classes)):
        return MG.compare_image("yolo", rows_gpu, rows_ref, geom, gpu_ids, gpu_keep, gpu_boxes, thr, max_boxes,
                                iou_thr, num_classes)
