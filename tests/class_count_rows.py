"""Test helpers for YOLOv3 / FCOS candidate rows of any class count: num_classes + 5 floats per row.

oracle/tails.py and tests/margins.py read the 25-float rows of 20 classes; the restatements here are the same
operations with the class count as a parameter, and `compare_image` runs the margin-aware checker of tests/margins.py
unchanged on them."""
from unittest import mock

import numpy as np

import margins as MG
from oracle import tails as OT


def rows_to_levels(rows, levels, kind, num_classes):
    """Inverse of oracle.tails.yolo_rows / fcos_rows: rows [B, N, num_classes + 5] -> the per-level tensors the oracle's
    *_scores_boxes / *_detect and loss functions take (`levels`: [(H, W, A)] in candidate order).
    kind 'yolo' -> preds [B, H, W, A * row]; 'fcos' -> (cls [B, H, W, nc], ctr [B, H, W, 1], reg [B, H, W, 4])."""
    nc, row = num_classes, num_classes + 5
    b, off, out = rows.shape[0], 0, []
    for h, w, a in levels:
        r = rows[:, off:off + h * w * a]
        if kind == "yolo":
            out.append(r.reshape(b, h, w, a * row))
        else:
            r = r.reshape(b, h, w, row)
            out.append((r[..., :nc], r[..., nc:nc + 1], r[..., nc + 1:nc + 5]))
        off += h * w * a
    assert off == rows.shape[1]
    return out


def per_row(kind, rows, geom, num_classes):
    """rows [N, num_classes + 5] of ONE image -> (scores [N, nc], boxes [N, 4], valid [N], None): tests/margins.py's
    per_row for the sigmoid families (kind 'yolo': geom levels, priors; 'fcos': levels)."""
    rows = np.asarray(rows, np.float32)
    if kind == "yolo":
        preds = rows_to_levels(rows[None], geom["levels"], "yolo", num_classes)
        conf, boxes = OT.yolo_scores_boxes(preds, geom["priors"], num_classes=num_classes)
    elif kind == "fcos":
        heads = rows_to_levels(rows[None], geom["levels"], "fcos", num_classes)
        conf, boxes = OT.fcos_scores_boxes(heads, num_classes=num_classes)
    else:
        raise ValueError("%s: only the sigmoid families take other class counts" % kind)
    return conf, boxes, np.ones(conf.shape[0], bool), None


def compare_image(kind, rows_gpu, rows_ref, geom, gpu_ids, gpu_keep, gpu_boxes, thr, max_boxes, iou_thr, n_classes,
                  num_classes):
    """margins.compare_image on rows of `num_classes` classes (n_classes: the classes NMS visits): the checker's own
    decision logic, with its row -> (scores, boxes) restatement taken from per_row above."""
    with mock.patch.object(MG, "per_row", lambda k, r, g: per_row(k, r, g, num_classes)):
        return MG.compare_image(kind, rows_gpu, rows_ref, geom, gpu_ids, gpu_keep, gpu_boxes, thr, max_boxes, iou_thr,
                                n_classes)
