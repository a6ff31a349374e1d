"""References and bars of tests/test_gpu_workloads.py: the oracle tail (oracle/tails.py, oracle/yolov2.py) on the
candidate rows of any of the six families, the score thresholds of the three regimes the workloads run at, the oracle
forward, and the comparisons that hold the GPU's packed records, its pipelined records and its detection stream to
them.  Pure numpy: the bars themselves are checked on the CPU against planted faults."""
from unittest import mock

import numpy as np

import margins as MG
from helpers import assert_boxes_close

F32 = np.float32
SMEM_WINDOW = 1024  # entries of the NMS kernel's shared-memory list window; longer lists take the prefilter path
_MG_PER_ROW = MG.per_row

# model kind -> tail family (the `kind` of tests/margins.py, plus 'yolo2')
FAMILY = {"ssd300": "ssd", "ssd512": "ssd", "retinanet": "retina", "yolov3": "yolo", "fcos": "fcos",
          "yolov2": "yolo2"}


def geometry(kind, levels, cfg, in_h):
    """The geometry dict of tests/margins.py for a network: levels [(H, W, A)] in candidate order, its config and
    input height."""
    fam = FAMILY[kind]
    shapes = [(h, w) for h, w, _ in levels]
    if fam == "ssd":
        return {"size": int(in_h), "shapes": shapes}
    if fam == "retina":
        return {"data_shape": list(cfg["data_shape"]), "shapes": shapes}
    if fam in ("yolo", "yolo2"):
        return {"levels": [tuple(lv) for lv in levels], "priors": cfg["priors"]}
    return {"levels": [tuple(lv) for lv in levels]}


def nms_classes(fam, num_classes=20):
    """Classes the per-class NMS visits: FCOS skips its last one (FCOS.py:252)."""
    return num_classes - 1 if fam == "fcos" else num_classes


def per_row(fam, rows, geom):
    """margins.per_row for one image's rows, with YOLOv2's one-level decode (oracle/yolov2.py) added."""
    if fam != "yolo2":
        return _MG_PER_ROW(fam, rows, geom)
    from oracle import yolov2 as OY
    (h, w, _), = geom["levels"]
    rows = np.asarray(rows, F32)
    conf, boxes = OY.yolo2_scores_boxes(rows.reshape(1, h, w, -1), geom["priors"], num_classes=rows.shape[1] - 5)
    return conf, boxes, np.ones(conf.shape[0], bool), None


def oracle_tail(fam, rows, geom, thr, max_boxes, iou_thr):
    """The oracle tail on ONE image's candidate rows [N, row] -> (scores, boxes, class ids, keep indices)."""
    from oracle import tails as OT
    r = np.asarray(rows, F32)
    if fam in ("ssd", "retina"):
        if fam == "ssd":
            _, _, ayx, ahw = OT.ssd_anchors(geom["size"], geom["shapes"])
        else:
            _, _, ayx, ahw = OT.retina_anchors(geom["data_shape"], geom["shapes"])
        return OT.softmax_tail(r[:, :21], r[:, 21:23], r[:, 23:], ayx, ahw, 20, thr, max_boxes, iou_thr)
    if fam == "yolo":
        return OT.yolo_detect(OT.rows_to_levels(r[None], geom["levels"], "yolo"), geom["priors"], thr, max_boxes,
                              iou_thr)
    if fam == "fcos":
        return OT.fcos_detect(OT.rows_to_levels(r[None], geom["levels"], "fcos"), thr, max_boxes, iou_thr)
    from oracle import yolov2 as OY
    (h, w, _), = geom["levels"]
    return OY.yolo2_detect(r.reshape(1, h, w, -1), geom["priors"], thr, max_boxes, iou_thr,
                           num_classes=r.shape[1] - 5)


def candidate_scores(fam, rows, geom):
    """Per image, the scores [N, C] of the rows that reach NMS (softmax families: the rows whose arg-max is a
    foreground class), as margins.per_row computes them."""
    out = []
    for r in rows:
        S, _, V, _ = per_row(fam, r, geom)
        out.append(S[V])
    return out


def dense_threshold(scores, frac, N):
    """The score at which about `frac` * N candidates per class and image pass, over all images of the batch (the dense
    regime of bench.py, quantile as test_gpu_models._dense_threshold takes it); `scores` from candidate_scores, N the
    rows per image."""
    v = np.concatenate([s.reshape(-1) for s in scores])
    k = int(min(max(frac * N * scores[0].shape[1] * len(scores), 40), v.size - 1))
    return float(np.partition(v, v.size - k)[v.size - k])


def long_list_threshold(scores, n_classes, length=SMEM_WINDOW + 64):
    """A threshold at which at least one (image, class) list NMS visits holds `length` candidates or more: the largest
    `length`-th score over the lists."""
    best = -np.inf
    for s in scores:
        if s.shape[0] < length:
            continue
        part = np.partition(s[:, :n_classes], s.shape[0] - length, axis=0)[s.shape[0] - length]
        best = max(best, float(part.max()))
    assert np.isfinite(best), "no list can hold %d candidates" % length
    return best


def check_records(rec, anchors, counts, want):
    """The GPU's packed records [B, D*6+2] (per image D rows of (score, y1, x1, y2, x2, class), then the count and the
    overflow flag), keep indices [B, D] and counts [B] against the oracle tail's result for every image: the count and
    a clear flag as the oracle's keep list implies, class ids and keep indices identical and in order, scores within
    1e-6 relative, boxes within assert_boxes_close.  Returns (worst relative score error, worst box error)."""
    rec, anchors, counts = np.asarray(rec, F32), np.asarray(anchors), np.asarray(counts)
    B, D = rec.shape[0], (rec.shape[1] - 2) // 6
    assert rec.shape[1] == D * 6 + 2 and len(want) == B, (rec.shape, len(want))
    ws = wb = 0.0
    for b in range(B):
        s, bx, cid, kp = want[b]
        n = len(cid)
        assert n <= D
        assert rec[b, D * 6 + 1] == 0, "image %d: overflow flag set" % b
        assert rec[b, D * 6] == n, "image %d: the record counts %r detections, the oracle keeps %d" % (b, rec[b, D * 6], n)
        assert int(counts[b]) == n, "image %d: det_count %d, the oracle keeps %d" % (b, int(counts[b]), n)
        d = rec[b, :n * 6].reshape(n, 6)
        np.testing.assert_array_equal(d[:, 5], np.asarray(cid, F32), err_msg="image %d: class ids" % b)
        np.testing.assert_array_equal(anchors[b, :n], kp, err_msg="image %d: keep indices" % b)
        np.testing.assert_allclose(d[:, 0], s, rtol=1e-6, atol=0, err_msg="image %d: scores" % b)
        assert_boxes_close(d[:, 1:5], bx, what="image %d: boxes" % b)
        if n:
            ws = max(ws, float((np.abs(d[:, 0] - s) / np.abs(s)).max()))
            wb = max(wb, float(np.abs(d[:, 1:5] - bx).max()))
    return ws, wb


def pack_records(want, D):
    """What a correct NMS kernel writes for the oracle results `want`: (records [B, D*6+2], keep indices [B, D],
    counts [B]).  Rows past an image's count are left at zero."""
    B = len(want)
    rec = np.zeros((B, D * 6 + 2), F32)
    anchors = np.zeros((B, D), np.int32)
    counts = np.zeros(B, np.int32)
    for b, (s, bx, cid, kp) in enumerate(want):
        n = len(cid)
        d = rec[b, :D * 6].reshape(D, 6)
        d[:n, 0], d[:n, 1:5], d[:n, 5] = s, bx, cid
        anchors[b, :n], counts[b] = kp, n
        rec[b, D * 6] = n
    return rec, anchors, counts


def check_stream(got, want):
    """Every batch of a detection stream, every image and every array ([scores, boxes, class ids]) equal to the
    synchronous call's, dtype included.  Returns the number of detections compared."""
    got = list(got)
    assert len(got) == len(want), (len(got), len(want))
    n = 0
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w), "batch %d: %d images, expected %d" % (i, len(g), len(w))
        for b in range(len(w)):
            gi, wi = g[b], w[b]
            assert len(gi) == len(wi) == 3
            for a, c, what in zip(gi, wi, ("scores", "boxes", "class ids")):
                assert a.dtype == c.dtype, (i, b, what, a.dtype, c.dtype)
                np.testing.assert_array_equal(a, c, err_msg="batch %d image %d: %s" % (i, b, what))
            n += len(wi[2])
    return n


def check_pipelined_records(got, want):
    """A pipelined step's records against run()'s on the same images: counts and overflow flags exact, each image's
    rows up to its count bit-identical (the rows past the count hold whatever an earlier batch left: not compared).
    Returns the number of detections compared."""
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (got.shape, want.shape)
    np.testing.assert_array_equal(got[:, -2:], want[:, -2:], err_msg="counts and overflow flags")
    n = 0
    for b in range(want.shape[0]):
        k = int(want[b, -2]) * 6
        np.testing.assert_array_equal(got[b, :k].view(np.uint32), want[b, :k].view(np.uint32),
                                      err_msg="image %d: detections" % b)
        n += k // 6
    return n


def oracle_rows(kind, weights, img, cfg):
    """Candidate rows [B, N, row] of the oracle's forward of the whole network on images [B, H, W, 3]."""
    from oracle import nets as ON
    from oracle import tails as OT
    if kind in ("ssd300", "ssd512"):
        return OT.ssd_rows(ON.ssd_heads(weights, img, int(kind[3:])))
    if kind == "retinanet":
        if not cfg.get("is_bottleneck", True):
            import basic_block_ref
            return basic_block_ref.rows(weights, img, cfg["residual_block_list"])
        return OT.retina_rows(ON.retinanet_heads(weights, img, tuple(cfg["residual_block_list"]),
                                                 cfg["init_conv_filters"]))
    if kind == "yolov3":
        return OT.yolo_rows(ON.yolov3_heads(weights, img))
    if kind == "yolov2":
        from oracle import yolov2 as OY
        return OY.yolo2_rows(OY.yolov2_heads(weights, img), cfg["num_classes"])
    return OT.fcos_rows(ON.fcos_heads(weights, img))


def compare_decisions(fam, rows_gpu, rows_ref, geom, ids, keep, boxes, thr, max_boxes, iou_thr):
    """margins.compare_image for any family (YOLOv2 through its own per-row decode)."""
    n = nms_classes(fam)
    with mock.patch.object(MG, "per_row", lambda k, r, g: per_row(fam, r, g)):
        return MG.compare_image("yolo" if fam == "yolo2" else fam, rows_gpu, rows_ref, geom, ids, keep, boxes, thr,
                                max_boxes, iou_thr, n)
