"""CenterNet restated on the CPU in numpy (test oracle): the network (CenterNet.py:50-135, inference BN, float32, sums
in the reference's order), its candidate rows, the peak + top-k tail (:159-185) and the per-image loss (:187-270, in
float64).  Not product code -- see oracle/__init__.py."""
import numpy as np

from . import tfops as T
from .nets import Ctx
from .pfpnet import avg_pool_same, conv2d_transpose_same

F32 = np.float32
MEAN = np.array([0.485, 0.456, 0.406], F32)
STD = np.array([0.229, 0.224, 0.225], F32)
STRIDE = 4


def centernet_heads(weights, images, num_classes=20):
    """images [B,S,S,3] RGB 0..255 -> (keypoints [B,h,w,C], offset [B,h,w,2], size [B,h,w,2]), inference BN."""
    c = Ctx(weights)
    w = weights
    x = ((np.asarray(images, F32) / F32(255.0) - MEAN) / STD).astype(F32)

    def cba(t, k, stride=1, act=True):  # _conv_bn_activation
        y = c.bn(c.conv(t, k, stride))
        return T.relu(y) if act else y

    def dcba(t):  # _dconv_bn_activation
        vs = c.n.unique("conv2d_transpose")
        return T.relu(c.bn(conv2d_transpose_same(t, w[vs + "/kernel"], w[vs + "/bias"])))

    def basic_block(t, f):
        y = cba(cba(t, 3), 3)
        vs, bs = c.n.unique("conv2d"), c.n.unique("batch_normalization")  # tf.cond's untaken branch is built too
        if t.shape[-1] == f:
            return (y + t).astype(F32)
        sc = T.relu(T.batch_norm_inference(T.conv2d_same(t, w[vs + "/kernel"], w[vs + "/bias"]),
                                           w[bs + "/gamma"], w[bs + "/beta"], w[bs + "/moving_mean"],
                                           w[bs + "/moving_variance"]))
        return (y + sc).astype(F32)

    def dla(t, f, levels):
        if levels == 1:
            b1 = basic_block(t, f)
            b2 = basic_block(b1, f)
        else:
            b1 = dla(t, f, levels - 1)
            b2 = dla(b1, f, levels - 1)
        return cba((b1 + b2).astype(F32), 3)

    def stage(t, f, levels):
        d = dla(t, f, levels)
        r = avg_pool_same(cba(t, 1))
        return (T.max_pool_same(d, 2, 2) + r).astype(F32)

    with c.n.scope("backone"):
        x = cba(cba(cba(x, 7), 3), 3, 2)
        s3 = T.max_pool_same(dla(x, 64, 1), 2, 2)
        s4 = stage(s3, 128, 2)
        s5 = stage(s4, 256, 2)
        s6 = stage(s5, 512, 1)
    with c.n.scope("upsampling"):
        s6 = cba(s6, 1)
        u6_5 = dcba(s6)
        u6_4 = dcba(u6_5)
        u6_3 = dcba(u6_4)
        s5 = cba(s5, 1)
        u5_4 = dcba(cba((s5 + u6_5).astype(F32), 3))
        u5_3 = dcba(u5_4)
        s4 = cba(s4, 1)
        u4_3 = dcba(cba(((s4 + u5_4).astype(F32) + u6_4).astype(F32), 3))
        feats = cba(cba(((u6_3 + u5_3).astype(F32) + u4_3).astype(F32), 3), 1)
    with c.n.scope("center_detector"):
        return cba(feats, 3, act=False), cba(feats, 3, act=False), cba(feats, 3, act=False)


def centernet_rows(heads):
    """(keypoints, offset, size) -> candidate rows [B, h*w, C + 4]."""
    kp, off, size = heads
    b = kp.shape[0]
    return np.concatenate([kp.reshape(b, -1, kp.shape[-1]), off.reshape(b, -1, 2), size.reshape(b, -1, 2)],
                          axis=-1).astype(F32)


def sigmoid_f32(x):
    """The float32 value nearest 1 / (1 + exp(-x)): computed in float64, rounded once (what the tail kernel does)."""
    return (1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))).astype(F32)


def centernet_tail(rows, h, w, score_thr, top_k):
    """CenterNet.py:159-185 for ONE image's rows [h*w, C + 4]: best class sigmoid per cell (first maximum), kept where it
    equals its 3x3 SAME max pool (0 elsewhere) and > score_thr, the top min(n, top_k) by descending score with the lower
    cell index first, boxes ((i, j) + (dy, dx) -/+ (h, w) / 2) * 4.  Returns scores, boxes, class ids, cell indices."""
    rows = np.asarray(rows, F32)
    nc = rows.shape[1] - 4
    s = sigmoid_f32(rows[:, :nc])
    cls = np.argmax(s, axis=1).astype(np.int32)
    best = s[np.arange(len(s)), cls].reshape(1, h, w, 1)
    peak = T.max_pool_same(best, 3, 1)
    score = np.where(best == peak, best, F32(0)).reshape(-1)
    idx = np.nonzero(score > F32(score_thr))[0]
    order = idx[np.lexsort((idx, -score[idx].astype(np.float64)))][:top_k]
    yy, xx = (order // w).astype(F32), (order % w).astype(F32)
    cy, cx = (yy + rows[order, nc]).astype(F32), (xx + rows[order, nc + 1]).astype(F32)
    h2, w2 = (rows[order, nc + 2] * F32(0.5)).astype(F32), (rows[order, nc + 3] * F32(0.5)).astype(F32)
    boxes = np.stack([cy - h2, cx - w2, cy + h2, cx + w2], axis=1).astype(F32) * F32(STRIDE)
    return score[order], boxes.astype(F32), cls[order], order.astype(np.int64)


def gaussian_radius(h, w, min_overlap=0.7):
    """CenterNet.py:254-270 before its reduce_min: the three radii (b + sqrt(b^2 - 4ac)) / 2, float64."""
    h, w = np.asarray(h, np.float64), np.asarray(w, np.float64)
    b1, c1 = h + w, w * h * (1 - min_overlap) / (1 + min_overlap)
    b2, c2 = 2 * (h + w), (1 - min_overlap) * w * h
    a3, b3, c3 = 4 * min_overlap, -2 * min_overlap * (h + w), (min_overlap - 1) * w * h
    return ((b1 + np.sqrt(b1 ** 2 - 4 * c1)) / 2, (b2 + np.sqrt(b2 ** 2 - 16 * c2)) / 2,
            (b3 + np.sqrt(b3 ** 2 - 4 * a3 * c3)) / 2)


def centernet_image_loss(rows, h, w, gt):
    """_compute_one_image_loss (CenterNet.py:187-251) for ONE image's rows [h*w, C + 4], in float64; gt [G, 5]
    (y, x, h, w, id) padded with -1.  An image without boxes is 0 (the reference's 0 / 0).  Returns (loss, sigma)."""
    rows = np.asarray(rows, np.float64)
    nc = rows.shape[1] - 4
    gt = np.asarray(gt, F32)
    cnt = int(np.argmin(gt, axis=0)[0])
    if cnt == 0:
        return 0.0, None
    g = (gt[:cnt, :4] * F32(0.25)).astype(np.float64)
    cid = gt[:cnt, 4].astype(np.int64)
    fy = np.clip(np.floor(g[:, 0]).astype(np.int64), 0, h - 1)
    fx = np.clip(np.floor(g[:, 1]).astype(np.int64), 0, w - 1)
    cell = fy * w + fx
    sigma = float(np.min(np.stack(gaussian_radius(g[:, 2], g[:, 3]))))
    yy, xx = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    heat = np.exp(-((g[:, 0, None, None] - yy) ** 2 + (g[:, 1, None, None] - xx) ** 2) / (2 * sigma ** 2))
    red = np.zeros((h * w, nc))
    pos = np.zeros((h * w, nc))
    for c in range(nc):
        m = cid == c
        if m.any():
            red[:, c] = heat[m].max(axis=0).reshape(-1)
            pos[cell[m], c] = 1.0
    k = rows[:, :nc]
    ls = -np.logaddexp(0.0, -k)
    p = np.exp(ls)
    kp = (-(1 - p) ** 2 * ls * pos).sum() / cnt + (-(1 - red) ** 4 * p ** 2 * (-k + ls) * (1 - pos)).sum() / cnt
    at = rows[cell]
    off = np.abs(np.stack([g[:, 0] - np.floor(g[:, 0]), g[:, 1] - np.floor(g[:, 1])], 1) - at[:, nc:nc + 2]).mean()
    size = np.abs(g[:, 2:4] - at[:, nc + 2:nc + 4]).mean()
    return float(kp + 0.1 * size + off), sigma
