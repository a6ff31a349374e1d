"""PFPNet-R restated on the CPU in numpy fp32 (test oracle): the three TF ops the other oracles lack --
conv2d_transpose (4x4 / 2, SAME) by its scatter definition, resize_bilinear(align_corners=True) and SAME average
pooling --, the network (PFPNetR.py:74-108,230-431, inference BN), its candidate rows and the two-step decode / NMS
tail (:187-228,447-467).  Not product code -- see oracle/__init__.py."""
import numpy as np

from . import tfops as T
from .nets import Ctx, _VGG
from .tails import _per_class_nms

F32 = np.float32
STRIDES = (8, 16, 32, 64)
RATIOS = (0.5, 1.0, 2.0)


def conv2d_transpose_same(x, kernel, bias, stride=2):
    """tf.layers.conv2d_transpose(padding='same') (App. A.1 geometry run backwards): kernel [kh, kw, out, in];
    out size = in * stride, pad_before = total // 2 of the forward conv's SAME padding, and every input pixel i
    scatters x[i] * kernel[k] to output i * stride + k - pad_before.  Sums in float64, rounded once."""
    b, h, w, _ = x.shape
    kh, kw, cout, _ = kernel.shape
    oh, ow = h * stride, w * stride
    pt = max((h - 1) * stride + kh - oh, 0) // 2
    pl = max((w - 1) * stride + kw - ow, 0) // 2
    out = np.zeros((b, oh, ow, cout), np.float64)
    x64, k64 = x.astype(np.float64), kernel.astype(np.float64)
    for ky in range(kh):
        for kx in range(kw):
            contrib = np.einsum("bhwi,oi->bhwo", x64, k64[ky, kx])
            for i in range(h):
                oy = i * stride + ky - pt
                if not 0 <= oy < oh:
                    continue
                xs = np.arange(w) * stride + kx - pl
                ok = (xs >= 0) & (xs < ow)
                out[:, oy, xs[ok]] += contrib[:, i, ok]
    return (out + np.asarray(bias, np.float64)).astype(F32)


def resize_bilinear_ac(x, out_h, out_w):
    """tf.image.resize_bilinear(align_corners=True), TF 1.13: src = dst * scale with scale = (in - 1) / (out - 1) in
    float32 (in / out when out == 1, where the only sample is 0); lower = floor, upper = min(ceil, in - 1),
    top = tl + (tr - tl) * lx, bottom likewise, out = top + (bottom - top) * ly."""
    _, h, w, _ = x.shape

    def axis(n_in, n_out):
        sc = F32(n_in - 1) / F32(n_out - 1) if n_out > 1 else F32(n_in) / F32(n_out)
        src = (np.arange(n_out, dtype=F32) * F32(sc)).astype(F32)
        lo = np.floor(src).astype(np.int64)
        hi = np.minimum(np.ceil(src).astype(np.int64), n_in - 1)
        return lo, hi, (src - np.floor(src)).astype(F32)

    y0, y1, ly = axis(h, out_h)
    x0, x1, lx = axis(w, out_w)
    ly, lx = ly.reshape(1, out_h, 1, 1), lx.reshape(1, 1, out_w, 1)
    x = x.astype(F32)
    tl, tr = x[:, y0][:, :, x0], x[:, y0][:, :, x1]
    bl, br = x[:, y1][:, :, x0], x[:, y1][:, :, x1]
    top = (tl + ((tr - tl).astype(F32) * lx).astype(F32)).astype(F32)
    bot = (bl + ((br - bl).astype(F32) * lx).astype(F32)).astype(F32)
    return (top + ((bot - top).astype(F32) * ly).astype(F32)).astype(F32)


def avg_pool_same(x, k=2, stride=2):
    """tf.layers.average_pooling2d(k, stride, 'same'): SAME geometry, the window's cells inside the image summed
    (row-major) and divided by their count."""
    b, h, w, c = x.shape
    oh, pt, _ = T.same_pad(h, k, stride)
    ow, pl, _ = T.same_pad(w, k, stride)
    out = np.zeros((b, oh, ow, c), F32)
    for i in range(oh):
        for j in range(ow):
            s, n = np.zeros((b, c), F32), 0
            for dy in range(k):
                for dx in range(k):
                    y, xx = i * stride + dy - pt, j * stride + dx - pl
                    if 0 <= y < h and 0 <= xx < w:
                        s = (s + x[:, y, xx]).astype(F32)
                        n += 1
            out[:, i, j] = (s / F32(n)).astype(F32)
    return out


def pfpnet_heads(weights, images, num_classes=21):
    """images [B,S,S,3] RGB 0..255 -> per level i (strides 8..64): (arm_loc [B,h,w,12], arm_conf [B,h,w,6],
    odm_loc [B,h,w,12], odm_conf [B,h,w,3*num_classes]), inference BN."""
    c = Ctx(weights)
    w = weights
    x = (np.asarray(images, F32) - np.array([123.68, 116.779, 103.979], F32)).astype(F32)
    f = 512 // 6

    def cl(t, cout, k, act=False):  # _conv_layer: conv + bias -> BN (-> ReLU)
        y = c.bn(c.conv(t, k))
        return T.relu(y) if act else y

    def dcl(t):  # _dconv_layer: conv2d_transpose + bias -> BN
        vs = c.n.unique("conv2d_transpose")
        return c.bn(conv2d_transpose_same(t, w[vs + "/kernel"], w[vs + "/bias"]))

    with c.n.scope("feature_extractor"):
        for item in _VGG[:13]:
            if item == "pool":
                x = T.max_pool_same(x, 2, 2)
                continue
            x = T.relu(T.conv2d_same(x, w["feature_extractor/" + item[1]], w["feature_extractor/" + item[2]]))
        fh1 = x
        h1, w1 = fh1.shape[1], fh1.shape[2]
        fh2 = resize_bilinear_ac(fh1, h1 // 2, w1 // 2)
        fh3 = resize_bilinear_ac(fh1, h1 // 4, w1 // 4)
        fh4 = resize_bilinear_ac(fh1, h1 // 8, w1 // 8)
        fl1, fl2, fl3, fl4 = [cl(t, f, 1, True) for t in (fh1, fh2, fh3, fh4)]
        fl2_1 = cl((dcl(fl2) + fl1).astype(F32), f, 1, True)
        fl3_2 = cl((dcl(fl3) + fl2).astype(F32), f, 1, True)
        fl3_1 = cl((dcl(fl3_2) + fl1).astype(F32), f, 1, True)
        fl4_3 = cl((dcl(fl4) + fl3).astype(F32), f, 1, True)
        fl4_2 = cl((dcl(fl4_3) + fl2).astype(F32), f, 1, True)
        fl4_1 = cl((dcl(fl4_2) + fl1).astype(F32), f, 1, True)
        fl1_2 = cl(avg_pool_same(fl1), f, 1)
        fl1_3 = cl(avg_pool_same(fl1_2), f, 1)
        fl1_4 = cl(avg_pool_same(fl1_3), f, 1)
        fl2_3 = cl(avg_pool_same(fl2), f, 1)
        fl2_4 = cl(avg_pool_same(fl2_3), f, 1)
        fl3_4 = cl(avg_pool_same(fl3), f, 1)
        feat1 = np.concatenate([fh1, fl2_1, fl3_1, fl4_1], axis=-1)
        feat2 = np.concatenate([fl1_2, fh2, fl3_2, fl4_2], axis=-1)
        feat3 = np.concatenate([fl1_3, fl2_3, fh3, fl4_3], axis=-1)
        feat4 = np.concatenate([fl1_4, fl2_4, fl3_4, fh4], axis=-1)
        feat1 = (T.l2_normalize_channels(feat1) * w["feature_extractor/feat1_l2_norm"].reshape(1, 1, 1, 1)).astype(F32)
        feat2 = (T.l2_normalize_channels(feat2) * w["feature_extractor/feat2_l2_norm"].reshape(1, 1, 1, 1)).astype(F32)
    feats = [feat1, feat2, feat3, feat4]

    def tower(t):
        for _ in range(4):
            t = cl(t, 256, 3, True)
        return t

    arm = []
    with c.n.scope("ARM"):
        for i, t in enumerate(feats):
            with c.n.scope("arm%d" % (i + 1)):
                y = tower(t)
                arm.append((cl(y, 12, 3), cl(y, 6, 3)))
    tcb = [None] * 4
    with c.n.scope("TCB"):
        for i in (3, 2, 1, 0):
            with c.n.scope("tcb%d" % (i + 1)):
                y = cl(cl(feats[i], 256, 3, True), 256, 3)
                if i < 3:
                    y = T.relu((y + dcl(tcb[i + 1])).astype(F32))
                tcb[i] = T.relu(y)
    out = []
    with c.n.scope("ODM"):
        for i, t in enumerate(tcb):
            with c.n.scope("odm%d" % (i + 1)):
                y = tower(t)
                out.append((arm[i][0], arm[i][1], cl(y, 12, 3), cl(y, 3 * num_classes, 3)))
    return out


def pfpnet_rows(heads, num_classes=21):
    """Per-level heads -> candidate rows [B, N, num_classes + 10]: [odm logits, odm t(4), arm logits(2), arm t(4)]."""
    b = heads[0][0].shape[0]
    parts = []
    for al, ac, ol, oc in heads:
        parts.append(np.concatenate([oc.reshape(b, -1, num_classes), ol.reshape(b, -1, 4), ac.reshape(b, -1, 2),
                                     al.reshape(b, -1, 4)], axis=-1))
    return np.concatenate(parts, axis=1).astype(F32)


def pfpnet_anchors(shapes):
    """_get_abbox (PFPNetR.py:447-467) of every level: (y1x1, y2x2, yx, hw), each [N, 2]."""
    parts = []
    for (h, w), stride in zip(shapes, STRIDES):
        size = 4 * stride
        pri = np.array([[size * (r ** 0.5), size / (r ** 0.5)] for r in RATIOS], F32).reshape(1, 1, -1, 2)
        yx = np.zeros((h, w, len(RATIOS), 2), F32)
        yx[..., 0] = ((np.arange(h, dtype=F32) + F32(0.5)) * F32(stride)).reshape(h, 1, 1)
        yx[..., 1] = ((np.arange(w, dtype=F32) + F32(0.5)) * F32(stride)).reshape(1, w, 1)
        y1x1 = (yx - pri / F32(2.0)).astype(F32).reshape(-1, 2)
        y2x2 = (yx + pri / F32(2.0)).astype(F32).reshape(-1, 2)
        parts.append((y1x1, y2x2, (y1x1 / F32(2.0) + y2x2 / F32(2.0)).astype(F32), (y2x2 - y1x1).astype(F32)))
    return [np.concatenate([p[i] for p in parts], axis=0) for i in range(4)]


def pfpnet_tail(rows, shapes, score_thr, max_boxes, iou_thr, num_fg=20):
    """PFPNetR.py:187-228 for ONE image's rows [N, num_fg + 11]: keep rows whose ARM background probability is below
    0.99 and whose ODM arg-max (first maximum) is a foreground class, decode ARM then ODM deltas, per-class NMS of the
    ODM foreground probabilities (>= score_thr).  Returns scores, boxes, class ids and keep indices."""
    nc = num_fg + 1
    rows = np.asarray(rows, F32)
    _, _, ayx, ahw = pfpnet_anchors(shapes)
    arm_p = T.softmax_lastdim(rows[:, nc + 4:nc + 6])
    odm_p = T.softmax_lastdim(rows[:, :nc])
    mask = (arm_p[:, 1] < F32(0.99)) & (np.argmax(odm_p, axis=-1) < num_fg)
    odm_t, arm_t = rows[:, nc:nc + 4], rows[:, nc + 6:nc + 10]
    arm_yx = ((arm_t[:, :2] * ahw).astype(F32) + ayx).astype(F32)
    arm_hw = (np.exp(arm_t[:, 2:]).astype(F32) * ahw).astype(F32)
    odm_yx = ((odm_t[:, :2] * arm_hw).astype(F32) + arm_yx).astype(F32)
    odm_hw = (np.exp(odm_t[:, 2:]).astype(F32) * arm_hw).astype(F32)
    boxes = np.concatenate([(odm_yx - odm_hw / F32(2.0)).astype(F32), (odm_yx + odm_hw / F32(2.0)).astype(F32)], -1)
    idx = np.nonzero(mask)[0].astype(np.int32)
    return _per_class_nms(odm_p[mask][:, :num_fg], boxes[mask], idx, num_fg, score_thr, max_boxes, iou_thr)


def _xent(logits, labels):
    """sparse_softmax_cross_entropy: logsumexp(x) - x[label], float32."""
    logits = np.asarray(logits, F32)
    if not len(labels):
        return np.zeros(0, F32)
    m = logits.max(axis=1, keepdims=True)
    z = (logits - m).astype(F32)
    lse = np.log(np.exp(z).astype(F32).sum(axis=1, dtype=F32)).astype(F32)
    return (lse - z[np.arange(len(labels)), labels]).astype(F32)


def _smooth_l1(x):
    ax = np.abs(x)
    return np.where(ax < 1, F32(0.5) * x * x, ax - F32(0.5)).astype(F32)


def _mean0(x):
    """tf.losses Reduction.MEAN over zero elements is 0 (div_no_nan, TF 1.13 _safe_mean) [TF-sem]; the kernels
    apply the same rule where tf.reduce_mean would give NaN."""
    return float(np.mean(x, dtype=np.float64)) if len(x) else 0.0


def pfpnet_image_loss(rows, shapes, gt, num_fg=20):
    """_compute_one_image_loss (PFPNetR.py:469-610) for ONE image's rows [N, num_fg + 11]; gt [G, 5] (y, x, h, w, id)
    padded with -1.  Returns (loss, info) with info = dict(num_pos, num_neg, num_mined, num_odm_neg)."""
    from . import tails as OT
    nc = num_fg + 1
    rows = np.asarray(rows, F32)
    a1, a2, ayx, ahw = pfpnet_anchors(shapes)
    gt = np.asarray(gt, F32)
    cnt = int(np.argmin(gt, axis=0)[0])                                   # :473-474
    g = gt[:cnt]
    gyx, ghw, label = g[:, 0:2], g[:, 2:4], g[:, 4].astype(np.int64)
    g1, g2 = (gyx - ghw / F32(2.0)).astype(F32), (gyx + ghw / F32(2.0)).astype(F32)
    inter = np.prod(np.maximum(np.minimum(a2[None], g2[:, None]) - np.maximum(a1[None], g1[:, None]), F32(0)),
                    axis=-1).astype(F32)
    iou = (inter / (np.prod(ahw, -1)[None] + np.prod(ghw, -1)[:, None] - inter)).astype(F32)   # :497-502
    N = rows.shape[0]
    best = np.argmax(iou, axis=1) if cnt else np.zeros(0, np.int64)       # :504
    other = np.ones(N, bool)
    other[best] = False
    o_idx = np.nonzero(other)[0]
    if cnt:
        o_best, rg = iou[:, o_idx].max(axis=0), np.argmax(iou[:, o_idx], axis=0)
    else:
        o_best, rg = np.full(len(o_idx), -np.inf, F32), np.zeros(len(o_idx), np.int64)
    pos, neg = o_best > F32(0.5), o_best < F32(0.4)                        # :535-536
    pos_idx = np.concatenate([best, o_idx[pos]]).astype(np.int64)
    pos_g = np.concatenate([np.arange(cnt), rg[pos]]).astype(np.int64)
    neg_idx = o_idx[neg]
    P, nneg = len(pos_idx), len(neg_idx)
    chosen = 3 * P if nneg > 3 * P else nneg                               # :570
    oc, ot, ac, at = rows[:, :nc], rows[:, nc:nc + 4], rows[:, nc + 4:nc + 6], rows[:, nc + 6:nc + 10]
    neg_arm = _xent(ac[neg_idx], np.ones(nneg, np.int64))
    nbox = np.concatenate([ayx[neg_idx] - ahw[neg_idx] / F32(2.0), ayx[neg_idx] + ahw[neg_idx] / F32(2.0)],
                          -1).astype(F32)
    sel = OT.nms_c(nbox, neg_arm, chosen, 0.7) if chosen else np.zeros(0, np.int64)   # :576-579
    mined = neg_idx[sel]
    mined_odm = mined[ac[mined, 1] < F32(0.99)]                            # :584: the raw logit
    sl1 = _smooth_l1
    pa, pyx, pt = ahw[pos_idx], ayx[pos_idx], at[pos_idx]
    tyx = ((gyx[pos_g] - pyx) / pa).astype(F32)
    thw = np.log((ghw[pos_g] / pa).astype(F32)).astype(F32)
    arm = (_mean0(neg_arm[sel]) + _mean0(_xent(ac[pos_idx], np.zeros(P, np.int64)))
           + _mean0(sl1(pt[:, :2] - tyx).sum(-1) + sl1(pt[:, 2:] - thw).sum(-1)))
    arm_yx = ((pt[:, :2] * pa).astype(F32) + pyx).astype(F32)             # :598-599
    arm_hw = (np.exp(pt[:, 2:]).astype(F32) * pa).astype(F32)
    oyx = ((gyx[pos_g] - arm_yx) / arm_hw).astype(F32)                     # :602-603
    ohw = np.log((ghw[pos_g] / arm_hw).astype(F32)).astype(F32)
    odm = (_mean0(_xent(oc[mined_odm], np.full(len(mined_odm), num_fg, np.int64)))
           + _mean0(_xent(oc[pos_idx], label[pos_g]))
           + _mean0(sl1(ot[pos_idx, :2] - oyx).sum(-1) + sl1(ot[pos_idx, 2:] - ohw).sum(-1)))
    return arm + odm, dict(num_pos=P, num_neg=nneg, num_mined=len(sel), num_odm_neg=len(mined_odm))
