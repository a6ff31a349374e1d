"""Layer graphs of SSD300 / SSD512 / RetinaNet / YOLOv3 / YOLOv2 / FCOS / PFPNet-R / CenterNet expressed on the
H100 engine (engine.Net).  Each builder mirrors the reference's layer creation
order so variables get the same TF1 names as in the reference checkpoints
(SURVEY.md App. D); citations give the reference lines each block stands for.
"""

import numpy as np

from . import lib as L
from .engine import ClassifyTail, Net, PeakTail, Tail

F32 = np.float32

_VGG = [("conv1_1", "kernel_conv1_1", "bias_conv1_1", 64), ("conv1_2", "kernel_conv1_2", "bias_conv1_2", 64),
        "pool",
        ("conv2_1", "kenrel_conv2_1", "bias_conv2_1", 128), ("conv2_2", "kernel_conv2_2", "bias_conv2_2", 128),
        "pool",
        ("conv3_1", "kernel_conv3_1", "bias_conv_3_1", 256), ("conv3_2", "kernel_conv3_2", "bias_conv3_2", 256),
        ("conv3_3", "kernel_conv3_3", "bias_conv3_3", 256), "pool",
        ("conv4_1", "kernel_conv4_1", "bias_conv4_1", 512), ("conv4_2", "kernel_conv4_2", "bias_conv4_2", 512),
        ("conv4_3", "kernel_conv4_3", "bias_conv4_3", 512), "pool",
        ("conv5_1", "kernel_conv5_1", "bias_conv5_1", 512), ("conv5_2", "kernel_conv5_2", "bias_conv5_2", 512),
        ("conv5_3", "kernel_conv5_3", "bias_conv5_3", 512)]


def check_num_classes(cfg):
    """The candidate-row layout of the whole path is 25 floats (20 class scores + 5, DESIGN.md section 2): head
    scatter, decode kernel, NMS and the loss kernels hard-code it, so only the VOC class count of every BASELINE
    config is supported.  Any other value would make the head convolutions write overlapping / out-of-bounds rows."""
    if cfg["num_classes"] != 20:
        raise ValueError("num_classes = %r: this path stores 25-float candidate rows and supports exactly 20 "
                         "foreground classes (VOC)" % (cfg["num_classes"],))


MAX_SIGMOID_CLASSES = 128


def check_sigmoid_num_classes(cfg):
    """YOLOv3 and FCOS score each class with its own sigmoid, so their candidate rows hold num_classes + 5 floats
    (DESIGN.md section 2) and any count from 1 to 128 runs.  The limit of 128 comes from the decode kernel: it stages 32
    rows of up to 133 floats (17 KB) per warp in shared memory and keeps one 4-word pass mask per row in registers."""
    nc = cfg["num_classes"]
    if isinstance(nc, bool) or not isinstance(nc, (int, np.integer)) or not 1 <= nc <= MAX_SIGMOID_CLASSES:
        raise ValueError("num_classes = %r: YOLOv3 and FCOS support 1 to %d classes"
                         % (nc, MAX_SIGMOID_CLASSES))


MAX_PRIORS = 9  # ODT_MAX_PRIORS: the prior sizes a level carries in odt_tail_params


def check_yolo_priors(cfg):
    """YOLOv3's anchors: `num_priors` from 1 to 9 and `priors` as three levels of exactly `num_priors` (h, w) pairs of
    positive finite numbers.  The reference reshapes each level with [1, 1, -1, 2] and lets TF broadcast a level of
    one pair over every prior; that is rejected here (DESIGN.md section 1)."""
    npri = cfg["num_priors"]
    if isinstance(npri, bool) or not isinstance(npri, (int, np.integer)) or not 1 <= npri <= MAX_PRIORS:
        raise ValueError("num_priors = %r: YOLOv3 supports 1 to %d priors per level" % (npri, MAX_PRIORS))
    priors = cfg["priors"]
    if not isinstance(priors, (list, tuple, np.ndarray)) or len(priors) != 3:
        raise ValueError("priors = %r: YOLOv3 takes 3 levels of num_priors = %d (h, w) pairs" % (priors, npri))
    for k, level in enumerate(priors):
        try:
            arr = np.asarray(level, dtype=np.float64)
        except (TypeError, ValueError):
            arr = None
        if arr is None or arr.shape != (npri, 2) or not (np.isfinite(arr).all() and (arr > 0).all()):
            raise ValueError("priors[%d] = %r: YOLOv3 takes num_priors = %d positive finite (h, w) pairs per level"
                             % (k, level, npri))


# ------------------------------------------------------------------- SSD ----
def ssd_scales(size):
    """ref SSD300.py:112-113, SSD512.py:116-118 (Python doubles like the reference)."""
    if size == 300:
        s = [(0.2 + (0.9 - 0.2) / 5 * (i - 1)) * size for i in range(1, 8)]
        return [[s[i], (s[i] * s[i + 1]) ** 0.5] for i in range(0, 6)]
    s = [0.07 * size] + [(0.15 + (0.9 - 0.15) / 5 * (i - 1)) * size for i in range(1, 8)]
    return [[s[i], (s[i] * s[i + 1]) ** 0.5] for i in range(0, 7)]


def ssd_ratios(size):
    a2, a4 = [2, 1 / 2], [2, 1 / 2, 3, 1 / 3]
    return [a2, a4, a4, a4, a2, a2] if size == 300 else [a2, a4, a4, a4, a4, a2, a2]


def build_ssd(size, batch, cfg, precision="fp16", device="cuda", allow_tc=True):
    """ref SSD300.py:71-90,192-314 (+SSD512.py:320-322)."""
    check_num_classes(cfg)
    nc = cfg["num_classes"] + 1
    net = Net(batch, size, size, precision, device, allow_tc)
    with net.scope("feature_extractor"):
        x = None
        for item in _VGG:  # VGG-16: conv3x3 + bias + ReLU (:193-302, :514-521)
            if item == "pool":
                x = net.maxpool(x, 2, 2)
                continue
            lname, kn, bnm, cout = item
            x = net.conv(x, cout, 3, kernel_var="feature_extractor/" + kn,
                         bias_var="feature_extractor/" + bnm, act="relu")
            if lname == "conv4_3":
                conv4_3 = x
        x = net.maxpool(x, 3, 1)  # pool5 (:303)

        def cl(x, cout, k, s, name, dil=1):  # _conv_layer: conv -> BN -> ReLU (:523-537)
            return net.conv(x, cout, k, s, dil, name=name, bn=True, act="relu")

        conv6 = cl(x, 1024, 3, 1, "conv6", dil=2)
        conv7 = cl(conv6, 1024, 1, 1, "conv7")
        conv8_2 = cl(cl(conv7, 256, 1, 1, "conv8_1"), 512, 3, 2, "conv8_2")
        conv9_2 = cl(cl(conv8_2, 128, 1, 1, "conv9_1"), 256, 3, 2, "conv9_2")
        conv10_2 = cl(cl(conv9_2, 128, 1, 1, "conv10_1"), 256, 3, 1, "conv10_2")
        conv11_2 = cl(cl(conv10_2, 128, 1, 1, "conv11_1"), 256, 3, 2, "conv11_2")
        feats = [conv4_3, conv7, conv8_2, conv9_2, conv10_2, conv11_2]
        if size == 512:
            feats.append(cl(cl(conv11_2, 128, 1, 1, "conv12_1"), 256, 3, 2, "conv12_2"))
        feats[0] = net.l2norm(feats[0], "feature_extractor/l2_norm_factor")  # :74-83
    ratios, scales = ssd_ratios(size), ssd_scales(size)
    with net.scope("regressor"):
        for i, f in enumerate(feats):  # pred convs: conv -> BN, no activation (:85-90)
            A = len(ratios[i]) + 2
            off = net.add_level(f.H, f.W, A)
            net.conv(f, A * (nc + 4), 3, 1, name="pred%d" % (i + 1), bn=True, act=None,
                     head=(off, 0, 0, 0, A))

    return net, ssd_tail(size, cfg)


def ssd_tail(size, cfg):
    """decode/NMS tail of SSD300/SSD512 (ref SSD300.py:157-190,323-343)."""
    nc = cfg["num_classes"] + 1
    ratios, scales = ssd_ratios(size), ssd_scales(size)

    def level_fn(i, h, w, lv):  # _get_abbox (:323-343)
        lv.cmul_y = lv.cmul_x = float(size)
        lv.cdiv_y, lv.cdiv_x = float(h), float(w)
        lv.out_mul = 1.0
        s = scales[i]
        pri = [[s[0], s[0]], [s[1], s[1]]] + [[s[0] * (ar ** 0.5), s[0] / (ar ** 0.5)] for ar in ratios[i]]
        for a, (ph, pw) in enumerate(pri):
            lv.prior_h[a], lv.prior_w[a] = float(F32(ph)), float(F32(pw))

    return Tail(L.DECODE_SSD, nc - 1, nc - 1, cfg["nms_score_threshold"], cfg["nms_iou_threshold"],
                cfg["nms_max_boxes"], level_fn)


# --------------------------------------------------------- pre-act ResNets --
def _bac(net, x, cout, k, stride, norm, residual=None, head=None, bias_init="zeros"):
    """_bn_activation_conv: norm -> ReLU -> conv (RetinaNet.py:594-619, FCOS.py:467-489)."""
    a = net.preact_bn(x) if norm == "bn" else net.preact_gn(x)
    return net.conv(a, cout, k, stride, residual=residual, head=head, bias_init=bias_init)


def _bottleneck(net, x, f, stride, scope, norm):
    """_residual_bottleneck (RetinaNet.py:634-643): conv + shortcut, shortcut always 3x3."""
    with net.scope(scope):
        with net.scope("identity_branch"):
            sc = _bac(net, x, f * 4, 3, stride, norm)
        with net.scope("conv_branch"):
            y = _bac(net, x, f, 1, 1, norm)
            y = _bac(net, y, f, 3, stride, norm)
            y = _bac(net, y, f * 4, 1, 1, norm, residual=sc)  # residual add fused
    return y


def _basic(net, x, f, stride, scope, norm):
    """_residual_block (RetinaNet.py:621-632): two 3x3 convs + shortcut.  The shortcut is x itself at stride 1 (no
    identity_branch variables) and a 3x3 conv of stride `stride` otherwise."""
    with net.scope(scope):
        sc = x
        if stride != 1:
            with net.scope("identity_branch"):
                sc = _bac(net, x, f, 3, stride, norm)
        with net.scope("conv_branch"):
            y = _bac(net, x, f, 3, stride, norm)
            y = _bac(net, y, f, 3, 1, norm, residual=sc)  # residual add fused
    return y


def _resnet(net, filters, blocks, stem_filters, norm, unit=_bottleneck):
    """stem 7x7 s2 + norm + ReLU, maxpool 3/2, residual-unit stacks
    (RetinaNet.py:258-285, FCOS.py:72-97)."""
    if norm == "bn":
        y = net.conv(None, stem_filters, 7, 2, bn=True, act="relu")
    else:
        y = net.preact_gn(net.conv(None, stem_filters, 7, 2))  # conv -> GN -> ReLU
    y = net.maxpool(y, 3, 2)
    ends = []
    for i in range(blocks[0]):
        y = unit(net, y, filters[0], 1, "block1_unit%d" % (i + 1), norm)
    ends.append(y)
    for i in range(1, len(blocks)):
        y = unit(net, y, filters[i], 2, "block%d_unit1" % (i + 1), norm)
        for j in range(1, blocks[i]):
            y = unit(net, y, filters[i], 1, "block%d_unit%d" % (i + 1, j + 1), norm)
        ends.append(y)
    return ends[-3], ends[-2], ends[-1]


def _pyramid(net, feat, top, norm):
    """_get_pyramid (RetinaNet.py:303-319)."""
    if top is None:
        return _bac(net, feat, 256, 3, 1, norm), None
    f = _bac(net, feat, 256, 1, 1, norm)
    total = net.upsample_add(top, f)
    return _bac(net, total, 256, 3, 1, norm), total


def _retinanet_resnet(net, cfg):
    """RetinaNet's `_feature_extractor` (RetinaNet.py:258-285) under the 'feature_extractor' scope of `net`."""
    blocks = cfg["residual_block_list"]
    filters = [7 * (2 ** i) for i in range(len(blocks))]  # RetinaNet.py:27 quirk
    unit = _bottleneck if cfg["is_bottleneck"] else _basic  # RetinaNet.py:272-275
    return _resnet(net, filters, blocks, cfg["init_conv_filters"], "bn", unit)


def build_retinanet_backbone(batch, cfg, precision="fp16", device="cuda", allow_tc=True):
    """ImageNet-pretraining graph (ref RetinaNet.py:120-127): the same ResNet as build_retinanet -- created first in
    both graphs, so the variable names match -- and a classification tail on its last unit's output (the raw
    conv + shortcut sum: 4 * 7 * 2^(stages-1) channels for the bottleneck variant, 224 logits for four stages;
    7 * 2^(stages-1) for the basic one, 56 logits)."""
    H, W, _ = cfg["data_shape"]
    net = Net(batch, H, W, precision, device, allow_tc)
    with net.scope("feature_extractor"):
        _, _, features = _retinanet_resnet(net, cfg)
    return net, ClassifyTail(features)


def build_retinanet(batch, cfg, precision="fp16", device="cuda", allow_tc=True):
    """ref RetinaNet.py:137-155,258-301."""
    check_num_classes(cfg)
    H, W, _ = cfg["data_shape"]
    nc = cfg["num_classes"] + 1
    net = Net(batch, H, W, precision, device, allow_tc)
    A = 9
    with net.scope("feature_extractor"):
        f1, f2, f3 = _retinanet_resnet(net, cfg)
        p5, _ = _pyramid(net, f3, None, "bn")
        p4, td = _pyramid(net, f2, p5, "bn")
        p3, _ = _pyramid(net, f1, td, "bn")
        p6 = _bac(net, p5, 256, 3, 2, "bn")
        p7 = _bac(net, p6, 256, 3, 2, "bn")
    with net.scope("regressor"):
        for p in (p3, p4, p5, p6, p7):  # towers not shared across levels (:146-155)
            off = net.add_level(p.H, p.W, A)
            y = p
            for _ in range(4):
                y = _bac(net, y, 256, 3, 1, "bn")
            _bac(net, y, nc * A, 3, 1, "bn", head=(off, 0, nc, nc + 4, A), bias_init="pi")
            y = p
            for _ in range(4):
                y = _bac(net, y, 256, 3, 1, "bn")
            _bac(net, y, 4 * A, 3, 1, "bn", head=(off, nc, 4, nc + 4, A))
    return net, retina_tail(cfg)


def retina_tail(cfg):
    """decode/NMS tail of RetinaNet (ref RetinaNet.py:224-256,328-355)."""
    nc = cfg["num_classes"] + 1
    W = cfg["data_shape"][1]
    sizes = [32, 64, 128, 256, 512]

    def level_fn(i, h, w, lv):  # _get_abbox (:328-355): stride = W_in / H_feat for both axes
        rate = float(F32(F32(W) / F32(h)))
        lv.cmul_y = lv.cmul_x = rate
        lv.cdiv_y = lv.cdiv_x = 1.0
        lv.out_mul = 1.0
        a = 0
        for r in [1, 1 / 2, 2]:
            for s in [2 ** 0, 2 ** (1 / 3), 2 ** (2 / 3)]:
                lv.prior_h[a] = float(F32(s * sizes[i] * (r ** 0.5)))
                lv.prior_w[a] = float(F32(s * sizes[i] / (r ** 0.5)))
                a += 1

    return Tail(L.DECODE_SSD, nc - 1, nc - 1, cfg["nms_score_threshold"], cfg["nms_iou_threshold"],
                cfg["nms_max_boxes"], level_fn)


# ---------------------------------------------------------------- YOLOv3 ----
def build_yolov3(batch, cfg, precision="fp16", device="cuda", allow_tc=True):
    """ref YOLOv3.py:81-113,387-417,485-507."""
    H, W, _ = cfg["data_shape"]
    check_sigmoid_num_classes(cfg)
    check_yolo_priors(cfg)
    nc, npri = cfg["num_classes"], cfg["num_priors"]
    net = Net(batch, H, W, precision, device, allow_tc)

    def cl(x, f, k, s, act=True, residual=None, head=None):  # conv -> BN -> leaky (:494-507)
        return net.conv(x, int(f), k, s, bn=True, act="leaky" if act else None, residual=residual,
                        head=head)

    def block(x, f, n, scope):  # _darknet_block (:485-492)
        with net.scope(scope):
            y = cl(x, f, 3, 2)
            for _ in range(n):
                y = cl(cl(y, f // 2, 1, 1), f, 3, 1, residual=y)
        return y

    with net.scope("backone"):
        y = cl(None, 32, 3, 1)
        b1 = block(y, 64, 1, "block1")
        b2 = block(b1, 128, 2, "block2")
        b3 = block(b2, 256, 8, "block3")
        b4 = block(b3, 512, 8, "block4")
        b5 = block(b4, 1024, 4, "block5")

    def header(bottom, f, scope, pyramid=None):  # _yolo3_header (:396-417)
        with net.scope(scope):
            if pyramid is not None:
                u = cl(pyramid, f, 1, 1, act=False)
                y = net.nearest_concat(bottom, u)
            else:
                y = bottom
            c1 = cl(y, f // 2, 1, 1)
            c2 = cl(c1, f, 3, 1)
            c3 = cl(c2, f // 2, 1, 1)
            c4 = cl(c3, f, 3, 1)
            c5 = cl(c4, f // 2, 1, 1)
            c6 = cl(c5, f, 3, 1)
            off = net.add_level(c6.H, c6.W, npri)
            cl(c6, (nc + 5) * npri, 1, 1, head=(off, 0, 0, 0, npri))  # pred has BN+leaky too
        return c5

    with net.scope("head"):
        td = header(b5, 1024, "pyd1")
        td = header(b4, 256, "pyd2", td)
        header(b3, 128, "pyd3", td)
    return net, yolo_tail(cfg)


def yolo_tail(cfg):
    """decode/NMS tail of YOLOv3 (ref YOLOv3.py:320-368,419-433)."""
    nc = cfg["num_classes"]
    stride = [8.0, 16.0, 32.0]
    mult = [stride[-1], stride[-1], stride[-2]]  # :346-348
    priors = cfg["priors"]

    def level_fn(i, h, w, lv):  # _get_priors (:419-433), priors/stride in config order (:38-41)
        lv.cmul_y = lv.cmul_x = lv.cdiv_y = lv.cdiv_x = 1.0
        lv.out_mul = mult[i]
        pr = (np.array(priors[i], dtype=F32) / F32(stride[i])).astype(F32)
        for a in range(cfg["num_priors"]):
            lv.prior_h[a], lv.prior_w[a] = float(pr[a][0]), float(pr[a][1])

    return Tail(L.DECODE_YOLO3, nc, nc, cfg["nms_score_threshold"], cfg["nms_iou_threshold"],
                cfg["nms_max_boxes"], level_fn)


# ---------------------------------------------------------------- YOLOv2 ----
def check_yolo2_config(cfg):
    """YOLOv2's classes and anchors: num_classes from 1 to 128 (the sigmoid rows of YOLOv3, see
    check_sigmoid_num_classes) and `priors` as 1 to 9 (h, w) pairs of positive finite numbers in grid cells; the prior
    count is len(priors) (YOLOv2.py:33), there is no num_priors key."""
    nc = cfg["num_classes"]
    if isinstance(nc, bool) or not isinstance(nc, (int, np.integer)) or not 1 <= nc <= MAX_SIGMOID_CLASSES:
        raise ValueError("num_classes = %r: YOLOv2 supports 1 to %d classes" % (nc, MAX_SIGMOID_CLASSES))
    priors = cfg["priors"]
    try:
        arr = np.asarray(priors, dtype=np.float64)
    except (TypeError, ValueError):
        arr = None
    if arr is None or arr.ndim != 2 or arr.shape[1] != 2 or not 1 <= arr.shape[0] <= MAX_PRIORS:
        raise ValueError("priors = %r: YOLOv2 takes 1 to %d (h, w) pairs" % (priors, MAX_PRIORS))
    if not (np.isfinite(arr).all() and (arr > 0).all()):
        raise ValueError("priors = %r: YOLOv2 takes positive finite (h, w) pairs" % (priors,))


# Darknet-19 of YOLOv2.py:255-303: (name, filters, kernel) of conv1 .. conv18, "pool" for a 2x2/2 SAME max-pool
_DARKNET19 = [("conv1", 32, 3), "pool", ("conv2", 64, 3), "pool",
              ("conv3", 128, 3), ("conv4", 64, 1), ("conv5", 128, 3), "pool",
              ("conv6", 256, 3), ("conv7", 128, 1), ("conv8", 256, 3), "pool",
              ("conv9", 512, 3), ("conv10", 256, 1), ("conv11", 512, 3), ("conv12", 256, 1), ("conv13", 512, 3), "pool",
              ("conv14", 1024, 3), ("conv15", 512, 1), ("conv16", 1024, 3), ("conv17", 512, 1), ("conv18", 1024, 3)]


def build_yolov2(batch, cfg, precision="fp16", device="cuda", allow_tc=True):
    """ref YOLOv2.py:75-100,255-303.  Every `_conv_layer` is conv + bias -> BN; the caller's leaky_relu(0.1) follows
    all of them but `predictions`.  The passthrough is conv17's output on the same 32-pixel grid, concatenated
    before the head's conv5 output (no space-to-depth reorg: the reference has none)."""
    check_yolo2_config(cfg)
    H, W, _ = cfg["data_shape"]
    nc, npri = cfg["num_classes"], len(cfg["priors"])
    net = Net(batch, H, W, precision, device, allow_tc)

    def cl(x, f, k, name, act=True, head=None):
        return net.conv(x, f, k, 1, name=name, bn=True, act="leaky" if act else None, head=head)

    with net.scope("backone"):
        y = None
        for item in _DARKNET19:
            if item == "pool":
                y = net.maxpool(y, 2, 2)
                continue
            y = cl(y, item[1], item[2], item[0])
            if item[0] == "conv17":
                passthrough = y
    with net.scope("head"):
        for i, (f, k) in enumerate([(1024, 3), (512, 1), (1024, 3), (512, 1), (1024, 3)]):
            y = cl(y, f, k, "conv%d" % (i + 1))
        y = net.concat([passthrough, y])
        off = net.add_level(y.H, y.W, npri)
        cl(y, (nc + 5) * npri, 1, "predictions", act=False, head=(off, 0, 0, 0, npri))
    return net, yolo2_tail(cfg)


def yolo2_tail(cfg):
    """decode/NMS tail of YOLOv2 (ref YOLOv2.py:183-210,230-244): YOLOv3's decode on one level -- centre = cell + 0.5 +
    sigmoid, size = prior + exp (additive), corners x 32 -- with the priors as given, in grid cells; per-class NMS over
    every class."""
    nc = cfg["num_classes"]
    priors = np.asarray(cfg["priors"], dtype=F32)

    def level_fn(i, h, w, lv):
        lv.cmul_y = lv.cmul_x = lv.cdiv_y = lv.cdiv_x = 1.0
        lv.out_mul = 32.0
        for a in range(len(priors)):
            lv.prior_h[a], lv.prior_w[a] = float(priors[a][0]), float(priors[a][1])

    return Tail(L.DECODE_YOLO3, nc, nc, cfg["nms_score_threshold"], cfg["nms_iou_threshold"],
                cfg["nms_max_boxes"], level_fn)


# ------------------------------------------------------------------ FCOS ----
def build_fcos(batch, cfg, precision="fp16", device="cuda", allow_tc=True, share_heads=True):
    """ref FCOS.py:70-107,350-364.  Row layout: [cls(num_classes), ctr, l, r, t, b] raw."""
    check_sigmoid_num_classes(cfg)
    H, W, _ = cfg["data_shape"]
    nc = cfg["num_classes"]
    net = Net(batch, H, W, precision, device, allow_tc)
    filters = [16 * (2 ** i) for i in range(4)]
    with net.scope("backone"):
        e3, e4, e5 = _resnet(net, filters, [3, 4, 6, 3], 16, "gn")
    with net.scope("pyramid"):
        c3 = _bac(net, e3, 256, 1, 1, "gn")
        c4 = _bac(net, e4, 256, 1, 1, "gn")
        c5 = _bac(net, e5, 256, 1, 1, "gn")
        p5, _ = _pyramid(net, c5, None, "gn")
        p4, td = _pyramid(net, c4, p5, "gn")
        p3, _ = _pyramid(net, c3, td, "gn")
        p6 = _bac(net, p5, 256, 3, 2, "gn")
        p7 = _bac(net, p6, 256, 3, 2, "gn")
    with net.scope("head"):
        for p in (p3, p4, p5, p6, p7):  # _detect_head, AUTO_REUSE (:350-364)
            if share_heads:
                net.namer.reset_under("head/")
            off = net.add_level(p.H, p.W, 1)
            with net.scope("classifier_head"):
                y = p
                for _ in range(4):
                    y = _bac(net, y, 256, 3, 1, "gn")
                _bac(net, y, nc, 3, 1, "gn", head=(off, 0, 0, 0, 1), bias_init="pi")
                _bac(net, y, 1, 3, 1, "gn", head=(off, nc, 0, 0, 1), bias_init="pi")
            with net.scope("regress_head"):
                y = p
                for _ in range(4):
                    y = _bac(net, y, 256, 3, 1, "gn")
                _bac(net, y, 4, 3, 1, "gn", head=(off, nc + 1, 0, 0, 1))
    return net, fcos_tail(cfg)


def fcos_tail(cfg):
    """decode/NMS tail of FCOS (ref FCOS.py:130-150,197-264); NMS visits num_classes - 1 classes (:252): 19 for VOC,
    none for a single class."""
    nc = cfg["num_classes"]
    strides = [8.0, 16.0, 32.0, 64.0, 128.0]

    def level_fn(i, h, w, lv):  # grid without +0.5 (:130-150), x stride (:242-246)
        lv.cmul_y = lv.cmul_x = lv.cdiv_y = lv.cdiv_x = 1.0
        lv.out_mul = strides[i]

    return Tail(L.DECODE_FCOS, nc, nc - 1, cfg["nms_score_threshold"], cfg["nms_iou_threshold"],
                cfg["nms_max_boxes"], level_fn)


# -------------------------------------------------------------- PFPNet-R ----
def check_pfpnet_config(cfg):
    """PFPNet-R's input size (a positive multiple of 64, PFPNetR.py:15: the pyramid halves the stride-8 grid three
    times) and class count (20: the 21-logit softmax rows of the SSD family, see check_num_classes)."""
    size = cfg["input_size"]
    if isinstance(size, bool) or not isinstance(size, (int, np.integer)) or size <= 0 or size % 64:
        raise ValueError("input_size = %r: PFPNet-R takes a positive multiple of 64" % (size,))
    check_num_classes(cfg)


PFPNET_STRIDES = (8, 16, 32, 64)  # PFPNetR.py:397-400
PFPNET_RATIOS = (0.5, 1.0, 2.0)   # PFPNetR.py:30


def build_pfpnet(batch, cfg, precision="fp16", device="cuda", allow_tc=True):
    """ref PFPNetR.py:74-108,230-431.  Every `_conv_layer` / `_dconv_layer` is conv (+ bias) -> BN (-> ReLU); the
    four 767-channel pyramid concats are stored 800 wide with their 85-channel parts at 32-aligned offsets
    (Net.padded_concat).  Candidate rows: [ODM logits(21), ODM t(4), ARM logits(2), ARM t(4)] per anchor."""
    check_pfpnet_config(cfg)
    size = cfg["input_size"]
    nc = cfg["num_classes"] + 1
    A = len(PFPNET_RATIOS)
    net = Net(batch, size, size, precision, device, allow_tc)
    f = 512 // 6

    def cl(x, cout, k, act=None):  # _conv_layer (:680-694)
        return net.conv(x, cout, k, 1, bn=True, act=act)

    with net.scope("feature_extractor"):
        x = None
        for item in _VGG[:13]:  # conv1_1 .. conv4_3 with the pools between (:231-315)
            if item == "pool":
                x = net.maxpool(x, 2, 2)
                continue
            _, kn, bnm, cout = item
            x = net.conv(x, cout, 3, kernel_var="feature_extractor/" + kn, bias_var="feature_extractor/" + bnm,
                         act="relu")
        fh1 = x
        fh2 = net.resize_ac(fh1, fh1.H // 2, fh1.W // 2)  # :319-326
        fh3 = net.resize_ac(fh1, fh1.H // 4, fh1.W // 4)
        fh4 = net.resize_ac(fh1, fh1.H // 8, fh1.W // 8)
        fl1, fl2, fl3, fl4 = (cl(t, f, 1, "relu") for t in (fh1, fh2, fh3, fh4))  # :332-335

        def up(low, lateral):  # _dconv_layer + lateral, then a 1x1 _conv_layer with ReLU (:336-347)
            return cl(net.deconv(low, f, residual=lateral), f, 1, "relu")

        fl2_1 = up(fl2, fl1)
        fl3_2 = up(fl3, fl2)
        fl3_1 = up(fl3_2, fl1)
        fl4_3 = up(fl4, fl3)
        fl4_2 = up(fl4_3, fl2)
        fl4_1 = up(fl4_2, fl1)
        fl1_2 = cl(net.avgpool(fl1), f, 1)  # avg-pool, then a 1x1 _conv_layer without activation (:349-362)
        fl1_3 = cl(net.avgpool(fl1_2), f, 1)
        fl1_4 = cl(net.avgpool(fl1_3), f, 1)
        fl2_3 = cl(net.avgpool(fl2), f, 1)
        fl2_4 = cl(net.avgpool(fl2_3), f, 1)
        fl3_4 = cl(net.avgpool(fl3), f, 1)
        feat1 = net.padded_concat([fh1, fl2_1, fl3_1, fl4_1])  # :364-395
        feat2 = net.padded_concat([fl1_2, fh2, fl3_2, fl4_2])
        feat3 = net.padded_concat([fl1_3, fl2_3, fh3, fl4_3])
        feat4 = net.padded_concat([fl1_4, fl2_4, fl3_4, fh4])
        feat1 = net.l2norm(feat1, "feature_extractor/feat1_l2_norm", 10.0)  # :77-93
        feat2 = net.l2norm(feat2, "feature_extractor/feat2_l2_norm", 8.0)
    feats = (feat1, feat2, feat3, feat4)
    offs = [net.add_level(t.H, t.W, A) for t in feats]

    def tower(x):  # four 3x3 / 256 _conv_layers with ReLU (:403-408, :423-428)
        for _ in range(4):
            x = cl(x, 256, 3, "relu")
        return x

    # head scatter: channel a * K + k of a K-wide prediction is column col + k of anchor a's row
    row = nc + 10
    with net.scope("ARM"):  # :94-98, :403-411
        for i, t in enumerate(feats):
            with net.scope("arm%d" % (i + 1)):
                y = tower(t)
                net.conv(y, 4 * A, 3, 1, bn=True, head=(offs[i], nc + 6, 4, row, A))
                net.conv(y, 2 * A, 3, 1, bn=True, head=(offs[i], nc + 4, 2, row, A))
    tcbs = [None] * 4
    with net.scope("TCB"):  # :99-103, :413-421
        for i in (3, 2, 1, 0):
            with net.scope("tcb%d" % (i + 1)):
                y = cl(feats[i], 256, 3, "relu")
                if i == 3:
                    tcbs[i] = cl(y, 256, 3, "relu")  # relu(conv2): the top level has no higher feature
                else:
                    c2 = cl(y, 256, 3)
                    tcbs[i] = net.deconv(tcbs[i + 1], 256, residual=c2, act="relu")  # relu(conv2 + BN(dconv))
    with net.scope("ODM"):  # :104-108, :423-431
        for i, t in enumerate(tcbs):
            with net.scope("odm%d" % (i + 1)):
                y = tower(t)
                net.conv(y, 4 * A, 3, 1, bn=True, head=(offs[i], nc, 4, row, A))
                net.conv(y, nc * A, 3, 1, bn=True, head=(offs[i], 0, nc, row, A))
    return net, pfpnet_tail(cfg)


def pfpnet_tail(cfg):
    """two-step decode / NMS tail of PFPNet-R (ref PFPNetR.py:187-228,447-467): anchors of size 4 * stride at ratios
    0.5 / 1 / 2 centred at (i + 0.5) * stride; a row survives when ARM's background probability is below 0.99 and
    ODM's arg-max is a foreground class; ODM's deltas refine the ARM-refined anchor."""
    nc = cfg["num_classes"] + 1

    def level_fn(i, h, w, lv):
        stride = PFPNET_STRIDES[i]
        lv.cmul_y = lv.cmul_x = float(stride)
        lv.cdiv_y = lv.cdiv_x = 1.0
        lv.out_mul = 1.0
        size = 4 * stride
        for a, r in enumerate(PFPNET_RATIOS):
            lv.prior_h[a], lv.prior_w[a] = float(F32(size * (r ** 0.5))), float(F32(size / (r ** 0.5)))

    return Tail(L.DECODE_TWO_STEP, nc - 1, nc - 1, cfg["nms_score_threshold"], cfg["nms_iou_threshold"],
                cfg["nms_max_boxes"], level_fn)


# ------------------------------------------------------------- CenterNet ----
CENTERNET_MEAN = (0.485, 0.456, 0.406)  # CenterNet.py:53-54, on images / 255
CENTERNET_STD = (0.229, 0.224, 0.225)
CENTERNET_STRIDE = 4                    # CenterNet.py:129
MAX_TOP_K = 1024                        # the peak tail selects in one 1024-thread CTA per image


def _positive_int(v):
    return not isinstance(v, bool) and isinstance(v, (int, np.integer)) and v > 0


def check_centernet_config(cfg):
    """CenterNet's input size (a positive multiple of 32: four 2x2 SAME pools after the stride-2 stem, and the
    upsampling sums of CenterNet.py:112-129 need equal sizes), class count (1..128, as YOLOv3 and FCOS) and
    top_k_results_output (1..1024)."""
    size = cfg["input_size"]
    if not _positive_int(size) or size % 32:
        raise ValueError("input_size = %r: CenterNet takes a positive multiple of 32" % (size,))
    nc = cfg["num_classes"]
    if not _positive_int(nc) or nc > MAX_SIGMOID_CLASSES:
        raise ValueError("num_classes = %r: CenterNet supports 1 to %d classes" % (nc, MAX_SIGMOID_CLASSES))
    k = cfg.get("top_k_results_output", 100)
    if not _positive_int(k) or k > MAX_TOP_K:
        raise ValueError("top_k_results_output = %r: CenterNet keeps 1 to %d detections" % (k, MAX_TOP_K))


def build_centernet(batch, cfg, precision="fp16", device="cuda", allow_tc=True):
    """ref CenterNet.py:50-135.  Every layer is conv (+ bias) -> BN (-> ReLU).  The input normalisation
    (x / 255 - mean) / std is the stem's mean subtraction of 255 * mean and a per-channel scale folded into its kernel.
    Sums run as convolution or pixel-shuffle residuals where one side is produced there, otherwise as DLA joins.
    Candidate rows: [keypoint logits(C), dy, dx, h, w] per cell of the stride-4 grid."""
    check_centernet_config(cfg)
    size, nc = cfg["input_size"], cfg["num_classes"]
    net = Net(batch, size, size, precision, device, allow_tc)
    for i in range(3):
        net.mean3[i] = 255.0 * CENTERNET_MEAN[i]
    net.in_scale = [1.0 / (255.0 * s) for s in CENTERNET_STD]

    def cba(x, cout, k, stride=1, act="relu", residual=None):  # _conv_bn_activation (:334-347)
        return net.conv(x, cout, k, stride, bn=True, act=act, residual=residual)

    def basic_block(x, f):
        """conv-BN-ReLU twice + shortcut (:378-389).  tf.cond builds both branches, so the 1x1 shortcut's variables
        exist even where the identity is taken; only the taken branch runs."""
        y = cba(x, f, 3)
        vs2 = net.namer.unique("conv2d")
        net.var(vs2 + "/kernel", (3, 3, f, f), "he")
        net.var(vs2 + "/bias", (f,), "zeros")
        bn2 = net.bn_vars(f)
        vs3 = net.namer.unique("conv2d")
        net.var(vs3 + "/kernel", (1, 1, x.C, f), "he")
        net.var(vs3 + "/bias", (f,), "zeros")
        bn3 = net.bn_vars(f)
        sc = x
        if x.C != f:
            sc = net.conv(x, f, 1, kernel_var=vs3 + "/kernel", bias_var=vs3 + "/bias", bn=True, bn_scope=bn3,
                          act="relu")
        return net.conv(y, f, 3, kernel_var=vs2 + "/kernel", bias_var=vs2 + "/bias", bn=True, bn_scope=bn2,
                        act="relu", residual=sc)

    def dla(x, f, levels, residual=None):
        """_dla_generator (:390-401): conv3x3-BN-ReLU(block1 + block2) (+ residual: the caller's sum)."""
        if levels == 1:
            b1 = basic_block(x, f)
            s = net.dla_join(b1, basic_block(b1, f), pooled=False)
        else:
            b1 = dla(x, f, levels - 1)
            s = dla(b1, f, levels - 1, residual=b1)
        return cba(s, f, 3, residual=residual)

    def stage(x, f, levels):  # max_pool(dla(x)) + avg_pool(conv1x1(x)) (:95-111)
        d = dla(x, f, levels)
        return net.dla_join(d, cba(x, f, 1), pooled=True)

    with net.scope("backone"):
        x = cba(None, 16, 7)
        x = cba(x, 16, 3)
        x = cba(x, 32, 3, 2)
        s3 = net.maxpool(dla(x, 64, 1), 2, 2)
        s4 = stage(s3, 128, 2)
        s5 = stage(s4, 256, 2)
        s6 = stage(s5, 512, 1)
    with net.scope("upsampling"):  # :112-129
        p6_5 = net.deconv_phases(cba(s6, 256, 1), 256, "relu")
        u6_5 = net.shuffle(p6_5)
        p6_4 = net.deconv_phases(u6_5, 256, "relu")
        u6_4 = net.shuffle(p6_4)
        u6_3 = net.shuffle(net.deconv_phases(u6_4, 256, "relu"))
        p5_4 = net.deconv_phases(cba(cba(s5, 256, 1, residual=u6_5), 256, 3), 256, "relu")  # conv(s5) + u6_5
        u5_4 = net.shuffle(p5_4)
        u5_3 = net.shuffle(net.deconv_phases(u5_4, 256, "relu"), residual=u6_3)
        sum4 = net.shuffle(p5_4, residual=cba(s4, 256, 1, residual=u6_4))       # u5_4 + (conv(s4) + u6_4)
        p4_3 = net.deconv_phases(cba(sum4, 256, 3), 256, "relu")
        feats = cba(cba(net.shuffle(p4_3, residual=u5_3), 256, 3), 256, 1)    # u4_3 + (u5_3 + u6_3)
    H = size // CENTERNET_STRIDE
    assert (feats.H, feats.W) == (H, H)
    net.add_level(H, H, 1)
    row = nc + 4
    with net.scope("center_detector"):  # :131-135: conv + bias -> BN, no activation
        net.conv(feats, nc, 3, bn=True, head=(0, 0, nc, row, 1))
        net.conv(feats, 2, 3, bn=True, head=(0, nc, 2, row, 1))
        net.conv(feats, 2, 3, bn=True, head=(0, nc + 2, 2, row, 1))
    return net, centernet_tail(cfg)


def centernet_tail(cfg):
    """Peak + top-k tail (CenterNet.py:159-185)."""
    return PeakTail(cfg["num_classes"], float(cfg.get("score_threshold", 0.1)), int(cfg.get("top_k_results_output",
                                                                                             100)))
