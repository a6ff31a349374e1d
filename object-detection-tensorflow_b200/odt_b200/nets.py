"""Layer graphs of SSD300 / SSD512 / RetinaNet / YOLOv3 / FCOS expressed on the
H100 engine (engine.Net).  Each builder mirrors the reference's layer creation
order so variables get the same TF1 names as in the reference checkpoints
(SURVEY.md App. D); citations give the reference lines each block stands for.
"""

import numpy as np

from . import lib as L
from .engine import Net, Tail

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


def _resnet(net, filters, blocks, stem_filters, norm):
    """stem 7x7 s2 + norm + ReLU, maxpool 3/2, bottleneck stacks
    (RetinaNet.py:258-285, FCOS.py:72-97)."""
    if norm == "bn":
        y = net.conv(None, stem_filters, 7, 2, bn=True, act="relu")
    else:
        y = net.preact_gn(net.conv(None, stem_filters, 7, 2))  # conv -> GN -> ReLU
    y = net.maxpool(y, 3, 2)
    ends = []
    for i in range(blocks[0]):
        y = _bottleneck(net, y, filters[0], 1, "block1_unit%d" % (i + 1), norm)
    ends.append(y)
    for i in range(1, len(blocks)):
        y = _bottleneck(net, y, filters[i], 2, "block%d_unit1" % (i + 1), norm)
        for j in range(1, blocks[i]):
            y = _bottleneck(net, y, filters[i], 1, "block%d_unit%d" % (i + 1, j + 1), norm)
        ends.append(y)
    return ends[-3], ends[-2], ends[-1]


def _pyramid(net, feat, top, norm):
    """_get_pyramid (RetinaNet.py:303-319)."""
    if top is None:
        return _bac(net, feat, 256, 3, 1, norm), None
    f = _bac(net, feat, 256, 1, 1, norm)
    total = net.upsample_add(top, f)
    return _bac(net, total, 256, 3, 1, norm), total


def build_retinanet(batch, cfg, precision="fp16", device="cuda", allow_tc=True):
    """ref RetinaNet.py:137-155,258-301."""
    check_num_classes(cfg)
    H, W, _ = cfg["data_shape"]
    nc = cfg["num_classes"] + 1
    blocks = cfg["residual_block_list"]
    assert cfg["is_bottleneck"], "only the bottleneck variant is on the hot path"
    filters = [7 * (2 ** i) for i in range(len(blocks))]  # RetinaNet.py:27 quirk
    net = Net(batch, H, W, precision, device, allow_tc)
    A = 9
    with net.scope("feature_extractor"):
        f1, f2, f3 = _resnet(net, filters, blocks, cfg["init_conv_filters"], "bn")
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
            _bac(net, y, nc * A, 3, 1, "bn", head=(off, 0, nc, 25, A), bias_init="pi")
            y = p
            for _ in range(4):
                y = _bac(net, y, 256, 3, 1, "bn")
            _bac(net, y, 4 * A, 3, 1, "bn", head=(off, nc, 4, 25, A))
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
    nc, npri = cfg["num_classes"], cfg["num_priors"]
    assert npri == 3 and nc == 20, "row layout is 20 classes + 4 box + 1 obj"
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
        for a in range(3):
            lv.prior_h[a], lv.prior_w[a] = float(pr[a][0]), float(pr[a][1])

    return Tail(L.DECODE_YOLO3, nc, nc, cfg["nms_score_threshold"], cfg["nms_iou_threshold"],
                cfg["nms_max_boxes"], level_fn)


# ------------------------------------------------------------------ FCOS ----
def build_fcos(batch, cfg, precision="fp16", device="cuda", allow_tc=True, share_heads=True):
    """ref FCOS.py:70-107,350-364.  Row layout: [cls(20), ctr, l, r, t, b] raw."""
    H, W, _ = cfg["data_shape"]
    nc = cfg["num_classes"]
    assert nc == 20, "row layout is 20 classes + centerness + 4 regressions"
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
    """decode/NMS tail of FCOS (ref FCOS.py:130-150,197-264); NMS visits 19 classes (:252)."""
    nc = cfg["num_classes"]
    strides = [8.0, 16.0, 32.0, 64.0, 128.0]

    def level_fn(i, h, w, lv):  # grid without +0.5 (:130-150), x stride (:242-246)
        lv.cmul_y = lv.cmul_x = lv.cdiv_y = lv.cdiv_x = 1.0
        lv.out_mul = strides[i]

    return Tail(L.DECODE_FCOS, nc, nc - 1, cfg["nms_score_threshold"], cfg["nms_iou_threshold"],
                cfg["nms_max_boxes"], level_fn)
