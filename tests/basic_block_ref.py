"""Test references for RetinaNet's basic-block ResNet (`is_bottleneck=False`), composed from the CPU oracle's pieces
(oracle/nets.py, oracle/tfops.py) and numpy: `_residual_block` (RetinaNet.py:621-632), the ResNet built from it, the
detection pyramid and heads on top, and an enumeration of the variables TF 1.13 creates for that graph."""
import numpy as np

F32 = np.float32


def _unit(c, x, stride, scope):
    """_residual_block: conv branch = two BN -> ReLU -> 3x3 convs; shortcut = x at stride 1, else a third one."""
    from oracle import nets as ON
    with c.n.scope(scope):
        with c.n.scope("conv_branch"):
            y = ON._bac(c, x, 3, stride)
            y = ON._bac(c, y, 3, 1)
        with c.n.scope("identity_branch"):
            sc = ON._bac(c, x, 3, stride) if stride != 1 else x
    assert y.shape == sc.shape, (scope, y.shape, sc.shape)
    return (y + sc).astype(F32)


def _resnet(c, x, block_list):
    """`_feature_extractor` with the basic unit (RetinaNet.py:258-285): the three last stage outputs."""
    from oracle import tfops as T
    y = T.relu(c.bn(c.conv(x, 7, 2)))
    y = T.max_pool_same(y, 3, 2)
    ends = []
    for i in range(block_list[0]):
        y = _unit(c, y, 1, "block1_unit%d" % (i + 1))
    ends.append(y)
    for i in range(1, len(block_list)):
        y = _unit(c, y, 2, "block%d_unit1" % (i + 1))
        for j in range(1, block_list[i]):
            y = _unit(c, y, 1, "block%d_unit%d" % (i + 1, j + 1))
        ends.append(y)
    return ends[-3], ends[-2], ends[-1]


def _centred(images):
    from oracle import tfops as T
    return (images.astype(F32) - T.RGB_MEAN.reshape(1, 1, 1, 3)).astype(F32)


def features(weights, images, block_list):
    """The last unit's conv + shortcut sum, NHWC float32 (what pretraining mode pools, RetinaNet.py:121-122)."""
    from oracle import nets as ON
    c = ON.Ctx(weights)
    with c.n.scope("feature_extractor"):
        return _resnet(c, _centred(images), block_list)[-1]


def heads(weights, images, block_list):
    """RetinaNet.py:137-155 on the basic ResNet: [(cls, reg)] per level P3..P7, as oracle.nets.retinanet_heads."""
    from oracle import nets as ON
    c = ON.Ctx(weights)
    with c.n.scope("feature_extractor"):
        f1, f2, f3 = _resnet(c, _centred(images), block_list)
        p5, _ = ON._pyramid(c, f3, None, "bn")
        p4, td = ON._pyramid(c, f2, p5, "bn")
        p3, _ = ON._pyramid(c, f1, td, "bn")
        p6 = ON._bac(c, p5, 3, 2)
        p7 = ON._bac(c, p6, 3, 2)
    out = []
    with c.n.scope("regressor"):
        for p in (p3, p4, p5, p6, p7):
            y = p
            for _ in range(4):
                y = ON._bac(c, y, 3, 1)
            cls = ON._bac(c, y, 3, 1)
            y = p
            for _ in range(4):
                y = ON._bac(c, y, 3, 1)
            out.append((cls, ON._bac(c, y, 3, 1)))
    return out


def rows(weights, images, block_list):
    """Candidate rows [B, N, 25] of the oracle's detection graph."""
    from oracle import tails as OT
    return OT.retina_rows(heads(weights, images, block_list))


def tf_variables(block_list, detection=True, init_conv_filters=7, num_classes=21):
    """name -> shape of every variable the reference graph creates (tf.layers default names, uniquified per variable
    scope in creation order), written out by hand from RetinaNet.py:137-155,258-319,594-632."""
    out = {}
    count = {}

    def unique(scope, base):
        k = count.get((scope, base), 0)
        count[(scope, base)] = k + 1
        return "%s/%s" % (scope, base if k == 0 else "%s_%d" % (base, k))

    def bn(scope, c):
        s = unique(scope, "batch_normalization")
        for v in ("gamma", "beta", "moving_mean", "moving_variance"):
            out[s + "/" + v] = (c,)

    def conv(scope, k, cin, cout):
        s = unique(scope, "conv2d")
        out[s + "/kernel"] = (k, k, cin, cout)
        out[s + "/bias"] = (cout,)

    def bac(scope, k, cin, cout):
        bn(scope, cin)
        conv(scope, k, cin, cout)

    fe = "feature_extractor"
    conv(fe, 7, 3, init_conv_filters)
    bn(fe, init_conv_filters)
    cin, ends = init_conv_filters, []
    for i, n in enumerate(block_list):
        f = 7 * 2 ** i
        for j in range(n):
            stride = 2 if (i > 0 and j == 0) else 1
            u = "%s/block%d_unit%d" % (fe, i + 1, j + 1)
            bac(u + "/conv_branch", 3, cin, f)
            bac(u + "/conv_branch", 3, f, f)
            if stride != 1:
                bac(u + "/identity_branch", 3, cin, f)
            cin = f
        ends.append(f)
    if not detection:
        return out
    c3, c4, c5 = ends[-3:]
    bac(fe, 3, c5, 256)                       # P5
    bac(fe, 1, c4, 256)                       # P4: lateral 1x1, then 3x3 on the sum
    bac(fe, 3, 256, 256)
    bac(fe, 1, c3, 256)                       # P3
    bac(fe, 3, 256, 256)
    bac(fe, 3, 256, 256)                      # P6
    bac(fe, 3, 256, 256)                      # P7
    for _ in range(5):
        for _ in range(4):
            bac("regressor", 3, 256, 256)
        bac("regressor", 3, 256, 9 * num_classes)
        for _ in range(4):
            bac("regressor", 3, 256, 256)
        bac("regressor", 3, 256, 9 * 4)
    return out
