"""PFPNet-R (no GPU): the constructor's checks, the variables against a hand enumeration of TF 1.13's names, the oracle's
three new TF ops against known answers, the host side of the transposed convolution (phase kernel) and of the padded
concat (filter-row scatter), the candidate-row layout, the oracle tail's two filters, the checkpoint rules and the
host-side checks of the new glue entry points."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import BASE_CFG

F32 = np.float32


def cfg(**over):
    c = dict(BASE_CFG)
    c.update(input_size=320)
    c.update(over)
    return c


def model(**over):
    import PFPNetR
    over.setdefault("bn_init", "trained")
    return PFPNetR.PFPNetR(cfg(**over), None)


# ------------------------------------------------------------------------------------------------ constructor ----
@pytest.mark.parametrize("size", [64, 320, 512])
def test_constructor_accepts_multiples_of_64(size):
    m = model(input_size=size)
    assert m.data_shape == [size, size, 3] and m.num_classes == 21 and m.num_anchors == 3


@pytest.mark.parametrize("size", [0, -64, 300, 96, 320.0, True, "320"])
def test_constructor_rejects_other_sizes(size):
    with pytest.raises(ValueError):
        model(input_size=size)


@pytest.mark.parametrize("nc", [1, 19, 21, 80])
def test_constructor_rejects_other_class_counts(nc):
    with pytest.raises(ValueError):
        model(num_classes=nc)


# --------------------------------------------------------------------------------------------- executor / loss --
@pytest.mark.parametrize("size", [128, 192])
def test_executor_matches_oracle_network(size):
    """train.GraphTrainer's replay of the layer list -- conv_transpose2d with padding 1, align-corners interpolate, the
    SAME average pool, the concats in real channel order -- against oracle/pfpnet.py, inference BN."""
    from odt_b200.train import GraphTrainer
    from oracle.pfpnet import pfpnet_heads, pfpnet_rows
    m = model(input_size=size)
    tr = GraphTrainer(m, "cpu")
    img = np.random.default_rng(size).integers(0, 256, (2, size, size, 3)).astype(F32)
    with torch.no_grad():
        rows = tr.forward_rows(img, training=False).numpy()
    ref = pfpnet_rows(pfpnet_heads(m.get_weights(), img))
    assert rows.shape == ref.shape == (2, 3 * sum((size // s) ** 2 for s in (8, 16, 32, 64)), 31)
    assert np.abs(rows - ref).max() <= 2e-4 * np.abs(ref).max(), (np.abs(rows - ref).max(), np.abs(ref).max())


def loss_rows(N, seed, arm_bg=None):
    """Random rows [N, 31] with O(1) deltas; arm_bg: a value for every raw ARM logit of class 1."""
    rng = np.random.default_rng(seed)
    r = (rng.standard_normal((N, 31)) * 1.5).astype(F32)
    r[:, 21:25] = rng.standard_normal((N, 4)).astype(F32) * 0.4
    r[:, 27:31] = rng.standard_normal((N, 4)).astype(F32) * 0.4
    if arm_bg is not None:
        r[:, 26] = F32(arm_bg)
    return r


def loss_gt(rng, size, n, G=8):
    gt = np.full((G, 5), -1.0, F32)
    gt[:n, 0:2] = rng.uniform(0.15 * size, 0.85 * size, (n, 2))
    gt[:n, 2:4] = rng.uniform(0.1 * size, 0.6 * size, (n, 2))
    gt[:n, 4] = rng.integers(0, 20, n)
    return gt


def trainer_on_levels(levels, dtype=torch.float32):
    """A CPU trainer whose loss restatement runs on the level table `levels` (tiny tables make the empty cases)."""
    from odt_b200.train import GraphTrainer
    tr = GraphTrainer(model(input_size=64), "cpu", dtype)
    tr.net.levels = list(levels)
    tr._anchor_cache = None
    return tr


LEVELS_320 = [(40, 40, 3), (20, 20, 3), (10, 10, 3), (5, 5, 3)]


def empty_cases():
    """(levels, rows, gt, what): an image without boxes; one without negatives (every anchor of a 1x1 level is a GT's
    best); one whose mined negatives all fail the raw-logit test."""
    one = [(1, 1, 3)]
    gt_all = np.full((4, 5), -1.0, F32)
    for a, r in enumerate((0.5, 1.0, 2.0)):
        gt_all[a] = [4.0, 4.0, 32 * r ** 0.5, 32 / r ** 0.5, a]
    return [(LEVELS_320, loss_rows(4800 + 1200 + 300 + 75, 1), np.full((8, 5), -1.0, F32), "no boxes"),
            (one, loss_rows(3, 2), gt_all, "no negatives"),
            (LEVELS_320, loss_rows(6375, 3, arm_bg=1.5), loss_gt(np.random.default_rng(3), 320, 5), "no ODM negative")]


def test_restated_loss_matches_oracle():
    """train.pfpnet_image_loss against oracle/pfpnet.py's numpy fp32 loss at 320², and the three empty cases."""
    from oracle.pfpnet import pfpnet_image_loss
    tr = trainer_on_levels(LEVELS_320)
    shapes = [(h, w) for h, w, _ in LEVELS_320]
    rows = loss_rows(6375, 11)
    rng = np.random.default_rng(4)
    for n in (1, 6, 8):
        gt = loss_gt(rng, 320, n)
        want, info = pfpnet_image_loss(rows, shapes, gt)
        assert info["num_mined"] > 0 and info["num_odm_neg"] > 0 and info["num_pos"] >= n
        got = float(tr.image_loss(torch.from_numpy(rows), gt))
        assert abs(got - want) <= 3e-5 * max(abs(want), 1.0), (n, got, want)
    for levels, r, gt, what in empty_cases():
        t = trainer_on_levels(levels)
        want, info = pfpnet_image_loss(r, [(h, w) for h, w, _ in levels], gt)
        got = float(t.image_loss(torch.from_numpy(r), gt))
        assert np.isfinite(want) and abs(got - want) <= 3e-5 * max(abs(want), 1.0), (what, got, want)
        if what == "no boxes":
            assert want == 0.0 and info["num_pos"] == 0
        elif what == "no negatives":
            assert info["num_neg"] == 0 and info["num_pos"] == 3 and want > 0
        else:
            assert info["num_mined"] > 0 and info["num_odm_neg"] == 0


def test_loss_gradient_matches_finite_differences():
    """d pfpnet_image_loss / d rows by autograd (float64) against central differences of the oracle's loss, on
    positive rows -- ARM and ODM logits and deltas -- and mined negatives.  The ARM deltas of a positive carry a term
    from the ODM smooth-L1 (its targets come from the decoded ARM box): the gradient differs from the ARM term alone."""
    from oracle.pfpnet import pfpnet_image_loss
    levels = [(10, 10, 3), (5, 5, 3), (3, 3, 3), (2, 2, 3)]
    shapes = [(h, w) for h, w, _ in levels]
    N = 3 * (100 + 25 + 9 + 4)
    tr = trainer_on_levels(levels, torch.float64)
    rows = loss_rows(N, 21)
    gt = loss_gt(np.random.default_rng(2), 80, 3)
    r0 = torch.from_numpy(rows.astype(np.float64)).requires_grad_(True)
    tr.image_loss(r0, gt).backward()
    grad = r0.grad.numpy()
    pos = sorted(set(np.nonzero(np.abs(grad[:, :21]).sum(-1) * (np.abs(grad[:, 21:25]).sum(-1) > 0))[0]))
    neg = [n for n in np.nonzero(np.abs(grad[:, 25:27]).sum(-1))[0] if n not in pos][:3]
    assert len(pos) >= 3 and neg
    entries = [(n, c) for n in pos for c in (0, 5, 20, 21, 24, 25, 27, 28, 29, 30)] + [(n, c) for n in neg
                                                                                       for c in (20, 25, 26)]

    def ref(r):
        return pfpnet_image_loss(r, shapes, gt)[0]

    eps = 1e-2
    for n, c in entries:
        up, dn = rows.copy(), rows.copy()
        up[n, c] += F32(eps)
        dn[n, c] -= F32(eps)
        fd = (ref(up) - ref(dn)) / (float(up[n, c]) - float(dn[n, c]))
        assert abs(fd - grad[n, c]) <= 2e-3 * max(abs(grad[n, c]), 0.05), (n, c, fd, grad[n, c])
    # the ARM deltas' gradient depends on the ODM deltas only through the ODM smooth-L1 against the decoded ARM box
    moved = rows.astype(np.float64)
    moved[pos, 21:25] += 0.3
    r1 = torch.from_numpy(moved).requires_grad_(True)
    tr.image_loss(r1, gt).backward()
    assert np.abs(r1.grad.numpy()[pos][:, 27:31] - grad[pos][:, 27:31]).max() > 1e-3


def test_one_step_is_momentum_on_the_restated_loss():
    """tr.step = v - lr * (dL/dv) on the first step (Momentum slots start at zero), L = batch mean of the image losses
    + weight_decay * sum(l2_loss); the BN moving statistics move toward the batch moments; global_step counts."""
    from odt_b200.train import GraphTrainer
    size = 64
    m = model(input_size=size)
    tr = GraphTrainer(m, "cpu")
    ref = GraphTrainer(m, "cpu")
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (2, size, size, 3)).astype(F32)
    gt = np.stack([loss_gt(rng, size, 3), loss_gt(rng, size, 0)])
    stats = []
    rows = ref.forward_rows(img, True, stats)
    data = (ref.image_loss(rows[0], gt[0]) + ref.image_loss(rows[1], gt[1])) / 2
    l2 = sum((p * p).sum() for p in ref.params.values()) * 0.5
    loss = data + float(m.weight_decay) * l2
    names = list(ref.params)
    grads = torch.autograd.grad(loss, [ref.params[k] for k in names], allow_unused=True)
    lr = 1e-3
    got = tr.step(img, gt, lr)
    assert abs(got - float(loss.detach())) <= 1e-5 * abs(float(loss.detach()))
    moved = 0
    for k, g in zip(names, grads):
        g = torch.zeros_like(ref.params[k]) if g is None else g
        want = ref.params[k].detach() - lr * g
        assert torch.allclose(tr.params[k].detach(), want, rtol=1e-5, atol=1e-7), k
        moved += bool((g != 0).any())
    assert moved > len(names) // 2
    for scope, mean, var in stats[:3]:
        mm = m.get_weights()[scope + "/moving_mean"]
        assert torch.allclose(tr.buffers[scope + "/moving_mean"], torch.from_numpy(mm * 0.99) + 0.01 * mean,
                              atol=1e-6)
    assert tr.global_step == 1


# ------------------------------------------------------------------------------------------------- variables ----
def _bn(scope, c):
    return [(scope + "/" + k, (c,)) for k in ("gamma", "beta", "moving_mean", "moving_variance")]


def _conv(scope, k, cin, cout, name="conv2d", transpose=False):
    shape = (k, k, cout, cin) if transpose else (k, k, cin, cout)
    return [(scope + "/" + name + "/kernel", shape), (scope + "/" + name + "/bias", (cout,))]


def _suffix(base, i):
    return base if i == 0 else "%s_%d" % (base, i)


def expected_variables():
    """TF 1.13's names in creation order (PFPNetR.py:74-108,230-431): tf.layers names each conv2d /
    conv2d_transpose / batch_normalization layer uniquely per variable scope, in creation order."""
    out = []
    fe = "feature_extractor"
    vgg = [("kernel_conv1_1", "bias_conv1_1", 3, 64), ("kernel_conv1_2", "bias_conv1_2", 64, 64),
           ("kenrel_conv2_1", "bias_conv2_1", 64, 128), ("kernel_conv2_2", "bias_conv2_2", 128, 128),
           ("kernel_conv3_1", "bias_conv_3_1", 128, 256), ("kernel_conv3_2", "bias_conv3_2", 256, 256),
           ("kernel_conv3_3", "bias_conv3_3", 256, 256), ("kernel_conv4_1", "bias_conv4_1", 256, 512),
           ("kernel_conv4_2", "bias_conv4_2", 512, 512), ("kernel_conv4_3", "bias_conv4_3", 512, 512)]
    for kn, bn, cin, cout in vgg:
        out += [(fe + "/" + kn, (3, 3, cin, cout)), (fe + "/" + bn, (cout,))]
    conv, bnk, dconv = [0], [0], [0]

    def cl(cin, cout=85):
        nonlocal out
        out += _conv(fe, 1, cin, cout, _suffix("conv2d", conv[0])) + _bn(fe + "/" + _suffix("batch_normalization",
                                                                                            bnk[0]), cout)
        conv[0] += 1
        bnk[0] += 1

    def dcl():
        nonlocal out
        out += _conv(fe, 4, 85, 85, _suffix("conv2d_transpose", dconv[0]), True)
        out += _bn(fe + "/" + _suffix("batch_normalization", bnk[0]), 85)
        dconv[0] += 1
        bnk[0] += 1

    for cin in (512, 512, 512, 512):  # fl1 .. fl4
        cl(cin)
    for _ in range(6):  # fl2_1, fl3_2, fl3_1, fl4_3, fl4_2, fl4_1: dconv then 1x1
        dcl()
        cl(85)
    for _ in range(6):  # fl1_2, fl1_3, fl1_4, fl2_3, fl2_4, fl3_4
        cl(85)
    out += [(fe + "/feat1_l2_norm", (1,)), (fe + "/feat2_l2_norm", (1,))]
    for i in range(1, 5):
        s = "ARM/arm%d" % i
        cins = [767, 256, 256, 256, 256, 256]
        couts = [256, 256, 256, 256, 12, 6]
        for j, (ci, co) in enumerate(zip(cins, couts)):
            out += _conv(s, 3, ci, co, _suffix("conv2d", j)) + _bn(s + "/" + _suffix("batch_normalization", j), co)
    for i in (4, 3, 2, 1):
        s = "TCB/tcb%d" % i
        out += _conv(s, 3, 767, 256) + _bn(s + "/batch_normalization", 256)
        out += _conv(s, 3, 256, 256, "conv2d_1") + _bn(s + "/batch_normalization_1", 256)
        if i < 4:
            out += _conv(s, 4, 256, 256, "conv2d_transpose", True) + _bn(s + "/batch_normalization_2", 256)
    for i in range(1, 5):
        s = "ODM/odm%d" % i
        couts = [256, 256, 256, 256, 12, 63]
        for j, co in enumerate(couts):
            out += _conv(s, 3, 256, co, _suffix("conv2d", j)) + _bn(s + "/" + _suffix("batch_normalization", j), co)
    return out


def test_variables_match_tf_names_and_shapes():
    got = [(k, v[0]) for k, v in model().variables().items()]
    assert got == expected_variables()


def test_initial_l2_norm_factors_and_vgg_pretraining_names():
    w = model().get_weights()
    assert w["feature_extractor/feat1_l2_norm"].tolist() == [10.0]
    assert w["feature_extractor/feat2_l2_norm"].tolist() == [8.0]
    from odt_b200.api import VGG16_CKPT_NAMES
    mine = [v for pair in VGG16_CKPT_NAMES.values() for v in pair if v in w]
    assert len(mine) == 20  # conv1_1 .. conv4_3 read from vgg_16.ckpt (PFPNetR.py:35,231-315); no conv5


# ------------------------------------------------------------------------------------- oracle ops: known answers --
@pytest.mark.parametrize("h,w", [(1, 1), (3, 5), (4, 4), (7, 2)])
def test_oracle_conv2d_transpose_is_the_scatter_definition(h, w):
    """Against PyTorch's conv_transpose2d with padding 1 (the same scatter: out = 2 * in, pad_before = 1), and at 1x1
    against the hand answer: the single input pixel reaches the four outputs through the taps [1:3, 1:3]."""
    from oracle.pfpnet import conv2d_transpose_same
    rng = np.random.default_rng(h * 10 + w)
    x = rng.standard_normal((2, h, w, 3)).astype(F32)
    k = rng.standard_normal((4, 4, 5, 3)).astype(F32)
    b = rng.standard_normal(5).astype(F32)
    got = conv2d_transpose_same(x, k, b)
    assert got.shape == (2, 2 * h, 2 * w, 5)
    t = F.conv_transpose2d(torch.from_numpy(x).double().permute(0, 3, 1, 2),
                           torch.from_numpy(k).double().permute(3, 2, 0, 1), torch.from_numpy(b).double(),
                           stride=2, padding=1)
    np.testing.assert_allclose(got, t.permute(0, 2, 3, 1).numpy(), rtol=1e-5, atol=1e-5)
    if h == w == 1:
        exp = np.einsum("bi,yxoi->byxo", x[:, 0, 0].astype(np.float64), k[1:3, 1:3].astype(np.float64)) + b
        np.testing.assert_allclose(got, exp, rtol=1e-6, atol=1e-6)


def test_oracle_resize_align_corners_known_answers():
    from oracle.pfpnet import resize_bilinear_ac
    x = np.arange(5 * 9, dtype=F32).reshape(1, 5, 9, 1)  # value = 9 y + x: bilinear reproduces it exactly
    y = resize_bilinear_ac(x, 3, 5)  # scale (5-1)/(3-1) = 2, (9-1)/(5-1) = 2: every sample on a grid point
    np.testing.assert_array_equal(y[0, :, :, 0], 9 * np.arange(0, 5, 2)[:, None] + np.arange(0, 9, 2)[None, :])
    y = resize_bilinear_ac(x, 2, 4)  # scale 4 and 8/3: the corners map to the corners, the rest interpolates
    np.testing.assert_allclose(y[0, :, :, 0], 9 * np.array([0, 4])[:, None] + np.arange(4)[None, :] * F32(8) / 3,
                               rtol=1e-6)
    y = resize_bilinear_ac(x, 1, 1)  # out == 1: the one sample is pixel (0, 0)
    assert y.shape == (1, 1, 1, 1) and y[0, 0, 0, 0] == 0.0
    z = resize_bilinear_ac(np.random.default_rng(0).standard_normal((2, 7, 6, 3)).astype(F32), 7, 6)
    np.testing.assert_array_equal(z, resize_bilinear_ac(z, 7, 6))  # same size: the identity


@pytest.mark.parametrize("h,w", [(3, 3), (5, 4), (1, 7), (6, 6)])
def test_oracle_avg_pool_same_divides_by_cells_inside(h, w):
    from oracle.pfpnet import avg_pool_same
    x = np.random.default_rng(h * w).standard_normal((1, h, w, 2)).astype(F32)
    y = avg_pool_same(x)
    assert y.shape == (1, (h + 1) // 2, (w + 1) // 2, 2)
    for i in range(y.shape[1]):
        for j in range(y.shape[2]):
            win = x[0, 2 * i:2 * i + 2, 2 * j:2 * j + 2].reshape(-1, 2).astype(np.float64)
            np.testing.assert_allclose(y[0, i, j], win.mean(0), rtol=1e-6, atol=1e-7)
    if (h, w) == (3, 3):
        assert y[0, 1, 1, 0] == x[0, 2, 2, 0]  # the corner window holds one cell: divided by 1, not 4


# ------------------------------------------------------------------------------ host side of the new layers ----
def _spec(size=128):
    m = model(input_size=size)
    net = m._build_spec()
    return m, net


@pytest.mark.parametrize("h,w", [(5, 5), (4, 7)])
def test_phase_kernel_is_the_transposed_convolution(h, w):
    """PhaseConvOp's 3x3 kernel of 4 * cout phase-major outputs (+ the tiled bias), placed on the 2x grid as
    odt_pixel_shuffle2x does, equals conv2d_transpose by the scatter definition."""
    from odt_b200 import engine as E
    from oracle import tfops as T
    from oracle.pfpnet import conv2d_transpose_same
    m, net = _spec()
    op = next(o for o in net.ops if isinstance(o, E.PhaseConvOp))
    rng = np.random.default_rng(3)
    wts = dict(m.get_weights())
    wts[op.kernel] = rng.standard_normal(wts[op.kernel].shape).astype(F32)
    wts[op.bias] = rng.standard_normal(wts[op.bias].shape).astype(F32)
    net.weights = wts
    kern, bias = op.host_weights(net)
    cout = wts[op.bias].shape[0]
    assert kern.shape == (3, 3, 85, 4 * cout) and bias.shape == (4 * cout,)
    x = rng.standard_normal((1, h, w, 85)).astype(F32)
    ph = T.conv2d_same(x, kern, bias)
    out = np.zeros((1, 2 * h, 2 * w, cout), F32)
    for py in range(2):
        for px in range(2):
            out[:, py::2, px::2] = ph[..., (2 * py + px) * cout:(2 * py + px + 1) * cout]
    np.testing.assert_allclose(out, conv2d_transpose_same(x, wts[op.kernel], wts[op.bias]), rtol=2e-4, atol=2e-4)
    sc, sh = op.host_bn(net)
    s1, h1 = net.bn_fold(op.bn)
    assert np.array_equal(sc, np.tile(s1, 4)) and np.array_equal(sh, np.tile(h1, 4))


def test_padded_concats_and_filter_row_scatter():
    """The four 767-channel concats are stored 800 wide, parts at 32-aligned offsets in the reference's order; a
    consumer's filter rows land on the stored channels and the gaps stay zero."""
    from odt_b200 import engine as E
    m, net = _spec()
    bases = []
    for t in net.acts:
        if t.base is not None and t.base not in bases:
            bases.append(t.base)
    assert [b.C for b in bases] == [800] * 4
    widths = [[p.C for p in b.parts] for b in bases]
    assert widths == [[512, 85, 85, 85], [85, 512, 85, 85], [85, 85, 512, 85], [85, 85, 85, 512]]
    for b in bases:
        assert [p.c0 for p in b.parts] == list(np.cumsum([0] + [(p.C + 31) // 32 * 32 for p in b.parts])[:4])
        assert np.array_equal(b.chan_map, np.concatenate([np.arange(p.c0, p.c0 + p.C) for p in b.parts]))
    arm = next(o for o in net.ops if isinstance(o, E.ConvOp) and o.kernel == "ARM/arm3/conv2d/kernel")
    wts = dict(m.get_weights())
    net.weights = wts
    kern, _ = arm.host_weights(net)
    assert kern.shape == (3, 3, 800, 256)
    cmap = arm.x.chan_map
    assert np.array_equal(kern[:, :, cmap], wts[arm.kernel])
    gaps = np.setdiff1d(np.arange(800), cmap)
    assert len(gaps) == 33 and not kern[:, :, gaps].any()


def test_candidate_rows_and_levels():
    from odt_b200 import lib
    for size, grids in ((320, (40, 20, 10, 5)), (512, (64, 32, 16, 8))):
        m, net = _spec(size)
        assert net.tail.kind == lib.DECODE_TWO_STEP and net.tail.row == 31 and net.tail.nms_classes == 20
        assert net.levels == [(g, g, 3) for g in grids]
        heads = [o.head for o in net.ops if getattr(o, "head", None) is not None]
        cols = sorted((h[1], h[2]) for h in heads)
        assert cols == [(0, 21)] * 4 + [(21, 4)] * 4 + [(25, 2)] * 4 + [(27, 4)] * 4
        p = net.tail.params(net.levels)
        for i, s in enumerate((8, 16, 32, 64)):
            lv = p.level[i]
            assert (lv.cmul_y, lv.cdiv_y) == (s, 1.0)
            np.testing.assert_allclose([lv.prior_h[a] for a in range(3)], [4 * s * r ** 0.5 for r in (0.5, 1, 2)],
                                       rtol=1e-7)


def test_oracle_tail_filters():
    """Rows just either side of ARM's 0.99 background cut, and rows whose ODM arg-max is the background, against the
    tail's rule (PFPNetR.py:188-192)."""
    from oracle.pfpnet import pfpnet_tail
    shapes = [(2, 2), (1, 1)]
    N = 3 * 5
    rows = np.zeros((N, 31), F32)
    rows[:, 0] = 5.0  # class 0 wins the ODM softmax ...
    rows[1, 20] = 5.0  # ... unless the background ties (first maximum: class 0 still) ...
    rows[2, 20] = 5.5  # ... or wins
    d = np.log(99.0)  # ARM p(bg) = sigmoid(a1 - a0): 0.99 at a1 - a0 = log 99
    rows[3, 26] = F32(d + 1e-3)
    rows[4, 26] = F32(d - 1e-3)
    s, b, c, k = pfpnet_tail(rows, shapes, 0.3, 100, 1.0)
    assert sorted(k.tolist()) == sorted(set(range(N)) - {2, 3})
    assert np.all(c == 0)


# --------------------------------------------------------------------------------------------- checkpoints ----
def test_checkpoint_round_trip(tmp_path):
    src = model()
    src.set_weights({k: v + np.float32(0.25) for k, v in src.get_weights().items()})
    src.global_step = 11
    path = src.save_weight("latest", str(tmp_path / "pfpnet" / "test"))
    assert path.endswith("test-11")
    dst = model()
    dst.load_weight(path)
    assert dst.global_step == 11
    assert all(np.array_equal(src.get_weights()[k], dst.get_weights()[k]) for k in src.get_weights())


def test_ssd_checkpoint_is_refused(tmp_path):
    from odt_b200 import tf_checkpoint
    from helpers import model_cfg
    import SSD300
    path = SSD300.SSD300(model_cfg("ssd"), None).save_weight("latest", str(tmp_path / "ssd"))
    dst = model()
    w0 = {k: v.copy() for k, v in dst.get_weights().items()}
    with pytest.raises(tf_checkpoint.CheckpointError):
        dst.load_weight(path)
    w1 = dst.get_weights()
    assert all(np.array_equal(w0[k], w1[k]) for k in w0), "nothing may be restored from a refused checkpoint"


def test_checkpoint_with_a_reshaped_variable_is_refused(tmp_path):
    from odt_b200 import tf_checkpoint
    src = model()
    w = dict(src.get_weights())
    w["ODM/odm1/conv2d_5/bias"] = np.zeros(64, F32)
    src._weights = w
    path = src.save_weight("latest", str(tmp_path / "bad"))
    with pytest.raises(tf_checkpoint.CheckpointError):
        model().load_weight(path)


# ------------------------------------------------------------------------------------------ C argument checks ----
def test_glue_entry_points_check_on_the_host(built):
    from odt_b200 import lib
    L = lib.load()
    fake = ctypes.c_void_p(64)  # never dereferenced: every call below is rejected first

    def refused(rc):
        return rc == -1 and b"args" in L.odt_last_error()

    assert refused(L.odt_pixel_shuffle2x(None, fake, None, 0, 1, 2, 2, 85, 384, 128, 0, 0, None))
    assert refused(L.odt_pixel_shuffle2x(fake, fake, None, 0, 1, 2, 2, 85, 339, 128, 0, 0, None))  # in_ld < 4C
    assert refused(L.odt_pixel_shuffle2x(fake, fake, fake, 0, 1, 2, 2, 85, 384, 128, 84, 0, None))  # res_ld < C
    assert refused(L.odt_pixel_shuffle2x(fake, fake, None, 0, 1, 2, 2, 85, 384, 128, 0, 3, None))  # act
    assert refused(L.odt_resize_bilinear_ac(fake, fake, None, 0, 1, 4, 4, 8, 8, 0, 2, 8, 0, None))  # OH = 0
    assert refused(L.odt_resize_bilinear_ac(fake, fake, fake, 0, 1, 4, 4, 8, 8, 2, 2, 8, 7, None))  # out2_ld < C
    assert refused(L.odt_avgpool2x2_same(fake, fake, 0, 1, 3, 3, 8, 7, 8, None))  # in_ld < C
    assert refused(L.odt_avgpool2x2_same(fake, None, 0, 1, 3, 3, 8, 8, 8, None))
    rc = L.odt_pixel_shuffle2x(fake, fake, None, 5, 1, 2, 2, 85, 384, 128, 0, 0, None)
    assert rc == -1 and b"dtype" in L.odt_last_error()


def test_two_step_tail_is_checked_on_the_host(built):
    """The decode and NMS entry points take the two-step kind at 20 classes only; the loss entry points refuse it."""
    from odt_b200 import lib
    L = lib.load()
    fake = ctypes.c_void_p(64)
    p = lib.TailParams()
    p.kind, p.num_levels, p.N, p.num_fg, p.nms_classes, p.cap, p.max_boxes = lib.DECODE_TWO_STEP, 1, 12, 19, 19, 12, 5
    p.level[0].H, p.level[0].W, p.level[0].A = 2, 2, 3
    assert L.odt_decode_candidates(fake, ctypes.byref(p), 1, fake, fake, None) == -1
    assert b"num_fg must be 20" in L.odt_last_error()
    p.kind = 4
    assert L.odt_decode_candidates(fake, ctypes.byref(p), 1, fake, fake, None) == -1
    assert b"kind" in L.odt_last_error()
    p.kind, p.num_fg, p.nms_classes = lib.DECODE_TWO_STEP, 20, 20
    assert L.odt_ssd_loss_fwd(fake, ctypes.byref(p), 1, fake, 4, fake, fake, None, None) == -1
    assert b"softmax-family head" in L.odt_last_error()


def test_driver_config_constructs_and_exposes_the_reference_surface():
    import PFPNetR as net
    config = {"mode": "test", "data_format": "channels_last", "input_size": 320, "num_classes": 20,
              "weight_decay": 1e-4, "keep_prob": 0.5, "batch_size": 32, "nms_score_threshold": 0.5,
              "nms_max_boxes": 20, "nms_iou_threshold": 0.5, "pretraining_weight": None}
    m = net.PFPNetR(config, None)
    for name in ("test_one_image", "detect_batch", "detect_stream", "train_one_epoch", "loss_forward",
                 "save_weight", "load_weight", "get_weights", "engine", "trainer"):
        assert callable(getattr(m, name)), name
    assert m.batch_size == 1 and m.input_size == 320
