"""YOLOv2 (no GPU): the constructor's class and prior ranges, the variables against a hand enumeration of TF 1.13's names,
the training executor against the oracle network, the restated loss against the oracle's (with finite differences of
its gradient), one Momentum step, the checkpoint rules and the host-side checks of the odt_yolo2_loss_* entry points."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import BASE_CFG, YOLO_PRIORS

F32 = np.float32
PRIORS = [[1.08, 1.19], [3.42, 4.41], [6.63, 11.38], [9.42, 5.11], [16.62, 10.52]]  # testYOLOv2.py:44


def cfg(**over):
    c = dict(BASE_CFG)
    c.update(data_shape=[480, 480, 3], coord_scale=1, noobj_scale=1, obj_scale=5., class_scale=1.,
             rescore_confidence=False, priors=PRIORS, nms_max_boxes=10)
    c.update(over)
    return c


def model(**over):
    import YOLOv2
    over.setdefault("bn_init", "trained")
    return YOLOv2.YOLOv2(cfg(**over), None)


def gt_boxes(rng, size, nc, B=2, G=8, n=(6, 0)):
    """Padded GT [B, G, 5]; image b holds n[b] boxes (the second none by default)."""
    gt = np.full((B, G, 5), -1.0, F32)
    for b in range(B):
        k = n[b]
        gt[b, :k, 0:2] = rng.uniform(0.1 * size, 0.9 * size, (k, 2))
        gt[b, :k, 2:4] = np.geomspace(0.05 * size, 1.2 * size, max(k, 1))[:k, None] * rng.uniform(0.7, 1.4, (k, 2))
        gt[b, :k, 4] = rng.integers(0, nc, k)
    return gt


# ---------------------------------------------------------------------------------------------- constructor ----
@pytest.mark.parametrize("nc,A", [(1, 1), (20, 5), (128, 9)])
def test_constructor_accepts_classes_and_priors(nc, A):
    m = model(num_classes=nc, priors=PRIORS[:A] if A <= 5 else PRIORS + PRIORS[:A - 5])
    assert (m.num_classes, m.num_priors, m.name, m.loss_kind, m.backbone_scope) == (nc, A, "YOLOv2", "yolo2", "backone")
    assert m._build_spec().levels == [(15, 15, A)]


@pytest.mark.parametrize("nc", [0, 129, 20.0, True, "20", None])
def test_constructor_rejects_other_class_counts(nc):
    with pytest.raises(ValueError, match=r"num_classes = .*YOLOv2 supports 1 to 128"):
        model(num_classes=nc)


@pytest.mark.parametrize("priors", [
    [], PRIORS + PRIORS,                                     # 0 and 10 priors
    [[1.0, 2.0, 3.0]], [[1.0]], [1.0, 2.0], None, [["a", 1.0]], YOLO_PRIORS,
])
def test_constructor_rejects_malformed_priors(priors):
    with pytest.raises(ValueError, match=r"priors = .*YOLOv2 takes 1 to 9 \(h, w\) pairs"):
        model(priors=priors)


@pytest.mark.parametrize("bad", [0.0, -1.0, float("inf"), float("nan")])
def test_constructor_rejects_non_positive_priors(bad):
    with pytest.raises(ValueError, match=r"priors = .*positive finite"):
        model(priors=[[1.0, 2.0], [3.0, bad]])


# ------------------------------------------------------------------------------------------------ variables ----
def tf_names():
    """TF 1.13's variables of the reference graph, in creation order: tf.layers.conv2d(name='convN') and the unnamed
    tf.layers.batch_normalization after it, under 'backone' and 'head'."""
    out = []
    for scope, convs in (("backone", ["conv%d" % i for i in range(1, 19)]),
                         ("head", ["conv1", "conv2", "conv3", "conv4", "conv5", "predictions"])):
        for i, c in enumerate(convs):
            bn = "batch_normalization" + ("_%d" % i if i else "")
            out += ["%s/%s/kernel" % (scope, c), "%s/%s/bias" % (scope, c)]
            out += ["%s/%s/%s" % (scope, bn, v) for v in ("gamma", "beta", "moving_mean", "moving_variance")]
    return out


def test_variables_match_tf_names_and_shapes():
    v = model().variables()
    assert list(v) == tf_names()
    chans = [32, 64, 128, 64, 128, 256, 128, 256, 512, 256, 512, 256, 512, 1024, 512, 1024, 512, 1024]
    ks = [3, 3, 3, 1, 3, 3, 1, 3, 3, 1, 3, 1, 3, 3, 1, 3, 1, 3]
    cin = 3
    for i, (c, k) in enumerate(zip(chans, ks)):
        assert v["backone/conv%d/kernel" % (i + 1)][0] == (k, k, cin, c)
        cin = c
    head = [(1024, 3), (512, 1), (1024, 3), (512, 1), (1024, 3)]
    for i, (c, k) in enumerate(head):
        assert v["head/conv%d/kernel" % (i + 1)][0] == (k, k, cin, c)
        cin = c
    assert v["head/predictions/kernel"][0] == (1, 1, 1536, 125)
    assert v["head/predictions/bias"][0] == (125,)
    assert v["head/batch_normalization_5/gamma"][0] == (125,)
    assert model(num_classes=80, priors=PRIORS[:3]).variables()["head/predictions/kernel"][0] == (1, 1, 1536, 255)


# --------------------------------------------------------------------------------------------- executor / loss --
@pytest.mark.parametrize("size,nc,A", [(64, 20, 5), (80, 1, 1), (100, 128, 9)])
def test_executor_matches_oracle_network(size, nc, A):
    """train.GraphTrainer's replay of the layer list (the concat included) against oracle/yolov2.py, inference BN."""
    from odt_b200.train import GraphTrainer
    from oracle import yolov2 as OY
    pri = (PRIORS * 2)[:A]
    m = model(num_classes=nc, priors=pri, data_shape=[size, size, 3])
    tr = GraphTrainer(m, "cpu")
    img = np.random.default_rng(size).integers(0, 256, (2, size, size, 3)).astype(F32)
    with torch.no_grad():
        rows = tr.forward_rows(img, training=False).numpy()
    ref = OY.yolo2_rows(OY.yolov2_heads(m.get_weights(), img), nc)
    g = -(-size // 32)
    assert rows.shape == ref.shape == (2, g * g * A, nc + 5)
    assert np.abs(rows - ref).max() <= 2e-4 * np.abs(ref).max(), (np.abs(rows - ref).max(), np.abs(ref).max())


def _rows(h, w, A, nc, seed):
    rng = np.random.default_rng(seed)
    r = (rng.standard_normal((2, h * w * A, nc + 5)) * 1.5).astype(F32)
    r[..., nc:] = (rng.standard_normal((2, h * w * A, 5)) * 0.5).astype(F32)
    return r


def _edge_gt(nc):
    """A GT on a cell border, three in one cell (two of them on one row), one past the grid (clamped), one matched to
    the last prior."""
    gt = np.full((2, 8, 5), -1.0, F32)
    gt[0, :7] = [[64.0, 96.0, 40.0, 30.0, 0], [70.0, 70.0, 20.0, 60.0, nc - 1], [75.0, 72.0, 300.0, 250.0, 1 % nc],
                 [480.0, 10.0, 50.0, 50.0, 2 % nc], [200.0, 300.0, 520.0, 340.0, 0], [71.0, 69.0, 22.0, 58.0, 0],
                 [250.0, 250.0, 30.0, 30.0, 0]]
    return gt


@pytest.mark.parametrize("nc,A", [(20, 5), (3, 1), (80, 9)])
def test_restated_loss_matches_oracle(nc, A):
    """train.yolo2_image_loss on rows against oracle/yolov2.py's numpy fp32 loss, an image without boxes included."""
    from odt_b200.train import GraphTrainer
    from oracle import yolov2 as OY
    pri = (PRIORS * 2)[:A]
    over = dict(coord_scale=2, noobj_scale=0.5, obj_scale=5, class_scale=1.5)
    m = model(num_classes=nc, priors=pri, **over)
    tr = GraphTrainer(m, "cpu")
    rows = _rows(15, 15, A, nc, nc)
    for gt in (gt_boxes(np.random.default_rng(A), 480, nc), _edge_gt(nc)):
        for b in range(2):
            got = float(tr.image_loss(torch.from_numpy(rows[b]), gt[b]))
            want = OY.yolo2_image_loss(rows.reshape(2, 15, 15, -1), pri, gt[b], image=b, num_classes=nc, **over)
            assert np.isfinite(want) and abs(got - want) <= 3e-5 * max(abs(want), 1.0), (b, got, want)
    # no boxes: only the no-object term, over every row
    empty = np.full((8, 5), -1.0, F32)
    r = torch.from_numpy(rows[0])
    want = 0.5 * float(torch.nn.functional.softplus(r[:, nc + 4]).sum())
    assert abs(float(tr.image_loss(r, empty)) - want) <= 1e-5 * want


def test_loss_gradient_matches_finite_differences():
    """d yolo2_image_loss / d rows by autograd against central differences of the oracle's loss: positive rows (a
    match on the last prior among them) and no-object rows."""
    from odt_b200.train import GraphTrainer
    from oracle import yolov2 as OY
    A, nc = 5, 20
    over = dict(coord_scale=2, noobj_scale=0.5, obj_scale=5, class_scale=1.5)
    tr = GraphTrainer(model(**over), "cpu")
    rows = _rows(15, 15, A, nc, 7)
    gt = _edge_gt(nc)[0]

    def ref(r):
        return OY.yolo2_image_loss(r.reshape(1, 15, 15, -1), PRIORS, gt, num_classes=nc, **over)

    r0 = torch.from_numpy(rows[0].copy()).requires_grad_(True)
    tr.image_loss(r0, gt).backward()
    grad = r0.grad.numpy()
    pos = sorted(set(np.nonzero(np.abs(grad[:, :nc]).sum(-1))[0]))
    assert len(pos) == 6 and any(n % A == A - 1 for n in pos), pos  # 7 GTs, two on one row
    noobj = [n for n in np.nonzero(grad[:, nc + 4])[0] if n not in pos][:4]
    entries = [(n, c) for n in pos for c in (0, nc, nc + 2, nc + 4)] + [(n, nc + 4) for n in noobj]
    eps = 1e-2
    for n, c in entries:
        up, dn = rows[:1].copy(), rows[:1].copy()
        up[0, n, c] += F32(eps)
        dn[0, n, c] -= F32(eps)
        fd = (ref(up) - ref(dn)) / (float(up[0, n, c]) - float(dn[0, n, c]))
        assert abs(fd - grad[n, c]) <= 1e-3 * max(abs(grad[n, c]), 0.05), (n, c, fd, grad[n, c])


def test_one_step_is_momentum_on_the_restated_loss():
    """tr.step = v - lr * (dL/dv) on the first step (Momentum slots start at zero), L = batch mean of the image losses
    (no 0.5) + weight_decay * sum(l2_loss); the BN moving statistics move 1% toward the batch moments."""
    from odt_b200.train import GraphTrainer
    size = 64
    m = model(data_shape=[size, size, 3])
    tr = GraphTrainer(m, "cpu")
    ref = GraphTrainer(m, "cpu")
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (2, size, size, 3)).astype(F32)
    gt = gt_boxes(rng, size, 20, n=(3, 0))
    stats = []
    rows = ref.forward_rows(img, True, stats)
    data = (ref.image_loss(rows[0], gt[0]) + ref.image_loss(rows[1], gt[1])) / 2
    l2 = sum((p * p).sum() for p in ref.params.values()) * 0.5
    loss = data + float(m.weight_decay) * l2
    names = list(ref.params)
    grads = torch.autograd.grad(loss, [ref.params[k] for k in names])
    lr = 1e-3
    got = tr.step(img, gt, lr)
    assert abs(got - float(loss.detach())) <= 1e-5 * abs(float(loss.detach()))
    for k, g in zip(names, grads):
        want = ref.params[k].detach() - lr * g
        assert torch.allclose(tr.params[k].detach(), want, rtol=1e-5, atol=1e-7), k
    scope, mean, var = stats[0]
    mm = m.get_weights()[scope + "/moving_mean"]
    assert torch.allclose(tr.buffers[scope + "/moving_mean"], torch.from_numpy(mm * 0.99) + 0.01 * mean, atol=1e-6)
    assert tr.global_step == 1


# ------------------------------------------------------------------------------------------------ checkpoints ---
def test_checkpoint_round_trip(tmp_path):
    src = model()
    src.set_weights({k: v + np.float32(0.25) for k, v in src.get_weights().items()})
    src.global_step = 7
    path = src.save_weight("latest", str(tmp_path / "yolo2" / "test"))
    assert path.endswith("test-7")
    dst = model()
    dst.load_weight(path)
    assert dst.global_step == 7
    assert all(np.array_equal(src.get_weights()[k], dst.get_weights()[k]) for k in src.get_weights())


@pytest.mark.parametrize("other", [dict(num_classes=80), dict(priors=PRIORS[:3]), "yolov3"])
def test_checkpoint_of_another_model_is_refused(tmp_path, other):
    """load_weight of a checkpoint of another class count, prior count, or of YOLOv3 (whose 'backone/' has other
    names): CheckpointError before anything is restored."""
    from odt_b200 import tf_checkpoint
    from helpers import model_cfg
    if other == "yolov3":
        import YOLOv3
        src = YOLOv3.YOLOv3(model_cfg("yolov3"), None)
    else:
        src = model(**other)
    path = src.save_weight("latest", str(tmp_path / "other"))
    dst = model()
    w0 = {k: v.copy() for k, v in dst.get_weights().items()}
    with pytest.raises(tf_checkpoint.CheckpointError):
        dst.load_weight(path)
    if other == "yolov3":
        with pytest.raises(tf_checkpoint.CheckpointError):
            dst.load_pretraining_weight(path)
    w1 = dst.get_weights()
    assert all(np.array_equal(w0[k], w1[k]) for k in w0), "nothing may be restored from a refused checkpoint"


def test_backbone_moves_between_class_and_prior_counts(tmp_path):
    """load_pretraining_weight restores the trainable 'backone/' variables only (no moving statistics), across
    class and prior counts."""
    src = model(num_classes=80, priors=PRIORS[:2])
    src.set_weights({k: v + np.float32(0.5) for k, v in src.get_weights().items()})
    path = src.save_weight("latest", str(tmp_path / "src"))
    dst = model()
    w0 = {k: v.copy() for k, v in dst.get_weights().items()}
    dst.load_pretraining_weight(path)
    names = dst.pretraining_variables()
    assert len(names) == 18 * 4 and all(n.startswith("backone/") for n in names)
    w1, ws = dst.get_weights(), src.get_weights()
    for k in w1:
        assert np.array_equal(w1[k], ws[k] if k in names else w0[k]), k


# ----------------------------------------------------------------------------------------- C argument checks ----
def test_yolo2_loss_entry_points_check_on_the_host(built):
    """odt_yolo2_loss_{fwd,grad} refuse, before any launch: bad B or G, another decode kind, num_levels != 1, A outside
    1..9, a level geometry that is not H * W * A rows, unaligned scratch, a null gradient.  The scratch size counts
    one occupancy byte per cell."""
    from odt_b200 import lib
    L = lib.load()
    fake = ctypes.c_void_p(64)  # never dereferenced: every call below is rejected first

    def params(A=5, H=15, W=15, levels=1, kind=lib.DECODE_YOLO3, nc=20):
        p = lib.TailParams()
        p.kind, p.num_levels, p.num_fg = kind, levels, nc
        off = 0
        for i in range(levels):
            p.level[i].H, p.level[i].W, p.level[i].A, p.level[i].offset = H, W, A, off
            off += H * W * A
        p.N = off
        return p

    def refused(p, B=1, G=4, scratch=fake, what=b"invalid argument"):
        ok = []
        for grad in (False, True):
            if grad:
                rc = L.odt_yolo2_loss_grad(fake, ctypes.byref(p), B, fake, G, 1.0, 1.0, 5.0, 1.0, scratch, fake, fake,
                                           None)
            else:
                rc = L.odt_yolo2_loss_fwd(fake, ctypes.byref(p), B, fake, G, 1.0, 1.0, 5.0, 1.0, scratch, fake, None)
            ok.append(rc == -1 and what in L.odt_last_error())
        return all(ok)

    for A in (1, 5, 9):
        assert refused(params(A), G=0, what=b"B/G"), A  # the geometry passes: the GT count is what fails
    assert refused(params(), B=0, what=b"B/G")
    assert refused(params(), G=129, what=b"B/G")
    assert refused(params(), scratch=ctypes.c_void_p(68), what=b"aligned")
    assert refused(params(kind=lib.DECODE_FCOS), what=b"YOLOv2 head")
    assert refused(params(levels=3), what=b"YOLOv2 head")
    assert refused(params(nc=0), what=b"YOLOv2 head")
    assert refused(params(nc=129), what=b"YOLOv2 head")
    for A in (0, 10):
        assert refused(params(A)), A
    p = params()
    p.N += 1
    assert refused(p)
    rc = L.odt_yolo2_loss_grad(fake, ctypes.byref(params()), 1, fake, 4, 1.0, 1.0, 5.0, 1.0, fake, fake, None, None)
    assert rc == -1 and b"null" in L.odt_last_error()
    n = L.odt_yolo2_loss_scratch_bytes(ctypes.byref(params()), 2)
    assert n == 2 * 4 * 4 + 2 * 64 * 4 + ((2 * 225 + 7) & ~7)
    # the YOLOv3 entry point keeps refusing one level
    rc = L.odt_yolo_loss_fwd(fake, ctypes.byref(params()), 1, fake, 4, 1.0, 1.0, 5.0, 1.0, fake, fake, None)
    assert rc == -1 and b"YOLOv3 head" in L.odt_last_error()


def test_driver_config_constructs_and_exposes_the_reference_surface():
    """testYOLOv2.py's config (mode 'train' with a provider): the attributes and methods its loop uses."""
    import YOLOv2 as yolov2
    c = cfg(mode="train", batch_size=32, is_pretraining=False)
    provider = {"data_shape": [480, 480, 3], "num_train": 64, "num_val": 0, "train_generator": (lambda: None, None),
                "val_generator": None}
    m = yolov2.YOLOv2(c, provider)
    assert m.num_priors == 5 and m.batch_size == 32 and m.rescore_confidence is False
    for name in ("train_one_epoch", "test_one_image", "save_weight", "load_weight", "load_pretraining_weight"):
        assert callable(getattr(m, name))
