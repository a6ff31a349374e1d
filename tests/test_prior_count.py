"""YOLOv3 with 1 to 9 priors per level (no GPU): the constructor's range check, the variables at 5 priors and 80 classes
against a hand enumeration, the any-A restatement against the oracle at 3 priors, the training executor and its loss
against the restatement (with finite differences), and the checkpoint rules between prior counts."""
import numpy as np
import pytest
import torch

import class_count_rows as CR
import prior_count_ref as PR
from helpers import YOLO_PRIORS, model_cfg

F32 = np.float32


def _model(A, nc=20, priors=None, **over):
    import YOLOv3
    return YOLOv3.YOLOv3(model_cfg("yolov3", num_classes=nc, num_priors=A,
                                   priors=PR.priors_for(A) if priors is None else priors, bn_init="trained", **over),
                         None)


@pytest.mark.parametrize("A", [1, 2, 3, 5, 9])
def test_constructor_accepts_1_to_9_priors(A):
    m = _model(A)
    assert m.num_priors == A
    assert [a for _, _, a in m._build_spec().levels] == [A, A, A]


@pytest.mark.parametrize("A", [0, 10, 3.0, True, -1, "3", None])
def test_constructor_rejects_other_prior_counts(A):
    with pytest.raises(ValueError, match=r"num_priors = .*1 to 9"):
        _model(A, priors=YOLO_PRIORS)


@pytest.mark.parametrize("A,priors", [
    (3, [YOLO_PRIORS[0], YOLO_PRIORS[1], YOLO_PRIORS[2][:2]]),               # a level one pair short
    (2, YOLO_PRIORS),                                                       # three pairs where two are configured
    (3, [YOLO_PRIORS[0], [[30, 61]], YOLO_PRIORS[2]]),                       # TF would broadcast one pair; not here
    (3, YOLO_PRIORS[:2]),                                                   # two levels
    (3, [YOLO_PRIORS[0], YOLO_PRIORS[1], [[116, 90], [156, 0], [373, 326]]]),  # a zero size
    (3, [YOLO_PRIORS[0], YOLO_PRIORS[1], [[116, 90], [156, -4], [373, 326]]]),
    (3, [YOLO_PRIORS[0], YOLO_PRIORS[1], [[116, 90], [156, float("inf")], [373, 326]]]),
    (3, [YOLO_PRIORS[0], YOLO_PRIORS[1], [[116, 90], [156, float("nan")], [373, 326]]]),
    (1, [[[10, 13, 5]], [[30, 61]], [[116, 90]]]),                          # not a pair
    (1, [[["a", 13]], [[30, 61]], [[116, 90]]]),
    (1, None),
])
def test_constructor_rejects_malformed_priors(A, priors):
    import YOLOv3
    with pytest.raises(ValueError, match=r"priors.*num_priors = %d" % A):
        YOLOv3.YOLOv3(model_cfg("yolov3", num_priors=A, priors=priors), None)


def test_yolov3_variables_at_5_priors_80_classes():
    """Names do not change; the three pyd* prediction convs (kernel, bias, BN) output (80 + 5) * 5 = 425 channels,
    every other variable keeps the shape it has at 3 priors and 20 classes."""
    v3 = _model(3, priors=YOLO_PRIORS).variables()
    v5 = _model(5, 80).variables()
    assert list(v5) == list(v3)
    # pyd2 / pyd3 create the upsampling 1x1 conv first, so their prediction conv is the eighth of the scope
    scopes = (("pyd1", 6), ("pyd2", 7), ("pyd3", 7))
    pred = {"head/%s/conv2d_%d/%s" % (s, i, v) for s, i in scopes for v in ("kernel", "bias")}
    pred |= {"head/%s/batch_normalization_%d/%s" % (s, i, v) for s, i in scopes
             for v in ("gamma", "beta", "moving_mean", "moving_variance")}
    assert {n for n, (s, _) in v3.items() if s[-1] == 75} == pred
    for name, (shape, kind) in v5.items():
        want = v3[name][0][:-1] + (425,) if name in pred else v3[name][0]
        assert shape == want and kind == v3[name][1], (name, shape, want)
    assert v5["head/pyd1/conv2d_6/kernel"][0] == (1, 1, 1024, 425)
    assert v5["head/pyd2/conv2d_7/kernel"][0] == (1, 1, 256, 425)
    assert v5["head/pyd3/conv2d_7/kernel"][0] == (1, 1, 128, 425)


def _rows(levels, nc, B, seed):
    rng = np.random.default_rng(seed)
    N = sum(h * w * a for h, w, a in levels)
    r = (rng.standard_normal((B, N, nc + 5)) * 1.5).astype(F32)
    r[..., nc:] = (rng.standard_normal((B, N, 5)) * 0.5).astype(F32)
    return r


def _gt(rng, size, nc, B=2, G=14):
    """GT boxes of every size from a few pixels to three times the image: the level-0 priors are compared with the GT
    divided by 32 (YOLOv3.py:435-442), so only boxes larger than a 160² image reach the last of 9 priors there."""
    gt = np.full((B, G, 5), -1.0, F32)
    for b in range(B):
        n = 12 - 2 * b  # padded: the GT count is the index of the first -1 row
        gt[b, :n, 0:2] = rng.uniform(0.15 * size, 0.85 * size, (n, 2))
        gt[b, :n, 2:4] = np.geomspace(0.04 * size, 3.0 * size, n)[:, None] * rng.uniform(0.7, 1.4, (n, 2))
        gt[b, :n, 4] = rng.integers(0, nc, n)
    gt[0, 0, 4] = nc - 1
    return gt


@pytest.mark.parametrize("nc", [20, 80])
def test_restatement_equals_oracle_at_3_priors(nc):
    """At 3 priors the any-A restatement of prior_count_ref is the oracle, bit for bit: scores, boxes, detections and
    losses."""
    from oracle import loss as OL
    from oracle import tails as OT
    levels = [(5, 5, 3), (10, 10, 3), (20, 20, 3)]
    rows = _rows(levels, nc, 2, seed=nc)
    preds = CR.rows_to_levels(rows, levels, "yolo", nc)
    gt = _gt(np.random.default_rng(nc), 160, nc)
    for b in range(2):
        c0, b0 = OT.yolo_scores_boxes(preds, YOLO_PRIORS, image=b, num_classes=nc)
        c1, b1 = PR.yolo_scores_boxes(preds, YOLO_PRIORS, image=b, num_classes=nc)
        assert np.array_equal(c0, c1) and np.array_equal(b0, b1)
        for x, y in zip(OT.yolo_detect(preds, YOLO_PRIORS, 0.3, 10, 0.45, image=b, num_classes=nc),
                        PR.yolo_detect(preds, YOLO_PRIORS, 0.3, 10, 0.45, image=b, num_classes=nc)):
            assert np.array_equal(x, y)
        kw = dict(coord_scale=2, noobj_scale=0.5, obj_scale=5, class_scale=1.5)
        assert OL.yolo_image_loss(preds, YOLO_PRIORS, gt[b], image=b, num_classes=nc, **kw) == \
            PR.yolo_image_loss(preds, YOLO_PRIORS, gt[b], image=b, num_classes=nc, **kw)


@pytest.mark.parametrize("A", [1, 2, 5, 9])
def test_ground_truth_reaches_every_prior(A):
    """The GT sets of these tests (and of the GPU ones) are matched to the last prior of some level, so the row index
    cell * A + (A - 1) is exercised."""
    for size in (160, 416):
        gt = _gt(np.random.default_rng(A), size, 20)
        got = {p for b in range(2) for _, p in PR.assignment(PR.priors_for(A), gt[b])}
        assert A - 1 in got, (size, got)


@pytest.mark.parametrize("A,nc", [(1, 1), (5, 80), (9, 20)])
def test_executor_matches_restated_forward(A, nc):
    """The engine's layer list replayed by train.GraphTrainer gives the oracle network's rows at A priors
    (oracle/nets.py::yolov3_heads takes num_priors), and their scores and boxes through the restatement equal those of
    the same rows read level by level."""
    from oracle import nets as ON
    from oracle import tails as OT
    from odt_b200.train import GraphTrainer
    size = 64
    m = _model(A, nc, data_shape=[size, size, 3])
    tr = GraphTrainer(m, "cpu")
    img = np.random.default_rng(3).integers(0, 256, (1, size, size, 3)).astype(F32)
    with torch.no_grad():
        rows = tr.forward_rows(img, training=False).numpy()
    heads = ON.yolov3_heads(m.get_weights(), img, num_classes=nc, num_priors=A)
    assert [h.shape[3] for h in heads] == [(nc + 5) * A] * 3
    ref = OT.yolo_rows(heads, num_classes=nc)
    N = sum(h * w * A for h, w in ((2, 2), (4, 4), (8, 8)))
    assert rows.shape == ref.shape == (1, N, nc + 5)
    assert np.abs(rows - ref).max() <= 2e-4 * np.abs(ref).max(), (np.abs(rows - ref).max(), np.abs(ref).max())
    # the executor's rows cut back into levels are the oracle's head tensors
    levels = list(tr.net.levels)
    assert levels == [(2, 2, A), (4, 4, A), (8, 8, A)]
    for got, want in zip(CR.rows_to_levels(ref, levels, "yolo", nc), heads):
        assert np.array_equal(got, want)
    conf, box = PR.yolo_scores_boxes(heads, m.config["priors"], num_classes=nc)
    assert conf.shape == (N, nc) and box.shape == (N, 4) and np.isfinite(conf).all()


def test_training_step_at_5_priors_matches_restated_loss():
    """At A = 5: the autograd loss of train.py against the restated loss on the executor's own rows, its gradient
    with respect to the rows against central finite differences of the restated loss (the positive rows, the last
    prior's included, and no-object rows), then one Momentum step."""
    from odt_b200.train import GraphTrainer
    A, nc, size = 5, 20, 160
    over = dict(coord_scale=2, noobj_scale=0.5, obj_scale=5, class_scale=1.5)
    m = _model(A, nc, data_shape=[size, size, 3], **over)
    tr = GraphTrainer(m, "cpu")
    priors = m.config["priors"]
    rng = np.random.default_rng(17)
    img = rng.integers(0, 256, (2, size, size, 3)).astype(F32)
    gt = _gt(rng, size, nc)
    with torch.no_grad():
        rows = tr.forward_rows(img, training=True).numpy()
    levels = list(tr.net.levels)
    assert rows.shape == (2, sum(h * w * A for h, w, _ in levels), nc + 5)

    def ref(r, b):
        return PR.yolo_image_loss(CR.rows_to_levels(r, levels, "yolo", nc), priors, gt[b], image=b, num_classes=nc,
                                  **over)

    for b in range(2):
        got = float(tr.image_loss(torch.from_numpy(rows[b]), gt[b]))
        want = ref(rows, b)
        assert np.isfinite(want) and abs(got - want) <= 3e-5 * max(abs(want), 1.0), (b, got, want)

    # gradient of image 0's loss: the rows the kernels and the restatement address as cell * A + prior
    r0 = torch.from_numpy(rows[0].copy()).requires_grad_(True)
    tr.image_loss(r0, gt[0]).backward()
    grad = r0.grad.numpy()
    offs = np.cumsum([0] + [h * w * A for h, w, _ in levels])
    pos = []
    for (k, a), g in zip(PR.assignment(priors, gt[0]), gt[0]):
        h, w, _ = levels[k]
        norm = [32.0, 16.0, 8.0][k]
        y = min(max(int(np.floor(g[0] / norm)), 0), h - 1)
        x = min(max(int(np.floor(g[1] / norm)), 0), w - 1)
        pos.append((offs[k] + (y * w + x) * A + a, a))
    assert any(a == A - 1 for _, a in pos), pos
    assert set(np.nonzero(np.abs(grad[:, :nc]).sum(-1))[0]) == {n for n, _ in pos}  # class terms: positives only
    noobj = [n for n in np.nonzero(grad[:, nc + 4])[0] if n not in {p for p, _ in pos}][:4]
    assert len(noobj) == 4
    entries = [(n, c) for n, _ in pos[:4] for c in (0, nc, nc + 2, nc + 4)] + [(n, nc + 4) for n in noobj]
    eps = 1e-2
    for n, c in entries:
        up, dn = rows.copy(), rows.copy()
        up[0, n, c] += F32(eps)
        dn[0, n, c] -= F32(eps)
        fd = (ref(up, 0) - ref(dn, 0)) / (float(up[0, n, c]) - float(dn[0, n, c]))
        assert abs(fd - grad[n, c]) <= 1e-3 * max(abs(grad[n, c]), 0.05), (n, c, fd, grad[n, c])

    head = "head/pyd1/conv2d_6/kernel"
    before = tr.params[head].detach().clone()
    loss = tr.step(img, gt, 1e-3)
    assert np.isfinite(loss) and tr.global_step == 1
    assert not torch.equal(before, tr.params[head].detach())


def test_detection_checkpoint_of_another_prior_count_is_refused(tmp_path):
    """load_weight of a 3-prior checkpoint into a 5-prior YOLOv3: CheckpointError before anything is restored."""
    from odt_b200 import tf_checkpoint
    m3 = _model(3, priors=YOLO_PRIORS)
    path = m3.save_weight("latest", str(tmp_path / "yolo3"))
    m5 = _model(5)
    w0 = {k: v.copy() for k, v in m5.get_weights().items()}
    with pytest.raises(tf_checkpoint.CheckpointError, match="another shape"):
        m5.load_weight(path)
    w1 = m5.get_weights()
    assert all(np.array_equal(w0[k], w1[k]) for k in w0), "nothing may be restored from a refused checkpoint"
    m3b = _model(3, priors=YOLO_PRIORS)
    m3b.load_weight(path)
    assert all(np.array_equal(m3.get_weights()[k], m3b.get_weights()[k]) for k in m3.get_weights())


def test_backbone_moves_between_prior_counts(tmp_path):
    """load_pretraining_weight: the 'backone/' variables of a 3-prior model go into a 9-prior model; everything outside
    the backbone keeps the 9-prior model's own values."""
    src = _model(3, priors=YOLO_PRIORS)
    src.set_weights({k: v + np.float32(0.5) for k, v in src.get_weights().items()})
    path = src.save_weight("latest", str(tmp_path / "yolo3"))
    dst = _model(9)
    w0 = {k: v.copy() for k, v in dst.get_weights().items()}
    dst.load_pretraining_weight(path)
    w1, ws = dst.get_weights(), src.get_weights()
    names = dst.pretraining_variables()
    assert names and all(n.startswith("backone/") for n in names)
    for k in w1:
        if k in names:
            assert np.array_equal(w1[k], ws[k]), k
        else:
            assert np.array_equal(w1[k], w0[k]), k
    assert w1["head/pyd1/conv2d_6/kernel"].shape == (1, 1, 1024, 225)


def test_yolo_loss_accepts_any_prior_count_and_checks_the_geometry(built):
    """odt_yolo_loss_fwd takes 1 to 9 priors, the same on every level, and rows laid out level after level
    (offset = rows before the level, N = sum of H * W * A); everything else is refused on the host, before any launch.
    The scratch size counts one occupancy byte per cell."""
    import ctypes
    from odt_b200 import lib
    L = lib.load()
    fake = ctypes.c_void_p(64)  # never dereferenced: every call below is rejected first

    def params(A, hw=((2, 3), (4, 5), (6, 7))):
        p = lib.TailParams()
        p.kind, p.num_levels, p.num_fg = lib.DECODE_YOLO3, 3, 20
        off = 0
        for i, (h, w) in enumerate(hw):
            p.level[i].H, p.level[i].W, p.level[i].A, p.level[i].offset = h, w, A, off
            off += h * w * A
        p.N = off
        return p

    def fwd(p, G=4):
        rc = L.odt_yolo_loss_fwd(fake, ctypes.byref(p), 1, fake, G, 1.0, 1.0, 5.0, 1.0, fake, fake, None)
        return rc == -1 and b"invalid argument" in L.odt_last_error()

    cells = 2 * 3 + 4 * 5 + 6 * 7
    base = L.odt_yolo_loss_scratch_bytes(ctypes.byref(params(3)), 2)
    for A in (1, 2, 5, 9):
        p = params(A)
        assert fwd(p, G=0) and b"B/G" in L.odt_last_error(), A  # the geometry passes: the GT count is what fails
        assert L.odt_yolo_loss_scratch_bytes(ctypes.byref(p), 2) == base  # one byte per cell, whatever A
    assert base == 2 * 4 * 4 + 2 * 64 * 4 + ((2 * cells + 7) & ~7)
    for A in (0, 10):
        assert fwd(params(A)), A
    p = params(3)
    p.level[2].A = 2
    assert fwd(p), "priors differ between levels"
    p = params(3)
    p.N += 1
    assert fwd(p), "N is not the sum of the levels"
    p = params(3)
    p.level[1].offset += 3
    assert fwd(p), "a level's offset"
    p = params(3, ((2, 3), (0, 5), (6, 7)))
    assert fwd(p), "an empty level"
