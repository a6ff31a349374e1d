"""YOLOv3 and FCOS at class counts other than 20 (no GPU): the constructor's range check, the variables of an 80-class
network against a hand enumeration, the training executor and losses against the oracle at 80 classes, and the
checkpoint rules between class counts (a detection checkpoint of another count is refused, a backbone moves)."""
import numpy as np
import pytest
import torch

import class_count_rows as CR
from helpers import YOLO_PRIORS, model_cfg


def _model(family, nc, **over):
    import FCOS
    import YOLOv3
    cls, kind = {"yolov3": (YOLOv3.YOLOv3, "yolov3"), "fcos": (FCOS.FCOS, "fcos")}[family]
    return cls(model_cfg(kind, num_classes=nc, bn_init="trained", **over), None)


@pytest.mark.parametrize("family", ["yolov3", "fcos"])
@pytest.mark.parametrize("nc,ok", [(0, False), (1, True), (20, True), (80, True), (128, True), (129, False),
                                   (80.0, False), (True, False)])
def test_constructor_accepts_1_to_128_classes(family, nc, ok):
    if ok:
        assert _model(family, nc).num_classes == nc
        return
    with pytest.raises(ValueError, match=r"num_classes = .*1 to 128"):
        _model(family, nc)


def test_softmax_families_keep_rejecting_other_counts():
    import RetinaNet
    import SSD300
    for nc in (1, 80, 128):
        with pytest.raises(ValueError):
            SSD300.SSD300(model_cfg("ssd", num_classes=nc), None)
        with pytest.raises(ValueError):
            RetinaNet.RetinaNet(model_cfg("retinanet", num_classes=nc), None)


def test_yolov3_variables_at_80_classes():
    """Names do not change; the three pyd* prediction convs (kernel, bias, BN) output (80 + 5) * 3 = 255 channels."""
    v20 = _model("yolov3", 20).variables()
    v80 = _model("yolov3", 80).variables()
    assert list(v80) == list(v20)
    pred = {n for n, (s, _) in v20.items() if s[-1] == 75}
    assert len(pred) == 3 * 6 and all(n.startswith(("head/pyd1/", "head/pyd2/", "head/pyd3/")) for n in pred)
    for name, (shape, kind) in v80.items():
        want = v20[name][0][:-1] + (255,) if name in pred else v20[name][0]
        assert shape == want and kind == v20[name][1], (name, shape, want)
    assert {n for n, (s, _) in v80.items() if s[-1] == 255} == pred
    assert v80["head/pyd1/conv2d_6/kernel"][0] == (1, 1, 1024, 255)


def test_fcos_variables_at_80_classes():
    """Names do not change; the classifier conv (kernel and bias) outputs 80 channels."""
    v20 = _model("fcos", 20).variables()
    v80 = _model("fcos", 80).variables()
    assert list(v80) == list(v20)
    cls = {n for n, (s, _) in v20.items() if s[-1] == 20}
    assert cls == {"head/classifier_head/conv2d_4/kernel", "head/classifier_head/conv2d_4/bias"}, cls
    for name, (shape, kind) in v80.items():
        want = v20[name][0][:-1] + (80,) if name in cls else v20[name][0]
        assert shape == want and kind == v20[name][1], (name, shape, want)
    assert v80["head/classifier_head/conv2d_4/kernel"][0] == (3, 3, 256, 80)
    # one class: the classifier has one output, the centre-ness conv still one
    v1 = _model("fcos", 1).variables()
    assert v1["head/classifier_head/conv2d_4/kernel"][0] == (3, 3, 256, 1)


@pytest.mark.parametrize("family,size,nc", [("yolov3", 64, 80), ("fcos", 128, 80), ("fcos", 128, 1),
                                            ("yolov3", 64, 33)])
def test_executor_matches_oracle_forward(family, size, nc):
    """The engine's layer list replayed by train.GraphTrainer in inference mode gives the oracle's rows
    (num_classes + 5 floats each)."""
    from oracle import nets as ON
    from oracle import tails as OT
    from odt_b200.train import GraphTrainer
    m = _model(family, nc, data_shape=[size, size, 3])
    tr = GraphTrainer(m, "cpu")
    assert tr.row == nc + 5
    img = np.random.default_rng(3).integers(0, 256, (1, size, size, 3)).astype(np.float32)
    with torch.no_grad():
        rows = tr.forward_rows(img, training=False).numpy()
    w = m.get_weights()
    if family == "yolov3":
        ref = OT.yolo_rows(ON.yolov3_heads(w, img, num_classes=nc), num_classes=nc)
    else:
        ref = OT.fcos_rows(ON.fcos_heads(w, img, num_classes=nc))
    assert rows.shape == ref.shape == (1, ref.shape[1], nc + 5)
    assert np.abs(rows - ref).max() <= 2e-4 * np.abs(ref).max(), (np.abs(rows - ref).max(), np.abs(ref).max())


def _gt(rng, size, nc, B=2, G=8):
    gt = np.full((B, G, 5), -1.0, np.float32)
    for b in range(B):
        n = 3 + 2 * b
        gt[b, :n, 0:2] = rng.uniform(0.2 * size, 0.8 * size, (n, 2))
        gt[b, :n, 2:4] = rng.uniform(0.1 * size, 0.6 * size, (n, 2))
        gt[b, :n, 4] = rng.integers(0, nc, n)
    gt[0, 0, 4] = nc - 1  # the last class id
    return gt


@pytest.mark.parametrize("family,size", [("yolov3", 160), ("fcos", 256)])
def test_training_step_at_80_classes_matches_oracle_losses(family, size):
    """The autograd loss restatement of train.py at 80 classes against oracle/loss.py on the executor's own rows,
    then one Momentum step: finite loss, the classifier's variables move."""
    from oracle import loss as OL
    from oracle import tails as OT
    from odt_b200.train import GraphTrainer
    nc = 80
    over = dict(coord_scale=2, noobj_scale=0.5, obj_scale=5, class_scale=1.5) if family == "yolov3" else {}
    m = _model(family, nc, data_shape=[size, size, 3], **over)
    tr = GraphTrainer(m, "cpu")
    rng = np.random.default_rng(17)
    img = rng.integers(0, 256, (2, size, size, 3)).astype(np.float32)
    gt = _gt(rng, size, nc)
    with torch.no_grad():
        rows = tr.forward_rows(img, training=True).numpy()
    assert rows.shape[2] == nc + 5
    levels = list(tr.net.levels)
    for b in range(2):
        got = float(tr.image_loss(torch.from_numpy(rows[b]), gt[b]))
        if family == "yolov3":
            preds = CR.rows_to_levels(rows, levels, "yolo", nc)
            ref = OL.yolo_image_loss(preds, YOLO_PRIORS, gt[b], image=b, num_classes=nc, **over)
        else:
            ref = OL.fcos_image_loss(CR.rows_to_levels(rows, levels, "fcos", nc), gt[b], image=b)
        assert np.isfinite(ref) and abs(got - ref) <= 3e-5 * max(abs(ref), 1.0), (b, got, ref)
    head = ("head/pyd1/conv2d_6/kernel" if family == "yolov3" else "head/classifier_head/conv2d_4/kernel")
    before = tr.params[head].detach().clone()
    loss = tr.step(img, gt, 1e-3)
    assert np.isfinite(loss) and tr.global_step == 1
    assert not torch.equal(before, tr.params[head].detach())


def test_detection_checkpoint_of_another_class_count_is_refused(tmp_path):
    """load_weight of a 20-class checkpoint into an 80-class FCOS: CheckpointError before anything is restored."""
    from odt_b200 import tf_checkpoint
    m20 = _model("fcos", 20)
    path = m20.save_weight("latest", str(tmp_path / "fcos20"))
    m80 = _model("fcos", 80)
    w0 = {k: v.copy() for k, v in m80.get_weights().items()}
    with pytest.raises(tf_checkpoint.CheckpointError, match="another shape"):
        m80.load_weight(path)
    w1 = m80.get_weights()
    assert all(np.array_equal(w0[k], w1[k]) for k in w0), "nothing may be restored from a refused checkpoint"
    # the same count loads
    m20b = _model("fcos", 20)
    m20b.load_weight(path)
    assert all(np.array_equal(m20.get_weights()[k], m20b.get_weights()[k]) for k in m20.get_weights())


def test_backbone_moves_between_class_counts(tmp_path):
    """load_pretraining_weight: the 'backone/' variables of a 20-class model go into an 80-class model (the usual
    start of a COCO run); everything outside the backbone keeps the 80-class model's own values."""
    src = _model("fcos", 20)
    src.set_weights({k: v + np.float32(0.5) for k, v in src.get_weights().items()})
    path = src.save_weight("latest", str(tmp_path / "fcos20"))
    dst = _model("fcos", 80)
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
    assert w1["head/classifier_head/conv2d_4/kernel"].shape == (3, 3, 256, 80)
