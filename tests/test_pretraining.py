"""RetinaNet's ImageNet-pretraining mode on the CPU: constructor, variables shared with the detection model, the
pretraining checkpoint and its hand-off to detection, the ImageNet record pipeline and one training step."""
import os

import numpy as np
import pytest
import torch

from helpers import model_cfg


def _model(provider=None, **over):
    import RetinaNet
    return RetinaNet.RetinaNet(model_cfg("retinanet", is_pretraining=True, **over), provider)


SMALL = dict(data_shape=[64, 64, 3], residual_block_list=[1, 1, 1, 1], bn_init="trained")


@pytest.mark.parametrize("num_classes", [20, 1000, 3])
def test_constructor_accepts_any_num_classes(num_classes):
    m = _model(num_classes=num_classes)
    assert m.is_pretraining and m.num_logits == 224


def test_detection_still_rejects_other_class_counts():
    import RetinaNet
    with pytest.raises(ValueError, match="num_classes"):
        RetinaNet.RetinaNet(model_cfg("retinanet", num_classes=10), None)


def test_variables_are_the_detection_resnet():
    """Created first in both graphs: the pretraining variables are the detection model's first variables, name for
    name and shape for shape, all under 'feature_extractor'; the detection model adds the pyramid and the heads."""
    import RetinaNet
    pre = list(_model().variables().items())
    det = list(RetinaNet.RetinaNet(model_cfg("retinanet"), None).variables().items())
    assert len(det) > len(pre) and det[:len(pre)] == pre
    assert all(k.startswith("feature_extractor/") for k, _ in pre)
    # the last bottleneck's 1x1 expansion: 4 * 56 = 224 channels, the logit width
    assert pre[-1][0] == "feature_extractor/block4_unit3/conv_branch/conv2d_2/bias" and pre[-1][1][0] == (224,)


def test_save_weight_and_detection_handoff(tmp_path):
    import RetinaNet
    from odt_b200 import tf_checkpoint as ck
    pre = _model()
    rng = np.random.default_rng(4)
    pre.set_weights({k: rng.standard_normal(v.shape).astype(np.float32) for k, v in pre.get_weights().items()})
    pre.global_step = 7
    out = pre.save_weight("latest", str(tmp_path / "pre" / "model"))
    assert out.endswith("model-7")
    names = pre.pretraining_variables()
    r = ck.open_checkpoint(out)
    assert set(r.get_variable_to_shape_map()) == set(names)      # no moving statistics, no global_step
    assert len(names) == sum(1 for k in pre.get_weights() if not k.endswith(("moving_mean", "moving_variance")))

    det = RetinaNet.RetinaNet(model_cfg("retinanet"), None)
    w0 = {k: v.copy() for k, v in det.get_weights().items()}
    det.load_pretraining_weight(out)
    w1 = det.get_weights()
    src = pre.get_weights()
    for k in w0:
        np.testing.assert_array_equal(w1[k], src[k] if k in names else w0[k], err_msg=k)
    # a file with the whole detection backbone (pyramid convolutions included) still restores all of it
    full = {k: rng.standard_normal(v.shape).astype(np.float32) for k, v in w0.items()}
    ck.write_checkpoint(str(tmp_path / "full"), full)
    det.load_pretraining_weight(str(tmp_path / "full"))
    w2 = det.get_weights()
    for k in w0:
        np.testing.assert_array_equal(w2[k], full[k] if k in det.pretraining_variables() else w1[k], err_msg=k)
    assert len(det.pretraining_variables()) > len(names)

    # pretraining load_weight restores exactly that set and refuses a file that lacks one of it
    other = _model()
    other.load_weight(out)
    for k in names:
        np.testing.assert_array_equal(other.get_weights()[k], src[k])
    holed = str(tmp_path / "holed")
    ck.write_checkpoint(holed, {k: src[k] for k in names[1:]})
    with pytest.raises(ck.CheckpointError, match="lacks"):
        other.load_weight(holed)
    with pytest.raises(AttributeError):
        other.load_pretraining_weight(out)


def _write_jpeg_tree(root, classes, per_class, rng):
    import cv2
    for c in classes:
        os.makedirs(os.path.join(root, c))
        for i in range(per_class):
            h, w = int(rng.integers(20, 40)), int(rng.integers(20, 40))
            img = rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
            assert cv2.imwrite(os.path.join(root, c, "%d.jpg" % i), img)


def test_imagenet_records_round_trip(tmp_path):
    import cv2
    from utils import tfrecord_imagenet_utils as U
    from odt_b200 import tfrecord as TR
    rng = np.random.default_rng(0)
    classes = ["n02", "n01", "n10"]          # ids follow the sorted directory names: n01 -> 0, n02 -> 1, n10 -> 2
    _write_jpeg_tree(str(tmp_path / "img"), classes, 4, rng)
    files = U.dataset2tfrecord(str(tmp_path / "img"), str(tmp_path / "rec"), "train", total_shards=2, seed=1)
    assert [os.path.basename(f) for f in files] == ["train_00001-of-00002.tfrecord", "train_00002-of-00002.tfrecord"]
    seen = {}
    for f in files:
        for rec in TR.read_records(f):
            img, label = TR.decode_imagenet_example(rec)
            assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3
            seen.setdefault(int(label), []).append(img.shape)
    assert sorted(seen) == [0, 1, 2] and all(len(v) == 4 for v in seen.values())
    # every stored image decodes to its source file's pixels, under its directory's id
    for cid, c in enumerate(sorted(classes)):
        shapes = sorted(cv2.imread(str(tmp_path / "img" / c / ("%d.jpg" % i))).shape for i in range(4))
        assert sorted(seen[cid]) == shapes
    cfg = {"output_shape": [32, 32], "data_format": "channels_last"}
    init, it = U.get_generator(files, 5, 3, cfg)
    init()
    for _ in range(3):
        images, labels = it.get_next()
        assert images.shape == (5, 32, 32, 3) and images.dtype == np.float32
        assert labels.shape == (5,) and labels.dtype == np.int64 and set(labels.tolist()) <= {0, 1, 2}
    cfg_cf = dict(cfg, data_format="channels_first")
    init, it = U.get_generator(files, 2, 1, cfg_cf)
    assert it.get_next()[0].shape == (2, 3, 32, 32)


def test_preprocess_without_boxes_matches_the_box_path():
    from odt_b200 import tfrecord as TR
    img = np.random.default_rng(1).integers(0, 256, (30, 40, 3)).astype(np.uint8)
    cfg = {"output_shape": [24, 24], "zoom_size": [28, 28], "crop_method": "random", "flip_prob": [0.5, 0.5],
           "color_jitter_prob": 0.5, "rotate": [0.5, -5, 5]}
    gt = np.array([[5, 20, 5, 30, 1]], np.float32)
    for seed in range(4):
        alone = TR.preprocess(img, None, cfg, np.random.default_rng(seed))
        with_boxes, _ = TR.preprocess(img, gt, cfg, np.random.default_rng(seed))
        assert isinstance(alone, np.ndarray) and alone.shape == (24, 24, 3)
        np.testing.assert_array_equal(alone, with_boxes)


def _trainer(**over):
    from odt_b200.train import GraphTrainer
    m = _model(**dict(SMALL, **over))
    return m, GraphTrainer(m, "cpu")


def test_features_match_the_oracle():
    import pretraining_ref as PR
    m, tr = _trainer()
    img = np.random.default_rng(3).integers(0, 256, (2, 64, 64, 3)).astype(np.float32)
    with torch.no_grad():
        got = tr.forward_features(img, training=False).permute(0, 2, 3, 1).numpy()
    ref = PR.retinanet_features(m.get_weights(), img, SMALL["residual_block_list"])
    assert got.shape == ref.shape == (2, 2, 2, 224)
    assert np.abs(got - ref).max() <= 2e-4 * np.abs(ref).max()


def test_one_training_step():
    """loss = oracle fp32 CE + weight_decay * sum(l2_loss); from zero slots v1 = v0 - lr * dL/dv; BN moving statistics
    move 1 % towards the batch's; the step reports the training-mode accuracy."""
    import pretraining_ref as PR
    m, tr = _trainer()
    rng = np.random.default_rng(21)
    img = rng.integers(0, 256, (4, 64, 64, 3)).astype(np.float32)
    labels = rng.integers(0, 224, 4)
    lab = torch.from_numpy(labels)
    stats = []
    feats = tr.forward_features(img, True, stats)
    loss, data, logits = tr.classify_loss(feats, lab)
    ref_data = PR.sparse_softmax_xent(logits.detach().numpy(), labels).mean(dtype=np.float32)
    w = m.get_weights()
    l2 = sum(float((np.asarray(w[k], np.float64) ** 2).sum()) for k in m.pretraining_variables()) * 0.5
    ref = float(ref_data) + m.weight_decay * l2
    assert abs(float(loss) - ref) <= 1e-5 * abs(ref), (float(loss), ref)
    names = list(tr.params)
    assert sorted(names) == sorted(m.pretraining_variables())
    grads = torch.autograd.grad(loss, [tr.params[k] for k in names])
    before = {k: v.detach().clone() for k, v in tr.params.items()}
    buf0 = {k: v.clone() for k, v in tr.buffers.items()}
    l1, acc = tr.step(img, labels, 1e-3)
    assert abs(l1 - float(loss)) <= 1e-5 * abs(float(loss))
    want_acc = float(torch.eq(logits.argmax(1), lab).float().mean())
    assert acc == want_acc, (acc, want_acc)
    for k, g in zip(names, grads):
        np.testing.assert_allclose(tr.params[k].detach().numpy(), (before[k] - 1e-3 * g).numpy(), rtol=2e-5, atol=1e-7)
    scope, mean, _ = stats[0]
    np.testing.assert_allclose(tr.buffers[scope + "/moving_mean"].numpy(),
                               (0.99 * buf0[scope + "/moving_mean"] + 0.01 * mean).numpy(), rtol=1e-5, atol=1e-7)
    assert tr.global_step == 1


def test_pool_xent_gradient_matches_finite_differences():
    from odt_b200.train import pooled_xent
    rng = np.random.default_rng(8)
    f = torch.tensor(rng.standard_normal((3, 20, 3, 4)), dtype=torch.float64, requires_grad=True)
    labels = torch.tensor([0, 7, 19])
    loss, _ = pooled_xent(f, labels)
    g = torch.autograd.grad(loss, f)[0]
    e = 1e-6
    for idx in [(0, 0, 0, 0), (1, 7, 2, 3), (2, 19, 1, 1), (2, 5, 0, 2), (0, 13, 2, 0)]:
        fp, fm = f.detach().clone(), f.detach().clone()
        fp[idx] += e
        fm[idx] -= e
        fd = (float(pooled_xent(fp, labels)[0]) - float(pooled_xent(fm, labels)[0])) / (2 * e)
        assert abs(fd - float(g[idx])) <= 1e-8 + 1e-6 * abs(fd), (idx, fd, float(g[idx]))


@pytest.mark.parametrize("bad", [224, -1, 10 ** 6])
def test_out_of_range_labels_raise_before_any_launch(bad):
    m, tr = _trainer()
    img = np.zeros((2, 64, 64, 3), np.float32)
    labels = np.array([3, bad])
    with pytest.raises(ValueError, match="outside"):
        m.loss_forward(img, labels)
    with pytest.raises(ValueError, match="outside"):
        tr.step(img, labels, 1e-3)
    assert tr.global_step == 0


def test_train_one_epoch_surface(tmp_path):
    rng = np.random.default_rng(2)

    class It:
        n = 0

        def initialize(self):
            self.n = 0

        def get_next(self):
            self.n += 1
            return rng.integers(0, 256, (2, 64, 64, 3)).astype(np.float32), rng.integers(0, 224, 2)

    it = It()
    provider = {"num_train": 4, "num_val": 0, "train_generator": (it.initialize, it), "val_generator": None}
    m = _model(provider, **dict(SMALL, mode="train", batch_size=2))
    m.device = "cpu"
    k = "feature_extractor/conv2d/kernel"
    w0 = m.get_weights()[k].copy()
    loss, acc = m.train_one_epoch(1e-3)
    assert np.isfinite(loss) and 0.0 <= acc <= 1.0 and it.n == 2 and m.global_step == 2
    assert not np.array_equal(m.get_weights()[k], w0)
    assert m.save_weight("best", str(tmp_path / "m")).endswith("m-2")
