"""RetinaNet's basic-block ResNet (`is_bottleneck=False`, RetinaNet.py:272-275,621-632) on the CPU: variable names,
the configuration checks, the layer-list executor against the oracle, one training step in each mode, the detection
loss gradient, and the pretraining -> detection checkpoint hand-off with cross-variant loads refused."""
import numpy as np
import pytest
import torch

import basic_block_ref as BR
from helpers import model_cfg

BLOCKS = {"2222": [2, 2, 2, 2], "3463": [3, 4, 6, 3]}


def _model(blocks, provider=None, **over):
    import RetinaNet
    cfg = dict(dict(is_bottleneck=False, init_conv_filters=7, residual_block_list=BLOCKS[blocks]), **over)
    return RetinaNet.RetinaNet(model_cfg("retinanet", **cfg), provider)


def _trainer(m, dtype=torch.float32):
    from odt_b200.train import GraphTrainer
    return GraphTrainer(m, "cpu", dtype)


def _gt(B, size, seed):
    rng = np.random.default_rng(seed)
    gt = np.full((B, 6, 5), -1.0, np.float32)
    for b in range(B):
        n = 2 + b
        gt[b, :n, 0:2] = rng.uniform(0.25 * size, 0.75 * size, (n, 2))
        gt[b, :n, 2:4] = rng.uniform(0.2 * size, 0.6 * size, (n, 2))
        gt[b, :n, 4] = rng.integers(0, 20, n)
    return gt


@pytest.mark.parametrize("pretraining", [False, True])
@pytest.mark.parametrize("blocks", sorted(BLOCKS))
def test_variable_names_and_shapes(blocks, pretraining):
    m = _model(blocks, is_pretraining=pretraining)
    got = {k: shape for k, (shape, _) in m.variables().items()}
    want = BR.tf_variables(BLOCKS[blocks], detection=not pretraining)
    assert got == want, (sorted(set(got) ^ set(want))[:6])
    assert "feature_extractor/block2_unit1/conv_branch/conv2d_1/kernel" in got
    assert "feature_extractor/block2_unit1/identity_branch/batch_normalization/gamma" in got
    # stride-1 units create no identity_branch variables; every stride-2 unit does
    for k in got:
        if "/identity_branch/" in k:
            assert "_unit1/" in k and "/block1_" not in k, k
    n_stride2 = len(BLOCKS[blocks]) - 1
    assert sum(1 for k in got if k.endswith("identity_branch/conv2d/kernel")) == n_stride2


def test_pretraining_variables_are_the_detection_resnet():
    pre = list(_model("3463", is_pretraining=True).variables().items())
    det = list(_model("3463").variables().items())
    assert len(det) > len(pre) and det[:len(pre)] == pre
    assert pre[-1][0] == "feature_extractor/block4_unit3/conv_branch/conv2d_1/bias" and pre[-1][1][0] == (56,)


@pytest.mark.parametrize("pretraining", [False, True])
@pytest.mark.parametrize("filters", [16, 1, 3])
def test_init_conv_filters_other_than_7_are_rejected(filters, pretraining):
    with pytest.raises(ValueError, match=r"init_conv_filters = %d\b.*must be 7" % filters):
        _model("2222", init_conv_filters=filters, is_pretraining=pretraining)


def test_num_logits():
    assert _model("3463", is_pretraining=True).num_logits == 56
    assert _model("2222", is_pretraining=True).num_logits == 56
    assert _model("2222", is_pretraining=True, residual_block_list=[2, 2, 2]).num_logits == 28
    import RetinaNet
    assert RetinaNet.RetinaNet(model_cfg("retinanet", is_pretraining=True), None).num_logits == 224


def test_bottleneck_variant_is_unchanged():
    """The bottleneck builder keeps its op list and names; init_conv_filters stays free there."""
    import RetinaNet
    m = RetinaNet.RetinaNet(model_cfg("retinanet", init_conv_filters=32), None)
    names = list(m.variables())
    assert "feature_extractor/block1_unit1/identity_branch/conv2d/kernel" in names
    assert "feature_extractor/block4_unit3/conv_branch/conv2d_2/kernel" in names


@pytest.mark.parametrize("blocks", sorted(BLOCKS))
def test_executor_matches_the_oracle(blocks):
    """Inference-mode replay of the layer list (GraphTrainer, BN on the moving statistics) against the oracle's
    restatement: detection rows and pretraining features within 2e-4 x max|ref|."""
    img = np.random.default_rng(3).integers(0, 256, (2, 64, 64, 3)).astype(np.float32)
    det = _model(blocks, data_shape=[64, 64, 3], bn_init="trained")
    with torch.no_grad():
        got = _trainer(det).forward_rows(img, training=False).numpy()
    ref = BR.rows(det.get_weights(), img, BLOCKS[blocks])
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 2e-4 * np.abs(ref).max()
    pre = _model(blocks, data_shape=[64, 64, 3], bn_init="trained", is_pretraining=True)
    with torch.no_grad():
        f = _trainer(pre).forward_features(img, training=False).permute(0, 2, 3, 1).numpy()
    fr = BR.features(pre.get_weights(), img, BLOCKS[blocks])
    assert f.shape == fr.shape == (2, 2, 2, 56)
    assert np.abs(f - fr).max() <= 2e-4 * np.abs(fr).max()


def _check_step(m, tr, step_args, loss, stats):
    """From zero slots: v1 = v0 - lr * dL/dv for every trainable variable; moving = 0.99 * moving + 0.01 * batch."""
    names = list(tr.params)
    grads = torch.autograd.grad(loss, [tr.params[k] for k in names], allow_unused=True)
    before = {k: v.detach().clone() for k, v in tr.params.items()}
    buf0 = {k: v.clone() for k, v in tr.buffers.items()}
    out = tr.step(*step_args, 1e-3)
    l1 = out[0] if isinstance(out, tuple) else out
    assert abs(l1 - float(loss)) <= 1e-5 * abs(float(loss))
    for k, g in zip(names, grads):
        assert g is not None, k
        np.testing.assert_allclose(tr.params[k].detach().numpy(), (before[k] - 1e-3 * g).numpy(), rtol=2e-5,
                                   atol=1e-7, err_msg=k)
    assert len(stats) == sum(1 for k in tr.buffers if k.endswith("moving_mean"))
    for scope, mean, var in stats:
        np.testing.assert_allclose(tr.buffers[scope + "/moving_mean"].numpy(),
                                   (0.99 * buf0[scope + "/moving_mean"] + 0.01 * mean).numpy(), rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(tr.buffers[scope + "/moving_variance"].numpy(),
                                   (0.99 * buf0[scope + "/moving_variance"] + 0.01 * var).numpy(), rtol=1e-5,
                                   atol=1e-7)
    assert tr.global_step == 1
    return out


def test_one_detection_training_step():
    m = _model("2222", data_shape=[64, 64, 3], bn_init="trained")
    tr = _trainer(m)
    img = np.random.default_rng(5).integers(0, 256, (2, 64, 64, 3)).astype(np.float32)
    gt = _gt(2, 64, 6)
    stats = []
    loss, data = tr.total_loss(tr.forward_rows(img, True, stats), gt)
    w = m.get_weights()
    l2 = sum(float((np.asarray(w[k], np.float64) ** 2).sum()) for k in tr.params) * 0.5
    lv = float(loss.detach())
    assert abs(lv - (float(data.detach()) + m.weight_decay * l2)) <= 1e-5 * abs(lv)
    _check_step(m, tr, (img, gt), loss, stats)


def test_one_pretraining_training_step():
    import pretraining_ref as PR
    m = _model("2222", data_shape=[64, 64, 3], bn_init="trained", is_pretraining=True)
    tr = _trainer(m)
    rng = np.random.default_rng(21)
    img = rng.integers(0, 256, (4, 64, 64, 3)).astype(np.float32)
    labels = np.array([0, 55, 17, 31])
    lab = torch.from_numpy(labels)
    stats = []
    loss, _, logits = tr.classify_loss(tr.forward_features(img, True, stats), lab)
    assert logits.shape == (4, 56)
    ref_data = PR.sparse_softmax_xent(logits.detach().numpy(), labels).mean(dtype=np.float32)
    l2 = sum(float((np.asarray(m.get_weights()[k], np.float64) ** 2).sum()) for k in m.pretraining_variables()) * 0.5
    ref = float(ref_data) + m.weight_decay * l2
    assert abs(float(loss) - ref) <= 1e-5 * abs(ref), (float(loss), ref)
    assert sorted(tr.params) == sorted(m.pretraining_variables())
    want_acc = float(torch.eq(logits.argmax(1), lab).float().mean())
    _, acc = _check_step(m, tr, (img, labels), loss, stats)
    assert acc == want_acc
    with pytest.raises(ValueError, match="outside"):
        tr.step(img, np.array([0, 1, 2, 56]), 1e-3)


def test_detection_loss_gradient_matches_finite_differences():
    """Training-mode forward + focal / smooth-L1 loss + L2 on a float64 copy: autograd against central differences
    for variables of a stride-1 unit (whose shortcut is its input), a stride-2 unit's shortcut conv, a BN and the
    class head.  (The stem is left out: its inputs are raw pixels, so a step small enough for the ReLU / max-pool
    pattern to hold is below the float64 resolution of the loss.)"""
    m = _model("2222", data_shape=[64, 64, 3], bn_init="trained")
    tr = _trainer(m, torch.float64)
    img = np.random.default_rng(9).integers(0, 256, (2, 64, 64, 3)).astype(np.float64)
    gt = _gt(2, 64, 10)

    def loss():
        return tr.total_loss(tr.forward_rows(img, True, []), gt)[0]

    picks = [("feature_extractor/block1_unit2/conv_branch/conv2d/kernel", (1, 1, 5, 2)),
             ("feature_extractor/block1_unit2/conv_branch/conv2d_1/kernel", (2, 0, 3, 6)),
             ("feature_extractor/block3_unit1/identity_branch/conv2d/kernel", (1, 2, 9, 20)),
             ("feature_extractor/block2_unit2/conv_branch/batch_normalization_1/gamma", (4,)),
             ("regressor/conv2d_4/bias", (20,))]
    names = [k for k, _ in picks]
    grads = torch.autograd.grad(loss(), [tr.params[k] for k in names])
    e = 1e-6
    for (k, idx), g in zip(picks, grads):
        p = tr.params[k]
        with torch.no_grad():
            v = float(p[idx])
            p[idx] = v + e
            lp = float(loss())
            p[idx] = v - e
            lm = float(loss())
            p[idx] = v
        fd = (lp - lm) / (2 * e)
        assert abs(fd - float(g[idx])) <= 1e-7 + 1e-5 * abs(fd), (k, idx, fd, float(g[idx]))


def test_checkpoint_handoff_and_cross_variant_loads(tmp_path):
    import RetinaNet
    from odt_b200 import tf_checkpoint as ck
    rng = np.random.default_rng(4)
    pre = _model("3463", is_pretraining=True)
    pre.set_weights({k: rng.standard_normal(v.shape).astype(np.float32) for k, v in pre.get_weights().items()})
    pre.global_step = 3
    out = pre.save_weight("latest", str(tmp_path / "basic" / "model"))
    names = pre.pretraining_variables()
    assert set(ck.open_checkpoint(out).get_variable_to_shape_map()) == set(names)
    assert len(names) == sum(1 for k in pre.get_weights() if not k.endswith(("moving_mean", "moving_variance")))

    det = _model("3463")
    w0 = {k: v.copy() for k, v in det.get_weights().items()}
    det.load_pretraining_weight(out)
    for k, v in det.get_weights().items():
        np.testing.assert_array_equal(v, pre.get_weights()[k] if k in names else w0[k], err_msg=k)

    # the bottleneck variant's checkpoint holds every basic name (with other shapes); the basic one lacks the
    # bottleneck's third conv: both refused, nothing restored
    bpre = RetinaNet.RetinaNet(model_cfg("retinanet", is_pretraining=True), None)
    bout = bpre.save_weight("latest", str(tmp_path / "bottleneck" / "model"))
    before = {k: v.copy() for k, v in det.get_weights().items()}
    with pytest.raises(ck.CheckpointError, match="another shape"):
        det.load_pretraining_weight(bout)
    with pytest.raises(ck.CheckpointError, match="another shape"):
        _model("3463", is_pretraining=True).load_weight(bout)
    for k, v in det.get_weights().items():
        np.testing.assert_array_equal(v, before[k], err_msg=k)
    bdet = RetinaNet.RetinaNet(model_cfg("retinanet"), None)
    bw = {k: v.copy() for k, v in bdet.get_weights().items()}
    with pytest.raises(ck.CheckpointError, match="lacks .*identity_branch"):
        bdet.load_pretraining_weight(out)
    with pytest.raises(ck.CheckpointError, match="lacks"):
        bpre.load_weight(out)
    for k, v in bdet.get_weights().items():
        np.testing.assert_array_equal(v, bw[k], err_msg=k)


@pytest.mark.parametrize("pretraining", [False, True])
@pytest.mark.parametrize("blocks", sorted(BLOCKS))
def test_fp16_planner_keeps_its_invariants(blocks, pretraining):
    """The fp16 engine's fusion and layout planning (Net.fuse / assign_halos / fuse_pools) on the basic graph at
    800^2 / 224^2, without a GPU: every residual has its output's halo, the identity shortcut stays the residual input
    of the second conv (the add is fused) and stays materialised, and the stem is eligible for the packed stem."""
    from odt_b200 import engine as E
    from odt_b200 import nets
    m = _model(blocks, is_pretraining=pretraining, data_shape=[224, 224, 3] if pretraining else [800, 800, 3])
    E.Net.spec_only = True
    try:
        build = nets.build_retinanet_backbone if pretraining else nets.build_retinanet
        net, _ = build(2, m.config, "fp16", "cpu", True)
    finally:
        E.Net.spec_only = False
    n_units = sum(BLOCKS[blocks])
    net.fuse()
    net.assign_halos()
    net.fuse_pools()
    res = [op for op in net.ops if isinstance(op, E.ConvOp) and op.residual is not None]
    assert len(res) == n_units
    read = {id(t) for op in net.ops for t in op.reads}
    for op in res:
        assert op.residual.halo == op.y.halo and op.residual.needed
        assert op.k == 3 and op.residual.C == op.y.C
        assert op.y.needed == (id(op.y) in read or (pretraining and op is res[-1])), op.kernel
    stem = net.ops[0]
    assert stem.is_image and (stem.k, stem.stride, stem.y.C) == (7, 2, 7) and stem.pre is None
    assert not any(isinstance(op, E.ConvOp) and op.pool for op in net.ops)
