"""RetinaNet's ImageNet-pretraining mode on the H100: the pooled-logit classification kernel (odt_pool_classify)
against float64 numpy, the whole network against the CPU oracle, graph replay against eager launches, the kernel's
loss against autograd, and two training steps whose checkpoint seeds a detection model."""
import numpy as np
import pytest
import torch

from helpers import model_cfg

pytestmark = pytest.mark.gpu


def _launch(feat, dtype_code, B, H, W, Cc, ld, halo, labels=None):
    from odt_b200 import lib as L
    logits = torch.empty((B, Cc), dtype=torch.float32, device="cuda")
    pred = torch.empty((B,), dtype=torch.int64, device="cuda")
    loss = torch.empty((B,), dtype=torch.float32, device="cuda") if labels is not None else None
    L.check(L.load().odt_pool_classify(feat.data_ptr(), dtype_code, B, H, W, Cc, ld, halo, logits.data_ptr(),
                                       pred.data_ptr(), labels.data_ptr() if labels is not None else None,
                                       loss.data_ptr() if loss is not None else None,
                                       torch.cuda.current_stream().cuda_stream), "pool_classify")
    torch.cuda.synchronize()
    return logits.cpu().numpy(), pred.cpu().numpy(), (loss.cpu().numpy() if loss is not None else None)


SHAPES = [(1, 1, 1), (20, 7, 7), (224, 7, 7), (224, 16, 16), (1000, 1, 1), (1000, 7, 7), (20, 64, 64),
          (224, 64, 64), (1000, 64, 64), (224, 1, 64), (3, 5, 9)]


@pytest.mark.parametrize("dtype", ["fp16", "fp32"])
@pytest.mark.parametrize("halo", [0, 1])
@pytest.mark.parametrize("ld_kind", ["padded", "dense"])
@pytest.mark.parametrize("Cc,H,W", SHAPES)
def test_pool_classify_kernel(dtype, halo, ld_kind, Cc, H, W):
    """Logits within 1e-6 relative of the float64 mean, the first maximum exactly (ties included), the loss within
    1e-6 of float64 on the kernel's logits, bit-identical replays; NaN in every pad lane and halo pixel shows that
    none of them is summed.  'padded' ld takes the 16-byte path, 'dense' ld = C the scalar one when C is odd."""
    from odt_b200 import lib as L
    import pretraining_ref as PR
    B = 3
    ld = (-(-Cc // 8) * 8 + 8) if ld_kind == "padded" else Cc
    tdt = torch.float16 if dtype == "fp16" else torch.float32
    rng = np.random.default_rng(Cc * 1000 + H * 10 + W + halo)
    full = np.full((B, H + 2 * halo, W + 2 * halo, ld), np.nan, np.float32)
    vals = (rng.standard_normal((B, H, W, Cc)) * 2.0 + rng.standard_normal((1, 1, 1, Cc))).astype(np.float32)
    if Cc >= 3:   # image 1: a tie for the maximum between channels 1 and Cc-1 (first index wins)
        vals[1, :, :, Cc - 1] = vals[1, :, :, 1]
        vals[1, :, :, 1] += 50.0
        vals[1, :, :, Cc - 1] += 50.0
    full[:, halo:halo + H, halo:halo + W, :Cc] = vals
    feat = torch.from_numpy(full).to(tdt).cuda()
    stored = feat.float().cpu().numpy()[:, halo:halo + H, halo:halo + W, :Cc].astype(np.float64)
    ref = stored.mean(axis=(1, 2))
    labels = torch.from_numpy(rng.integers(0, Cc, B)).cuda()
    code = L.ODT_F16 if dtype == "fp16" else L.ODT_F32
    lg, pred, loss = _launch(feat, code, B, H, W, Cc, ld, halo, labels)
    assert np.all(np.abs(lg - ref) <= 1e-6 * np.abs(ref) + 1e-30), float(np.abs(lg - ref).max())
    np.testing.assert_array_equal(pred, np.argmax(lg, axis=1))
    if Cc >= 3:
        assert pred[1] == 1 and lg[1, 1] == lg[1, Cc - 1]
    want = PR.sparse_softmax_xent64(lg, labels.cpu().numpy())
    assert np.all(np.abs(loss - want) <= 1e-6 * np.abs(want) + 1e-7), (loss, want)
    lg2, pred2, loss2 = _launch(feat, code, B, H, W, Cc, ld, halo, labels)
    assert lg2.tobytes() == lg.tobytes() and np.array_equal(pred2, pred) and loss2.tobytes() == loss.tobytes()
    lg3, pred3, none = _launch(feat, code, B, H, W, Cc, ld, halo)
    assert none is None and lg3.tobytes() == lg.tobytes() and np.array_equal(pred3, pred)


def _model(**over):
    import RetinaNet
    return RetinaNet.RetinaNet(model_cfg("retinanet", is_pretraining=True, bn_init="trained", **over), None)


@pytest.fixture(scope="module")
def oracle_cases():
    """(size, model, images, oracle logits float64) at 224^2 and 500^2, B = 2."""
    import pretraining_ref as PR
    out = {}
    for size in (224, 500):
        m = _model(data_shape=[size, size, 3])
        img = np.random.default_rng(size).integers(0, 256, (2, size, size, 3)).astype(np.float32)
        ref = PR.pooled_logits(PR.retinanet_features(m.get_weights(), img))
        out[size] = (m, img, ref)
    return out


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("size", [224, 500])
def test_network_matches_the_oracle(oracle_cases, size, precision):
    """fp32: 2e-4 x max|ref| (the detection rows' fp32 bar; measured 1.4e-7 .. 3.4e-7); fp16: 2e-3 x max|ref|, four
    times the measured 4.2e-4 .. 5.0e-4 and tighter than the detection rows' 5e-3.  pred equals the oracle's arg-max
    wherever the top-2 margin exceeds the measured logit error."""
    m, img, ref = oracle_cases[size]
    net = m._classify(img, precision)
    got = net.tail.logits.cpu().numpy()
    pred = net.tail.results()
    assert got.shape == ref.shape == (2, 224) and pred.dtype == np.int64
    err, scale = float(np.abs(got - ref).max()), float(np.abs(ref).max())
    print("pretraining %d^2 %s: max|logit err| %.3g, max|ref| %.3g (%.2g relative)" % (size, precision, err, scale,
                                                                                      err / scale))
    assert err <= (2e-4 if precision == "fp32" else 2e-3) * scale
    top2 = np.sort(ref, axis=1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > err
    np.testing.assert_array_equal(pred[clear], np.argmax(ref, axis=1)[clear])
    np.testing.assert_array_equal(pred, np.argmax(got, axis=1))
    if precision == m.precision:
        np.testing.assert_array_equal(m.test_one_image(img), pred)


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_graph_replay_equals_eager_and_loss_matches_autograd(precision):
    from odt_b200.train import pooled_xent
    m = _model(data_shape=[224, 224, 3])
    img = np.random.default_rng(7).integers(0, 256, (2, 224, 224, 3)).astype(np.float32)
    labels = np.array([5, 223])
    net = m._classify(img, precision)                         # the captured graph
    assert net.graph is not None
    g_logits, g_pred = net.tail.logits.clone(), net.tail.pred.clone()
    eager, tail = m._build(2, precision)
    eager.finalize(m.get_weights(), tail)
    eager.image_buf.copy_(torch.from_numpy(img))
    eager.forward()
    torch.cuda.synchronize()
    assert torch.equal(tail.logits, g_logits) and torch.equal(tail.pred, g_pred)
    assert net.num_launches() == eager.num_launches()

    loss = m.loss_forward(img, labels, precision)
    f = net.tail.feat
    feats = f.buf[:, f.halo:f.halo + f.H, f.halo:f.halo + f.W, :f.C].double().permute(0, 3, 1, 2).cpu()
    for b in range(2):
        want = float(pooled_xent(feats[b:b + 1], torch.tensor(labels[b:b + 1]))[0])
        assert abs(float(loss[b]) - want) <= 1e-6 * abs(want), (b, float(loss[b]), want)
    with pytest.raises(ValueError, match="outside"):
        m.loss_forward(img, np.array([0, 224]), precision)


def test_two_training_steps_then_detection_handoff(tmp_path):
    import RetinaNet
    rng = np.random.default_rng(2)

    class It:
        n = 0

        def initialize(self):
            self.n = 0

        def get_next(self):
            self.n += 1
            return rng.integers(0, 256, (2, 128, 128, 3)).astype(np.float32), rng.integers(0, 224, 2)

    it = It()
    provider = {"num_train": 4, "num_val": 0, "train_generator": (it.initialize, it), "val_generator": None}
    cfg = model_cfg("retinanet", is_pretraining=True, mode="train", batch_size=2)
    m = RetinaNet.RetinaNet(cfg, provider)
    loss, acc = m.train_one_epoch(1e-3)
    assert np.isfinite(loss) and np.isfinite(acc) and it.n == 2 and m.global_step == 2
    assert m.test_one_image(it.get_next()[0]).shape == (2,)
    out = m.save_weight("latest", str(tmp_path / "pre" / "model"))
    det = RetinaNet.RetinaNet(model_cfg("retinanet"), None)
    det.load_pretraining_weight(out)
    k = "feature_extractor/block4_unit3/conv_branch/conv2d_2/kernel"
    np.testing.assert_array_equal(det.get_weights()[k], m.get_weights()[k])
    res = det.test_one_image(np.random.default_rng(3).integers(0, 256, (1, 128, 128, 3)).astype(np.float32))
    assert len(res) == 3
