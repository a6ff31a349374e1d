"""Training augmentation on the GPU (csrc/augment.cu behind BatchIterator.get_next(device)): bit for bit the numpy
step (tfrecord.augment_pixels) wherever the contrast step did not fire, and the numpy step fed the kernels' own
contrast means where it did; those means within 1 fp32 ulp of the float64 mean; replays and batch independence;
train_one_epoch on the device path against the numpy path."""
import numpy as np
import pytest
import torch

from odt_b200 import tfrecord as T
from test_augment import BASE, _boxes, _cfg, _pre_contrast, _same, _write_imagenet, _write_voc

pytestmark = pytest.mark.gpu

# sources: 1 x 1, smaller and larger than the outputs, odd sizes
SOURCES = [(1, 1), (3, 2), (37, 53), (375, 500), (17, 301), (64, 64), (299, 301), (8, 5)]
OUTPUT_CONFIGS = [
    _cfg(output_shape=[1, 1]),
    _cfg(output_shape=[1, 1], zoom_size=[5, 3], crop_method="random", color_jitter_prob=1., rotate=[1., -10., 10.]),
    _cfg(output_shape=[33, 47], fill_mode="BICUBIC", flip_prob=[0.5, 0.5], color_jitter_prob=0.5,
         rotate=[0.5, -10., 10.], pad_truth_to=6),
    _cfg(output_shape=[300, 300], zoom_size=[320, 320], crop_method="random", flip_prob=[0.5, 0.5],
         color_jitter_prob=1., rotate=[1., -10., 10.], pad_truth_to=10),
    _cfg(output_shape=[64, 80], fill_mode="NEAREST_NEIGHBOR", keep_aspect_ratios=True, constant_values=11.,
         color_jitter_prob=0.5, data_format="channels_first"),
    _cfg(output_shape=[41, 29], fill_mode="CONSTANT", constant_values=3., zoom_size=[50, 40], crop_method="random",
         flip_prob=[1., 0.], color_jitter_prob=0.5, rotate=[0.5, -10., 10.], data_format="channels_first"),
    _cfg(output_shape=[96, 96], fill_mode="BILINEAR", keep_aspect_ratios=True, color_jitter_prob=0.7),
]


def _items(cfg, seed, with_edge=True):
    rng = np.random.default_rng(seed)
    plan_rng = np.random.default_rng(seed + 1)
    items = []
    for k, (h, w) in enumerate(SOURCES):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        gt = _boxes(rng, h, w, 2, edge=with_edge and k % 3 == 2)       # some fall back to the legacy resize
        items.append((img,) + T.plan_augment(h, w, gt, cfg, plan_rng))
    return items


def _gpu(items, means=True):
    from odt_b200.augment import GpuAugmentor
    m = torch.full((len(items), 3), float("nan"), device="cuda") if means else None
    out = GpuAugmentor()(items, "cuda", m)
    torch.cuda.synchronize()
    return out.cpu().numpy(), (m.cpu().numpy() if means else None)


@pytest.mark.parametrize("ci", range(len(OUTPUT_CONFIGS)))
def test_kernels_equal_numpy_pixels(built, ci):
    cfg = OUTPUT_CONFIGS[ci]
    contrast_seen, worst_ulp, worst_np = 0, 0.0, 0.0
    for seed in range(3):
        items = _items(cfg, 17 * ci + seed)
        got, means = _gpu(items)
        for b, (img, plan, _) in enumerate(items):
            if plan.contrast is None:
                assert np.all(np.isnan(means[b]))
                assert _same(got[b], T.augment_pixels(img, plan)), (b, plan)
                continue
            contrast_seen += 1
            assert _same(got[b], T.augment_pixels(img, plan, means[b])), (b, plan)
            pre = _pre_contrast(img, plan)
            exact = pre.astype(np.float64).mean(axis=(0, 1))
            ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
            err = np.abs(means[b].astype(np.float64) - exact) / ulp
            np_err = np.abs(pre.mean(axis=(0, 1), dtype=np.float32).astype(np.float64) - exact) / ulp
            assert np.all(err <= 1.0), (b, err)
            worst_ulp, worst_np = max(worst_ulp, float(err.max())), max(worst_np, float(np_err.max()))
    print("config %d: %d contrast images; kernel mean error <= %.3f fp32 ulp of the float64 mean (numpy's float32 "
          "mean: %.3f ulp)" % (ci, contrast_seen, worst_ulp, worst_np))


def test_replay_and_batch_independence(built):
    cfg = OUTPUT_CONFIGS[3]
    items = _items(cfg, 5)
    a, ma = _gpu(items)
    b, mb = _gpu(items)
    assert a.tobytes() == b.tobytes() and ma.tobytes() == mb.tobytes()
    for k in (0, 3, len(items) - 1):
        alone, m1 = _gpu([items[k]])
        assert alone[0].tobytes() == a[k].tobytes() and m1[0].tobytes() == ma[k].tobytes()
    rev, mr = _gpu(items[::-1])
    assert rev[::-1].tobytes() == a.tobytes() and mr[::-1].tobytes() == ma.tobytes()


def test_rejected_plan_raises_before_launch(built):
    from odt_b200.augment import GpuAugmentor
    cfg = _cfg(output_shape=[40, 40], zoom_size=[30, 30], crop_method="center")   # zoom smaller than the output
    img = np.zeros((20, 20, 3), np.uint8)
    plan, _ = T.plan_augment(20, 20, None, cfg, None)
    with pytest.raises(ValueError, match="crop window"):
        GpuAugmentor()([(img, plan)], "cuda")


@pytest.mark.parametrize("fmt", ["channels_last", "channels_first"])
def test_get_next_on_the_device_equals_get_next(built, tmp_path, fmt):
    """Two iterators with the same seed over ragged records, several batches across refills and repeats: truth
    bit-identical; images bit-identical where contrast did not fire, and equal to the numpy step fed the kernels'
    means where it did (a third iterator with that seed gives the plans)."""
    path = _write_voc(str(tmp_path / "v.tfrecord"), 9, seed=4)
    cfg = _cfg(output_shape=[30, 26], zoom_size=[34, 30], crop_method="random", flip_prob=[0.5, 0.5],
               color_jitter_prob=0.5, rotate=[0.5, -10., 10.], pad_truth_to=5, data_format=fmt)
    dev, host, plans = (T.BatchIterator(path, 4, 3, cfg, seed=8) for _ in range(3))
    fired = 0
    for _ in range(6):
        gi, gg = dev.get_next("cuda")
        ci, cg = host.get_next()
        items = plans._next_items()
        assert gi.is_cuda and gi.dtype == torch.float32 and tuple(gi.shape) == ci.shape
        assert _same(gg, cg)
        _, means = _gpu(items)
        gi = gi.cpu().numpy()
        for b, (img, plan, _) in enumerate(items):
            if plan.contrast is None:
                assert _same(gi[b], ci[b])
            else:
                fired += 1
                assert _same(gi[b], T.augment_pixels(img, plan, means[b]))
    assert fired > 0
    for it in (dev, host, plans):
        it.close()


def test_imagenet_get_next_on_the_device(built, tmp_path):
    path = _write_imagenet(str(tmp_path / "i.tfrecord"), 6, seed=1)
    cfg = _cfg(output_shape=[24, 24], flip_prob=[0., 0.5], fill_mode="BICUBIC", data_format="channels_first")
    dev, host = T.ImageNetBatchIterator(path, 4, 2, cfg, seed=2), T.ImageNetBatchIterator(path, 4, 2, cfg, seed=2)
    for _ in range(4):
        (gi, gl), (ci, cl) = dev.get_next(torch.device("cuda")), host.get_next()
        assert _same(gi.cpu().numpy(), ci) and _same(gl, cl)


# ------------------------------------------------------------------------------------------ train_one_epoch ---
class _Plain:
    """Any iterator object that is not a BatchIterator: train_one_epoch takes its numpy batches."""

    def __init__(self, it):
        self.it = it

    def initialize(self):
        self.it.initialize()

    def get_next(self):
        return self.it.get_next()


def _epoch(mod, cfg, iterator, num_train, seen):
    import importlib
    provider = {"num_train": num_train, "num_val": 0, "train_generator": (iterator.initialize, iterator),
                "val_generator": None}
    m = getattr(importlib.import_module(mod), mod)(cfg, provider)
    tr = m.trainer()
    p0 = {k: v.detach().clone() for k, v in tr.params.items()}
    step = tr.step

    def spy(images, truth, lr):
        seen.append((images.is_cuda if isinstance(images, torch.Tensor) else False,
                     images.cpu().numpy() if isinstance(images, torch.Tensor) else np.array(images)))
        return step(images, truth, lr)
    tr.step = spy
    out = m.train_one_epoch(1e-3)
    return out, p0, tr.params


@pytest.mark.parametrize("name", ["ssd300", "yolov3", "retinanet_pretraining"])
def test_train_one_epoch_on_the_device_path(built, tmp_path, name):
    """Two steps of train_one_epoch fed by a BatchIterator (the device path) and by the same seeded iterator behind a
    plain wrapper (the numpy path), jitter off: the images tr.step receives are identical, and the parameters agree
    within the training-step bound of the loss-gradient tests (5e-3 of the largest update), or within twice the
    spread of the numpy path against itself where that is wider."""
    from helpers import model_cfg
    from test_gpu_loss_grad import STEP, STEP_PARAM_BOUND
    if name == "retinanet_pretraining":
        mod, size, data = "RetinaNet", 128, _write_imagenet(str(tmp_path / "p.tfrecord"), 5, seed=3)
        cfg = model_cfg("retinanet", is_pretraining=True, mode="train", batch_size=2)
        make = T.ImageNetBatchIterator
    else:
        mod, kind, size, over = STEP[name]
        data = _write_voc(str(tmp_path / "d.tfrecord"), 5, seed=3)
        cfg = model_cfg(kind, data_shape=[size, size, 3], bn_init="trained", mode="train", batch_size=2, **over)
        make = T.BatchIterator
    aug = dict(BASE, output_shape=[size, size], zoom_size=[size + 12, size + 12], crop_method="random",
               flip_prob=[0.5, 0.5], rotate=[0.5, -10., 10.], pad_truth_to=8,
               data_format=cfg.get("data_format", "channels_last"))
    dev_seen, np_seen, np2_seen = [], [], []
    dev = _epoch(mod, cfg, make(data, 2, 3, aug, seed=6), 4, dev_seen)
    ref = _epoch(mod, cfg, _Plain(make(data, 2, 3, aug, seed=6)), 4, np_seen)
    ref2 = _epoch(mod, cfg, _Plain(make(data, 2, 3, aug, seed=6)), 4, np2_seen)
    assert len(dev_seen) == len(np_seen) == 2
    assert all(s[0] for s in dev_seen) and not any(s[0] for s in np_seen)
    for (_, a), (_, b) in zip(dev_seen, np_seen):
        assert _same(a, b)
    p0, pd, pr, pr2 = dev[1], dev[2], ref[2], ref2[2]
    with torch.no_grad():
        upd = max(float((pr[k] - p0[k]).abs().max()) for k in p0)
        diff = max(float((pd[k] - pr[k]).abs().max()) for k in p0)
        noise = max(float((pr2[k] - pr[k]).abs().max()) for k in p0)
    # the inputs are identical, so what is left is the training step's own run-to-run spread (atomics in PyTorch's
    # convolution backward), which two steps compound: measured beside it on the numpy path run twice
    bound, binding = max((STEP_PARAM_BOUND * upd, "%g of the largest update" % STEP_PARAM_BOUND),
                         (2 * noise, "twice the numpy path's spread against itself"))
    print("%s: loss device path %r numpy path %r; max param difference %.3g of the largest update (numpy path run "
          "twice: %.3g); binding bound: %s" % (name, dev[0], ref[0], diff / upd, noise / upd, binding))
    assert diff <= bound, (diff / upd, binding)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_one_augmentor_on_two_devices(built):
    """The buffers follow the device a call names: a second device gets its own source copy and scratch."""
    from odt_b200.augment import GpuAugmentor
    items = _items(OUTPUT_CONFIGS[2], 3)
    g = GpuAugmentor()
    a = g(items, "cuda:0")
    b = g(items, "cuda:1")
    assert g._src.device == torch.device("cuda", 1) and b.device == torch.device("cuda", 1)
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
