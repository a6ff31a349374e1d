"""Training augmentation, CPU side: tfrecord.preprocess split into plan_augment (every draw and all box arithmetic) and
augment_pixels (numpy pixels), checked bit for bit against the one-piece preprocess it replaced (tests/augment_ref.py)
with the random stream included; the batch iterators against their former selves; the CUDA kernels' own per-pixel
functions (csrc/augment.cu, __host__ __device__) run on the CPU by tests/native/augment_host.cu against numpy; and
the C entry points' argument checks.  The kernels themselves need an H100 (tests/test_gpu_augment.py)."""
import ctypes as C
import itertools
import os
import shutil
import subprocess
import threading

import numpy as np
import pytest

import augment_ref as R
from odt_b200 import tfrecord as T

HERE = os.path.dirname(os.path.abspath(__file__))

BASE = {"data_format": "channels_last", "output_shape": [24, 20], "zoom_size": None, "crop_method": None,
        "flip_prob": None, "fill_mode": "BILINEAR", "keep_aspect_ratios": False, "constant_values": 0.,
        "color_jitter_prob": None, "rotate": None, "pad_truth_to": None}

# one axis at a time around BASE, then a few all-on mixes
CONFIGS = (
    [dict(fill_mode=f) for f in ("BILINEAR", "NEAREST_NEIGHBOR", "BICUBIC", "CONSTANT")]
    + [dict(fill_mode=f, keep_aspect_ratios=True, constant_values=c)
       for f, c in (("BILINEAR", 0.), ("NEAREST_NEIGHBOR", 7.5), ("BICUBIC", 128.))]
    + [dict(fill_mode="CONSTANT", constant_values=33., zoom_size=[30, 26], crop_method="random")]
    + [dict(zoom_size=[30, 26], crop_method=m) for m in ("random", "center", None)]
    + [dict(flip_prob=p) for p in ([0., 0.], [1., 1.], [1., 0.], [0.5, 0.5])]
    + [dict(color_jitter_prob=p) for p in (0., 1., 0.5)]
    + [dict(rotate=r) for r in ([0., -10., 10.], [1., -10., 10.], [1., 5., 5.])]
    + [dict(pad_truth_to=8), dict(pad_truth_to=2), dict(data_format="channels_first")]
    + [dict(fill_mode=f, zoom_size=[31, 27], crop_method="random", flip_prob=[0.5, 0.5], color_jitter_prob=0.5,
            rotate=[0.5, -10., 10.], pad_truth_to=6, data_format=d)
       for f, d in itertools.product(("BILINEAR", "NEAREST_NEIGHBOR", "BICUBIC", "CONSTANT"),
                                     ("channels_last", "channels_first"))]
    + [dict(fill_mode="BICUBIC", keep_aspect_ratios=True, zoom_size=[28, 28], crop_method="random",
            flip_prob=[1., 1.], color_jitter_prob=1., rotate=[1., -10., 10.], pad_truth_to=5)]
)
SIZES = [(37, 53), (1, 1), (24, 20), (80, 45), (9, 61)]


def _cfg(**kw):
    c = dict(BASE)
    c.update(kw)
    return c


def _boxes(rng, h, w, n, edge=False):
    if edge:   # boxes whose centres land on the border: filtered out -> gt_checker_helper's fallback
        return np.asarray([[0, 0, 0, 0.5, 3]] * n, np.float32)
    y = np.sort(rng.uniform(0, h, (n, 2)), 1)
    x = np.sort(rng.uniform(0, w, (n, 2)), 1)
    return np.concatenate([y, x, rng.integers(0, 20, (n, 1))], 1).astype(np.float32)


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("ci", range(len(CONFIGS)))
def test_plan_and_pixels_equal_the_one_piece_preprocess(ci):
    """plan_augment + augment_pixels == the former preprocess, pixels and boxes bit for bit, and the generator ends in
    the same state -- over every config, source sizes from 1 x 1 up, with boxes, with none left (fallback) and
    without ground truth."""
    kw = CONFIGS[ci]
    cfg = _cfg(**kw)
    fallbacks = 0
    for si, (h, w) in enumerate(SIZES):
        for seed in range(3):
            rng = np.random.default_rng(100 * ci + 10 * si + seed)
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            for gt in (_boxes(rng, h, w, 3), _boxes(rng, h, w, 2, edge=True), np.zeros((0, 5), np.float32), None):
                r1, r2 = np.random.default_rng(seed), np.random.default_rng(seed)
                ref = R.preprocess(img, gt, cfg, r1)
                plan, box = T.plan_augment(h, w, gt, cfg, r2)
                out = T.augment_pixels(img, plan)
                assert r1.bit_generator.state == r2.bit_generator.state
                if gt is None:
                    assert box is None and _same(out, ref)
                else:
                    assert _same(out, ref[0]) and _same(box, ref[1]), (kw, h, w, seed, plan)
                    assert _same(T.preprocess(img, gt, cfg, np.random.default_rng(seed))[0], ref[0])
                    fallbacks += plan.mode == "legacy"
    assert fallbacks > 0


def test_plan_without_a_generator_skips_the_random_steps():
    cfg = _cfg(zoom_size=[30, 26], crop_method="random", flip_prob=[1., 1.], color_jitter_prob=1.,
               rotate=[1., -10., 10.])
    img = np.random.default_rng(0).integers(0, 256, (37, 53, 3), dtype=np.uint8)
    plan, _ = T.plan_augment(37, 53, None, cfg, None)
    assert (plan.crop, plan.flip_y, plan.brightness, plan.angle) == ((3, 3), False, None, None)
    assert _same(T.augment_pixels(img, plan), R.preprocess(img, None, cfg, None))
    with pytest.raises(ValueError, match="color_jitter_prob"):
        T.plan_augment(5, 5, None, _cfg(color_jitter_prob=1.5), None)
    with pytest.raises(ValueError, match="rotate"):
        T.plan_augment(5, 5, None, _cfg(rotate=[0.5, 1.]), None)


# ------------------------------------------------------------------------------------------- batch iterators ---
def _write_voc(path, n, seed=0, bad=None):
    import cv2
    rng = np.random.default_rng(seed)
    recs = []
    for i in range(n):
        h, w = int(rng.integers(8, 60)), int(rng.integers(8, 60))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ok, enc = cv2.imencode(".jpg", img)
        assert ok
        data = b"not a jpeg" if i == bad else enc.tobytes()
        recs.append(T.encode_voc_example(data, [h, w, 3], _boxes(rng, h, w, int(rng.integers(1, 4)))))
    T.write_records(path, recs)
    return path


def _write_imagenet(path, n, seed=0):
    import cv2
    rng = np.random.default_rng(seed)
    recs = []
    for i in range(n):
        h, w = int(rng.integers(8, 60)), int(rng.integers(8, 60))
        ok, enc = cv2.imencode(".jpg", rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        recs.append(T.encode_imagenet_example(enc.tobytes(), [h, w, 3], i % 7))
    T.write_records(path, recs)
    return path


ITER_CFG = _cfg(output_shape=[16, 18], zoom_size=[20, 22], crop_method="random", flip_prob=[0.5, 0.5],
                color_jitter_prob=0.5, rotate=[0.5, -10., 10.], fill_mode="BILINEAR", pad_truth_to=4)


def _decode_threads():
    return [t for t in threading.enumerate() if t.name.startswith("odt-decode")]


@pytest.mark.parametrize("fmt", ["channels_last", "channels_first"])
def test_batch_iterator_equals_its_former_self(tmp_path, fmt):
    """7 records, shuffle buffer 3, batches of 2: 12 batches cross buffer refills and three `repeat` boundaries;
    identical batches and generator state to the one-piece iterator, and two seeded iterators agree."""
    path = _write_voc(str(tmp_path / "a.tfrecord"), 7)
    cfg = dict(ITER_CFG, data_format=fmt)
    ref, new, again = R.BatchIterator(path, 2, 3, cfg, seed=5), T.BatchIterator(path, 2, 3, cfg, seed=5), \
        T.BatchIterator([path], 2, 3, cfg, seed=5)
    for _ in range(12):
        (ri, rg), (ni, ng), (ai, ag) = ref.get_next(), new.get_next(), again.get_next()
        assert _same(ri, ni) and _same(rg, ng) and _same(ni, ai) and _same(ng, ag)
    assert ref.rng.bit_generator.state == new.rng.bit_generator.state
    new.close()
    again.close()
    assert not _decode_threads()


def test_imagenet_iterator_equals_its_former_self(tmp_path):
    path = _write_imagenet(str(tmp_path / "i.tfrecord"), 5)
    cfg = _cfg(output_shape=[12, 12], flip_prob=[0., 0.5], color_jitter_prob=0.5, data_format="channels_first")
    ref, new = R.ImageNetBatchIterator(path, 3, 2, cfg, seed=2), T.ImageNetBatchIterator(path, 3, 2, cfg, seed=2)
    for _ in range(6):
        (ri, rl), (ni, nl) = ref.get_next(), new.get_next()
        assert _same(ri, ni) and _same(rl, nl) and nl.dtype == np.int64
    del new
    assert not _decode_threads()


def test_undecodable_record_raises_at_the_same_batch(tmp_path):
    path = _write_voc(str(tmp_path / "b.tfrecord"), 9, bad=6)
    counts = []
    for it in (R.BatchIterator(path, 2, 2, ITER_CFG, seed=1), T.BatchIterator(path, 2, 2, ITER_CFG, seed=1)):
        n = 0
        with pytest.raises(T.RecordError, match="not decodable"):
            while True:
                it.get_next()
                n += 1
        counts.append(n)
    assert counts[0] == counts[1] == 2
    assert not _decode_threads()
    empty = str(tmp_path / "empty.tfrecord")
    T.write_records(empty, [])
    with pytest.raises(T.RecordError, match="no records"):
        T.BatchIterator(empty, 1, 1, ITER_CFG).get_next()


def test_a_new_initialize_restarts_the_stream_and_its_threads(tmp_path):
    path = _write_voc(str(tmp_path / "c.tfrecord"), 4)
    it = T.BatchIterator(path, 1, 1, ITER_CFG, seed=3)
    it.get_next()
    assert len(_decode_threads()) >= 1
    it.initialize()
    assert not _decode_threads()
    it.get_next()
    it.close()
    assert not _decode_threads()


# ------------------------------------------------------------------------------------- the kernels' own source ---
@pytest.fixture(scope="module")
def host():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(HERE, "native", "augment_host.cu")
    kern = os.path.join(HERE, "..", "object-detection-tensorflow_b200", "csrc", "augment.cu")
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    out = os.path.join(out_dir, "libaugment_host.so")
    deps = [src, kern, os.path.join(HERE, "..", "include", "odt_b200.h")]
    if not os.path.exists(out) or any(os.path.getmtime(f) > os.path.getmtime(out) for f in deps):
        # no contraction of a * b + c into an FMA on the host: the kernels' rounding is one rounding per operation
        subprocess.check_call([nvcc, "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler",
                               "-fPIC,-ffp-contract=off", "-shared", "-o", out, src])
    from odt_b200 import lib as L
    lib = C.CDLL(out)
    lib.odt_test_augment_host.restype = C.c_int
    lib.odt_test_augment_host.argtypes = [C.c_void_p, C.POINTER(L.AugmentParams), C.c_void_p, C.c_void_p]
    lib.odt_test_augment_hue.restype = None
    lib.odt_test_augment_hue.argtypes = [C.c_void_p, C.c_longlong, C.c_float]
    return lib


def _pre_contrast(img, plan):
    """augment_pixels up to (not including) the contrast step, HWC."""
    import copy
    p = copy.copy(plan)
    p.contrast = p.hue = p.angle = None
    p.channels_first = False
    return T.augment_pixels(img, p)


def _host_run(host, img, plan, means):
    from odt_b200.augment import kernel_params
    p = kernel_params(plan)
    out = np.empty((3, plan.oh, plan.ow) if plan.channels_first else (plan.oh, plan.ow, 3), np.float32)
    src = np.ascontiguousarray(img, np.uint8)
    m = np.ascontiguousarray(means if means is not None else np.zeros(3), np.float32)
    assert host.odt_test_augment_host(src.ctypes.data, C.byref(p), m.ctypes.data, out.ctypes.data) == 0
    return out


@pytest.mark.parametrize("ci", range(len(CONFIGS)))
def test_kernel_functions_equal_numpy_pixels(host, ci):
    """Every plan of the grid (all resize modes, canvas, crop, flips, each jitter step, rotation, the fallback, both
    layouts) through the kernels' per-pixel functions on the CPU == augment_pixels bit for bit, given the same
    contrast means (here the float64 mean of the pre-contrast image, rounded once)."""
    cfg = _cfg(**CONFIGS[ci])
    for si, (h, w) in enumerate(SIZES):
        for seed in range(3):
            rng = np.random.default_rng(1000 + 100 * ci + 10 * si + seed)
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            for gt in (_boxes(rng, h, w, 3), _boxes(rng, h, w, 2, edge=True), None):
                plan, _ = T.plan_augment(h, w, gt, cfg, np.random.default_rng(seed))
                means = None
                if plan.contrast is not None:
                    means = _pre_contrast(img, plan).astype(np.float64).mean(axis=(0, 1)).astype(np.float32)
                got = _host_run(host, img, plan, means)
                want = T.augment_pixels(img, plan, means)
                assert _same(got, want), (CONFIGS[ci], h, w, seed, plan)


def test_kernel_bicubic_and_nearest_tables_on_many_sizes(host):
    """Upscaling and downscaling by awkward ratios: every bicubic table offset class and nearest rounding case."""
    rng = np.random.default_rng(7)
    for (h, w), (oh, ow) in [((5, 7), (33, 29)), ((101, 67), (13, 17)), ((2, 2), (9, 3)), ((64, 48), (63, 49)),
                             ((1, 9), (4, 1)), ((300, 500), (97, 161))]:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        for fill in ("BILINEAR", "NEAREST_NEIGHBOR", "BICUBIC"):
            for keep in (False, True):
                cfg = _cfg(output_shape=[oh, ow], fill_mode=fill, keep_aspect_ratios=keep, constant_values=5.)
                plan, _ = T.plan_augment(h, w, None, cfg, None)
                assert _same(_host_run(host, img, plan, None), T.augment_pixels(img, plan)), (h, w, oh, ow, fill)


def test_kernel_hue_on_every_sector_and_tie(host):
    """adjust_hue of the kernel (aug_hue) == numpy on all six orderings of r, g, b, the ties r == g, g == b, r == b,
    grey, 0, 255.3, negative values (bicubic overshoot) and hue shifts that wrap past 0 and 6."""
    rng = np.random.default_rng(3)
    vals = [0., 255.3, 1., 2., 3., 128., -4.5, 300.25, 77.7]
    pix = [list(p) for p in itertools.product(vals, repeat=3)]
    pix += rng.uniform(-20, 280, (4000, 3)).tolist()
    pix += np.round(rng.uniform(0, 255, (2000, 3))).tolist()          # integer values: many exact ties
    rgb = np.asarray(pix, np.float32).reshape(-1, 1, 3)
    r, g, b = rgb[..., 0], rgb[..., 1], rgb[..., 2]
    assert np.any(r == g) and np.any(g == b) and np.any((r == g) & (g == b))
    for delta in (0.0, 0.1, -0.1, 0.0999, -0.0731, 0.05, 1e-9, -1e-9, 0.1 / 3):
        want = T.adjust_hue(rgb, delta)
        got = np.ascontiguousarray(rgb.copy())
        host.odt_test_augment_hue(got.ctypes.data, got.shape[0], float(np.float32(delta) * np.float32(6)))
        assert _same(got, want), delta


# ------------------------------------------------------------------------------------------------------- C ABI ---
def test_augment_symbols_and_argument_checks():
    """The entry points exist, size the scratch, and reject bad parameters before any CUDA call (no GPU here: an
    accepted call would reach the runtime)."""
    from odt_b200 import lib as L
    from odt_b200.augment import kernel_params
    lib = L.load()
    plan, _ = T.plan_augment(37, 53, None, _cfg(zoom_size=[30, 26], crop_method="center", color_jitter_prob=1.,
                                               rotate=[1., -5., 5.]), np.random.default_rng(0))

    def params(n=2, **kw):
        arr = (L.AugmentParams * n)(*[kernel_params(plan) for _ in range(n)])
        for k, v in kw.items():
            setattr(arr[n - 1], k, v)
        return arr
    good = params()
    assert lib.odt_augment_scratch_bytes(good, 2) > 2 * 24 * 20 * 3 * 4
    bad = [dict(h=0), dict(oh=0), dict(mode=7), dict(layout=2), dict(crop_y=7), dict(crop_x=-1), dict(flip_x=2),
           dict(hue_on=3), dict(rh=31), dict(ow=21), dict(src_offset=-1), dict(mode=L.AUG_PAD, rh=29),
           dict(mode=L.AUG_LEGACY), dict(zh=1 << 20, zw=1 << 20, oh=1 << 15, ow=1 << 15)]
    dummy = 256
    for kw in bad:
        p = params(**kw)
        assert lib.odt_augment_scratch_bytes(p, 2) == -1, kw
        assert lib.odt_augment_batch(dummy, p, 2, dummy, None, dummy, None) == -1, kw
        assert b"invalid argument" in lib.odt_last_error()
    assert lib.odt_augment_batch(dummy, None, 2, dummy, None, dummy, None) == -1
    assert lib.odt_augment_batch(dummy, good, 0, dummy, None, dummy, None) == -1
    assert lib.odt_augment_batch(None, good, 2, dummy, None, dummy, None) == -1
    assert lib.odt_augment_batch(dummy, good, 2, None, None, dummy, None) == -1
    assert lib.odt_augment_batch(dummy, good, 2, dummy, None, None, None) == -1
