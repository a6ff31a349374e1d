"""Input-pipeline timing: BatchIterator.get_next() (numpy augmentation) against get_next("cuda") (csrc/augment.cu),
the augmentation kernels alone, and train_one_epoch steps per second on each path, for the five configurations of
the input-pipeline table in DESIGN section 7.  Synthetic records (seeded images through cv2.imencode, 500 x 375 and
a ragged mix of sizes) are written to a temporary directory.

    python scripts/augment_bench.py [--batches 5] [--steps 6] [--only ssd300,yolov3,...] [--no-train]

Wall times are host clocks around a torch.cuda.synchronize(); kernel times are CUDA events around
odt_augment_batch on already staged sources.  The train_one_epoch line of each path also gives the fetch and
tr.step times measured inside that epoch.  The card name, its power limit and the CPU cores visible to the process are
printed with the numbers."""
import argparse
import gc
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "object-detection-tensorflow_b200"), os.path.join(ROOT, "tests")]

BASE = {"data_format": "channels_last", "zoom_size": None, "crop_method": None, "flip_prob": None,
        "fill_mode": "BILINEAR", "keep_aspect_ratios": False, "constant_values": 0., "color_jitter_prob": None,
        "rotate": None, "pad_truth_to": 60}
# name: (model module, model kind, batch, augmentation overrides, ImageNet records)
CONFIGS = {
    "ssd300": ("SSD300", "ssd", 32, dict(output_shape=[300, 300], zoom_size=[320, 320], crop_method="random",
                                         flip_prob=[0., 0.5]), False),
    "ssd300_jitter_rotate": ("SSD300", "ssd", 32, dict(output_shape=[300, 300], zoom_size=[320, 320],
                                                       crop_method="random", flip_prob=[0., 0.5],
                                                       color_jitter_prob=1., rotate=[1., -5., 5.]), False),
    "yolov3_416": ("YOLOv3", "yolov3", 16, dict(output_shape=[416, 416], flip_prob=[0., 0.5],
                                                color_jitter_prob=0.5), False),
    "retinanet_800": ("RetinaNet", "retinanet", 8, dict(output_shape=[800, 800], fill_mode="BICUBIC",
                                                        flip_prob=[0., 0.5]), False),
    "retinanet_pretraining_224": ("RetinaNet", "retinanet", 256, dict(output_shape=[224, 224], flip_prob=[0., 0.5],
                                                                      pad_truth_to=None), True),
}


# RetinaNet pretraining trains at B = 64 here: its B = 256 step holds ResNet-50 activations for 256 images in fp32
TRAIN_BATCH_CAP = 64


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "unknown (%s)" % e


def write_records(d, n, imagenet):
    import cv2
    from odt_b200 import tfrecord as T
    rng = np.random.default_rng(0)
    recs = []
    for i in range(n):
        h, w = (375, 500) if i % 2 == 0 else (int(rng.integers(200, 501)), int(rng.integers(200, 501)))
        img = cv2.GaussianBlur(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), (7, 7), 2)   # JPEG-like content
        ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])
        if imagenet:
            recs.append(T.encode_imagenet_example(enc.tobytes(), [h, w, 3], i % 1000))
        else:
            k = int(rng.integers(1, 6))
            y = np.sort(rng.uniform(0, h, (k, 2)), 1)
            x = np.sort(rng.uniform(0, w, (k, 2)), 1)
            gt = np.concatenate([y, x, rng.integers(0, 20, (k, 1))], 1)
            recs.append(T.encode_voc_example(enc.tobytes(), [h, w, 3], gt))
    path = os.path.join(d, "imagenet.tfrecord" if imagenet else "voc.tfrecord")
    T.write_records(path, recs)
    return path


def timed(fn, n):
    import torch
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(t))


def kernel_ms(items, reps=20):
    """CUDA-event time of odt_augment_batch alone, sources already on the device."""
    import ctypes as C
    import torch
    from odt_b200 import lib as L
    from odt_b200.augment import GpuAugmentor, kernel_params
    g = GpuAugmentor()
    out = g(items, "cuda")
    offs = np.concatenate([[0], np.cumsum([i[0].nbytes for i in items])])
    params = (L.AugmentParams * len(items))(*[kernel_params(i[1], o) for i, o in zip(items, offs[:-1])])
    lib = L.load()
    st = torch.cuda.current_stream()
    run = lambda: L.check(lib.odt_augment_batch(g._src.data_ptr(), params, len(items), out.data_ptr(), None,  # noqa
                                                g._scratch.data_ptr(), st.cuda_stream), "odt_augment_batch")
    run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(reps):
        run()
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, sum(C.sizeof(C.c_float) * o.numel() for o in [out]) / 1e6


class Plain:
    def __init__(self, it):
        self.it = it

    def initialize(self):
        self.it.initialize()

    def get_next(self):
        return self.it.get_next()


def train_rate(mod, kind, batch, aug, path, imagenet, steps, device_path):
    """One epoch of `steps` train_one_epoch steps after a one-step warm-up epoch (trainer, kernels, allocator).
    -> (steps/s of the whole epoch, median ms of the batch fetch and of tr.step inside it).  The epoch rate includes
    the shuffle-buffer fill of the iterator's restart and the trainer's export at the end; the fetch and step times
    are taken in the loop itself, each ended by a synchronise, so that the rate can be read against them."""
    import importlib
    import torch
    from helpers import model_cfg
    from odt_b200 import tfrecord as T
    size = aug["output_shape"][0]
    over = dict(is_pretraining=True) if imagenet else {}
    cfg = model_cfg(kind, data_shape=[size, size, 3], mode="train", batch_size=batch, **over)
    make = T.ImageNetBatchIterator if imagenet else T.BatchIterator
    it = make(path, batch, 2 * batch, aug, seed=0)
    it = it if device_path else Plain(it)
    fetch_ms, step_ms = [], []
    get_next = it.get_next

    def timed_get_next(*a):
        t0 = time.perf_counter()
        out = get_next(*a)
        torch.cuda.synchronize()
        fetch_ms.append(1e3 * (time.perf_counter() - t0))
        return out
    it.get_next = timed_get_next          # an instance attribute: the iterator stays a BatchIterator
    provider = {"num_train": batch, "num_val": 0, "train_generator": (it.initialize, it), "val_generator": None}
    m = getattr(importlib.import_module(mod), mod)(cfg, provider)
    tr = m.trainer()
    step = tr.step

    def timed_step(*a):
        t0 = time.perf_counter()
        out = step(*a)
        torch.cuda.synchronize()
        step_ms.append(1e3 * (time.perf_counter() - t0))
        return out
    tr.step = timed_step
    m.train_one_epoch(1e-4)
    fetch_ms.clear()
    step_ms.clear()
    m.num_train = batch * steps
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.train_one_epoch(1e-4)
    torch.cuda.synchronize()
    rate = steps / (time.perf_counter() - t0)
    (it.it if isinstance(it, Plain) else it).close()
    del m, tr
    gc.collect()
    torch.cuda.empty_cache()
    return rate, float(np.median(fetch_ms)), float(np.median(step_ms)), fetch_ms[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=5)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--only", default="")
    ap.add_argument("--no-train", action="store_true")
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from odt_b200 import tfrecord as T
    print("card: %s; torch %s; %d CPU cores visible" % (card(), torch.__version__, len(os.sched_getaffinity(0))))
    names = [n for n in CONFIGS if not a.only or n in a.only.split(",")]
    with tempfile.TemporaryDirectory() as d:
        voc, imnet = write_records(d, 64, False), write_records(d, 64, True)
        for name in names:
            mod, kind, batch, over, imagenet = CONFIGS[name]
            aug = dict(BASE, **over)
            path = imnet if imagenet else voc
            make = T.ImageNetBatchIterator if imagenet else T.BatchIterator
            host_it, dev_it = make(path, batch, 2 * batch, aug, seed=0), make(path, batch, 2 * batch, aug, seed=0)
            host_ms = timed(lambda: host_it.get_next(), a.batches)
            dev_ms = timed(lambda: dev_it.get_next("cuda"), a.batches)
            items = dev_it._next_items()
            k_ms, mb = kernel_ms(items)
            line = ("%-26s B=%-3d get_next() %8.1f ms/batch | get_next('cuda') %7.1f ms/batch | kernels %.3f ms "
                    "(%.1f MB out)" % (name, batch, host_ms, dev_ms, k_ms, mb))
            print(line, flush=True)
            if not a.no_train:
                tb = min(batch, TRAIN_BATCH_CAP)
                for dev_path in (False, True):
                    r, f, st, first = train_rate(mod, kind, tb, aug, path, imagenet, a.steps, dev_path)
                    print("%-26s   train_one_epoch B=%-3d %-6s path: %5.2f steps/s over %d steps (epoch: restart + "
                          "buffer fill + export included); in the loop: fetch %.1f ms median (first %.1f ms, with "
                          "the buffer fill), tr.step %.1f ms median" % (name, tb, "device" if dev_path else "numpy",
                                                                      r, a.steps, f, first, st), flush=True)
            host_it.close()
            dev_it.close()


if __name__ == "__main__":
    main()
