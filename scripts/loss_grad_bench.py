"""Cost of the training step's data term: the per-image autograd restatement (GraphTrainer.image_loss, one Python
loop over the images) against the loss-gradient kernels (odt_<family>_loss_grad behind one autograd Function).

For each workload it times loss + backward to the candidate rows on the same rows with both paths (CUDA events, and a
host clock around a synchronise), the whole `tr.step` with each path (alternated, 3 repeats), and the difference of
the parameters after one step from the same weights: the largest relative difference of any variable, and the largest
absolute difference over the largest update.  Prints one JSON
line with the card's name and power limit read in the same run.

    python scripts/loss_grad_bench.py [--reps 5] [--only yolov3_416_c80,...]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "object-detection-tensorflow_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

BASE = {"mode": "test", "data_format": "channels_last", "num_classes": 20, "weight_decay": 1e-4, "keep_prob": 0.5,
        "nms_score_threshold": 0.3, "nms_max_boxes": 20, "nms_iou_threshold": 0.5, "pretraining_weight": None,
        "bn_init": "trained"}
WORKLOADS = {  # name -> (module, size, batch, config overrides)
    "ssd300": ("SSD300", 300, 32, {}),
    "retinanet_800": ("RetinaNet", 800, 8, dict(is_bottleneck=True, residual_block_list=[3, 4, 6, 3],
                                                init_conv_filters=16, is_pretraining=False, gamma=2.0, alpha=0.25)),
    "yolov3_416_c20": ("YOLOv3", 416, 16, dict(coord_scale=1, noobj_scale=1, obj_scale=5, class_scale=1, num_priors=3,
                                               priors=[[[10, 13], [16, 30], [33, 23]], [[30, 61], [62, 45], [59, 119]],
                                                       [[116, 90], [156, 198], [373, 326]]])),
    "yolov3_416_c80": ("YOLOv3", 416, 16, None),
    "fcos_1024": ("FCOS", 1024, 4, {}),
}
WORKLOADS["yolov3_416_c80"] = ("YOLOv3", 416, 16, dict(WORKLOADS["yolov3_416_c20"][3], num_classes=80))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        power = None
    return name, power


def ground_truth(rng, B, size, nc, G=60):
    """Padded to 60 rows like the data drivers; 5 to 20 boxes of 5 % to 60 % of the image side."""
    gt = np.full((B, G, 5), -1.0, np.float32)
    for b in range(B):
        n = int(rng.integers(5, 21))
        gt[b, :n, 0:2] = rng.uniform(0.1 * size, 0.9 * size, (n, 2))
        gt[b, :n, 2:4] = rng.uniform(0.05 * size, 0.6 * size, (n, 2))
        gt[b, :n, 4] = rng.integers(0, nc, n)
    return gt


def timed(fn, reps):
    """Median of `reps` runs after one warm-up: (CUDA-event ms, host ms around a synchronise)."""
    fn()
    torch.cuda.synchronize()
    ev, host = [], []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        host.append((time.perf_counter() - t0) * 1e3)
        ev.append(a.elapsed_time(b))
    return float(np.median(ev)), float(np.median(host))


def run(name, reps):
    from odt_b200.train import GraphTrainer
    mod, size, B, over = WORKLOADS[name]
    cfg = dict(BASE, batch_size=B, data_shape=[size, size, 3], **over)
    m = getattr(importlib.import_module(mod), mod)(cfg, None)
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (B, size, size, 3)).astype(np.float32)
    gt = ground_truth(rng, B, size, int(cfg["num_classes"]))
    ker, ref = GraphTrainer(m, "cuda"), GraphTrainer(m, "cuda")
    ref._loss_kernels = None
    p0 = {k: v.detach().clone() for k, v in ker.params.items()}
    with torch.no_grad():
        rows = ker.forward_rows(img).detach()
    rows.requires_grad_(True)

    def data_ref():
        per = [ref.image_loss(rows[b], gt[b]) for b in range(B)]
        torch.autograd.grad(torch.stack(per).sum() / B, rows)

    def data_ker():
        torch.autograd.grad(ker._loss_kernels(rows, gt).sum() / B, rows)
    out = {"batch": B}
    out["data_restatement_ms"], out["data_restatement_host_ms"] = timed(data_ref, reps)
    out["data_kernels_ms"], out["data_kernels_host_ms"] = timed(data_ker, reps)
    # one step each from the same weights: parameter difference relative to the update
    ker.step(img, gt, 1e-3)
    ref.step(img, gt, 1e-3)
    upd = max(float((ref.params[k] - p0[k]).abs().max()) for k in p0)
    diff = max(float((ker.params[k] - ref.params[k]).abs().max()) for k in p0)
    out["param_max_rel_diff"] = max(float((ker.params[k] - ref.params[k]).abs().max())
                                    / max(float(ref.params[k].abs().max()), 1e-30) for k in p0)
    out["param_diff_over_largest_update"] = diff / upd
    steps = {"restatement": [], "kernels": []}
    for _ in range(3):
        for label, tr in (("restatement", ref), ("kernels", ker)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.step(img, gt, 1e-3)
            torch.cuda.synchronize()
            steps[label].append((time.perf_counter() - t0) * 1e3)
    out["step_restatement_ms"] = steps["restatement"]
    out["step_kernels_ms"] = steps["kernels"]
    del ker, ref, rows
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    import __graft_entry__  # noqa: F401  (paths)
    from odt_b200 import lib
    lib.load()
    name, power = card()
    res = {"card": name, "power_limit_w": power, "workloads": {}}
    for w in (a.only.split(",") if a.only else WORKLOADS):
        res["workloads"][w] = run(w, a.reps)
        print("%s: %s" % (w, json.dumps(res["workloads"][w])), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
