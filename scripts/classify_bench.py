#!/usr/bin/env python
"""RetinaNet ImageNet-pretraining inference on one GPU: images/s of the captured forward (fp16, graph replay) and the
CUDA-event time of the pooled-logit classification kernel alone, with the card's name and power limit read in the
same run.  Prints one JSON line.
usage: classify_bench.py [--batch 256] [--size 224] [--steps 50] [--warmup 10]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _odt_path  # noqa: F401,E402
from helpers import model_cfg  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout
    name, limit = [s.strip() for s in out.strip().splitlines()[0].split(",")]
    return name, limit


def event_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "classify_bench.py measures on the GPU"
    import RetinaNet
    m = RetinaNet.RetinaNet(model_cfg("retinanet", is_pretraining=True, data_shape=[a.size, a.size, 3],
                                      precision="fp16"), None)
    net = m.engine(a.batch)
    img = np.random.default_rng(0).integers(0, 256, (a.batch, a.size, a.size, 3)).astype(np.float32)
    net.image_buf.copy_(torch.from_numpy(img))
    step_ms = event_ms(net.run, a.steps, a.warmup)
    tail = net.tail
    pool_ms = event_ms(lambda: tail.launch(net, torch.cuda.current_stream().cuda_stream), a.steps * 4, a.warmup)
    f = tail.feat
    name, limit = card()
    print(json.dumps({"workload": "retinanet_pretraining_inference", "precision": "fp16", "batch": a.batch,
                      "size": a.size, "images_per_s": round(a.batch * 1000.0 / step_ms, 1),
                      "forward_ms": round(step_ms, 4), "pool_classify_ms": round(pool_ms, 5),
                      "feature": [f.H, f.W, f.C, f.ld, f.halo], "launches": net.num_launches(),
                      "gpu": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
