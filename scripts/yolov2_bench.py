"""YOLOv2 inference rate on one GPU: fp16 CUDA-graph replay of the whole network + decode + NMS at 480², B = 64,
20 classes, 5 priors (testYOLOv2.py's configuration), and the decode, NMS and loss-and-gradient kernels timed alone by
CUDA events.  The card's name and power limit are read in the same run and printed with the numbers; the achieved
rate is reported against the convolution FLOPs counted from the layer shapes.

    python scripts/yolov2_bench.py [--batch 64] [--size 480] [--steps 50] [--warmup 10]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__  # noqa: E402,F401  (puts the package on sys.path)

PRIORS = [[1.08, 1.19], [3.42, 4.41], [6.63, 11.38], [9.42, 5.11], [16.62, 10.52]]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        power = out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def events_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=480)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("yolov2_bench needs a GPU")
    import YOLOv2
    from odt_b200 import lib as L
    cfg = {"mode": "test", "data_format": "channels_last", "num_classes": 20, "weight_decay": 1e-4, "keep_prob": 0.5,
           "batch_size": 1, "nms_score_threshold": 0.5, "nms_max_boxes": 10, "nms_iou_threshold": 0.5,
           "pretraining_weight": None, "data_shape": [args.size, args.size, 3], "coord_scale": 1, "noobj_scale": 1,
           "obj_scale": 5., "class_scale": 1., "rescore_confidence": False, "priors": PRIORS, "bn_init": "trained",
           "precision": "fp16"}
    m = YOLOv2.YOLOv2(cfg, None)
    B = args.batch
    net = m.engine(B)
    img = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (B, args.size, args.size, 3)).astype(np.float32))
    net.image_buf.copy_(img)
    for _ in range(args.warmup):
        net.run()
    torch.cuda.synchronize()
    step_ms = events_ms(net.run, args.steps)
    ips = B / (step_ms / 1e3)
    flops = net.conv_flops / B

    st = torch.cuda.current_stream().cuda_stream
    tail = net.tail
    decode_ms = events_ms(lambda: tail.launch_decode(net, st), args.steps)
    nms_ms = events_ms(lambda: (tail.launch_decode(net, st), tail.launch_nms(net, st)), args.steps) - decode_ms
    gt = np.full((B, 60, 5), -1.0, np.float32)  # pad_truth_to 60 (testYOLOv2.py:61)
    rng = np.random.default_rng(1)
    for b in range(B):
        n = 1 + b % 8
        gt[b, :n, 0:2] = rng.uniform(20, args.size - 20, (n, 2))
        gt[b, :n, 2:4] = rng.uniform(16, args.size / 2, (n, 2))
        gt[b, :n, 4] = rng.integers(0, 20, n)
    gtd = torch.from_numpy(gt).cuda()
    p = C.byref(tail.p)
    nbytes = net.lib.odt_yolo2_loss_scratch_bytes(p, B)
    scratch = torch.zeros((nbytes + 7) // 8, dtype=torch.int64, device="cuda")
    loss = torch.zeros(B, dtype=torch.float32, device="cuda")
    grad = torch.empty_like(net.head_buf)

    def loss_grad():
        L.check(net.lib.odt_yolo2_loss_grad(net.head_buf.data_ptr(), p, B, gtd.data_ptr(), 60, 1.0, 1.0, 5.0, 1.0,
                                            scratch.data_ptr(), loss.data_ptr(), grad.data_ptr(), st), "yolo2_loss_grad")
    for _ in range(args.warmup):
        loss_grad()
    loss_ms = events_ms(loss_grad, args.steps)
    name, power = card()
    res = {"model": "YOLOv2", "size": args.size, "batch": B, "precision": "fp16", "classes": 20, "priors": 5,
           "images_per_s": round(ips, 1), "step_ms": round(step_ms, 3), "conv_gflop_per_image": round(flops / 1e9, 2),
           "achieved_conv_tflops": round(flops * ips / 1e12, 1), "decode_ms": round(decode_ms, 4),
           "nms_ms": round(nms_ms, 4), "loss_grad_ms": round(loss_ms, 4), "launches": net.num_launches(),
           "card": name, "power_limit_and_max_sm_clock": power}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
