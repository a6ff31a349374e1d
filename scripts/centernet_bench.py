"""CenterNet on one GPU: fp16 CUDA-graph replay of the whole network + peak / top-k tail at 384² (testcenternet.py's
size) for B = 15 (its batch) and B = 64, the tail and the loss-and-gradient kernels timed alone by CUDA events, and one
fp32 training step (the engine's layer list replayed with autograd, the loss from the kernels, Adam) at B = 15.  The
card's name and power limit are read in the same run and printed with the numbers.  Convolution FLOPs are counted from
the layer shapes as the reference defines them (4x4 transposed convolutions, real channel counts).

    python scripts/centernet_bench.py [--steps 50] [--warmup 10]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import __graft_entry__  # noqa: E402,F401  (puts the package on sys.path)
from pfpnet_bench import DENSE_FP16_TFLOPS, model_flops_per_image  # noqa: E402
from yolov2_bench import card, events_ms  # noqa: E402

CFG = {"mode": "test", "data_format": "channels_last", "num_classes": 20, "weight_decay": 1e-4, "keep_prob": 0.5,
       "batch_size": 15, "score_threshold": 0.1, "top_k_results_output": 100, "input_size": 384, "bn_init": "trained",
       "precision": "fp16"}


def ground_truth(B, size, seed=1):
    gt = np.full((B, 60, 5), -1.0, np.float32)
    rng = np.random.default_rng(seed)
    for b in range(B):
        n = 1 + b % 8
        gt[b, :n, 0:2] = rng.uniform(20, size - 20, (n, 2))
        gt[b, :n, 2:4] = rng.uniform(16, size / 2, (n, 2))
        gt[b, :n, 4] = rng.integers(0, 20, n)
    return gt


def run(B, steps, warmup):
    import CenterNet
    from odt_b200 import lib as L
    size = CFG["input_size"]
    m = CenterNet.CenterNet(dict(CFG), None)
    net = m.engine(B)
    img = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (B, size, size, 3)).astype(np.float32))
    net.image_buf.copy_(img)
    for _ in range(warmup):
        net.run()
    torch.cuda.synchronize()
    step_ms = events_ms(net.run, steps)
    ips = B / (step_ms / 1e3)
    flops = model_flops_per_image(net)
    st = torch.cuda.current_stream().cuda_stream
    tail = net.tail
    tail_ms = events_ms(lambda: tail.launch(net, st), steps)
    gtd = torch.from_numpy(ground_truth(B, size)).cuda()
    p = C.byref(tail.p)
    scratch = torch.zeros((net.lib.odt_centernet_loss_scratch_bytes(p, B) + 7) // 8, dtype=torch.int64, device="cuda")
    loss = torch.zeros(B, dtype=torch.float32, device="cuda")
    grad = torch.empty_like(net.head_buf)

    def loss_grad():
        L.check(net.lib.odt_centernet_loss_grad(net.head_buf.data_ptr(), p, B, gtd.data_ptr(), 60, scratch.data_ptr(),
                                                loss.data_ptr(), grad.data_ptr(), st), "centernet_loss_grad")
    for _ in range(warmup):
        loss_grad()
    loss_ms = events_ms(loss_grad, steps)
    achieved = flops * ips / 1e12
    return {"model": "CenterNet", "size": size, "batch": B, "precision": "fp16", "images_per_s": round(ips, 1),
            "step_ms": round(step_ms, 3), "conv_gflop_per_image": round(flops / 1e9, 2),
            "achieved_conv_tflops": round(achieved, 1),
            "share_of_dense_fp16_datasheet": round(achieved / DENSE_FP16_TFLOPS, 3),
            "tail_ms": round(tail_ms, 4), "loss_grad_ms": round(loss_ms, 4), "launches": net.num_launches()}


def train_step_ms(B, steps=5):
    """Wall time of GraphTrainer.step (fp32 forward and backward in PyTorch, the loss from the kernels, Adam)."""
    import CenterNet
    size = CFG["input_size"]
    m = CenterNet.CenterNet(dict(CFG, mode="test"), None)
    tr = m.trainer()
    img = np.random.default_rng(2).integers(0, 256, (B, size, size, 3)).astype(np.float32)
    gt = ground_truth(B, size, 3)
    tr.step(img, gt, 1e-4)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        tr.step(img, gt, 1e-4)  # returns the loss as a Python float: the step ends in a device synchronise
    return (time.perf_counter() - t) / steps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("centernet_bench needs a GPU")
    name, power = card()
    for B in (15, 64):
        res = run(B, args.steps, args.warmup)
        res.update(card=name, power_limit_and_max_sm_clock=power)
        print(json.dumps(res))
    print(json.dumps({"model": "CenterNet", "size": CFG["input_size"], "batch": 15, "precision": "fp32",
                      "train_step_ms": round(train_step_ms(15), 1), "card": name,
                      "power_limit_and_max_sm_clock": power}))


if __name__ == "__main__":
    main()
