"""PFPNet-R inference rate on one GPU: fp16 CUDA-graph replay of the whole network + decode + NMS at 320², B = 64 and
at 512², B = 16 (testpfpnet.py's two sizes), and the decode and NMS kernels timed alone by CUDA events.  The card's
name and power limit are read in the same run and printed with the numbers.  The convolution FLOPs are counted from
the layer shapes with the real channel counts (767-channel concats, 4x4 transposed convolutions as the reference
defines them), not from what the padded layouts and the phase convolutions execute.  The loss-and-gradient kernel
(odt_pfpnet_loss_grad) is timed on the network's own rows with 1 to 8 boxes per image.

    python scripts/pfpnet_bench.py [--steps 50] [--warmup 10]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import __graft_entry__  # noqa: E402,F401  (puts the package on sys.path)
from yolov2_bench import card, events_ms  # noqa: E402

DENSE_FP16_TFLOPS = 989.0  # H100 SXM data sheet, dense FP16, at up to 700 W


def model_flops_per_image(net):
    """Multiply-adds x 2 of every convolution as the reference defines it, per image."""
    from odt_b200 import engine as E
    total = 0
    for op in net.ops:
        if not isinstance(op, E.ConvOp):
            continue
        shape = net.vars[op.kernel][0]
        if isinstance(op, E.PhaseConvOp):  # [4, 4, cout, cin]: 4 taps per output pixel of the 2x grid
            cout, cin = shape[2], shape[3]
            total += 2 * (2 * op.x.H) * (2 * op.x.W) * cout * cin * 4
        else:
            k, _, cin, cout = shape
            oh, ow = op.out_hw
            total += 2 * oh * ow * cout * k * k * cin
    return total


def run(size, B, steps, warmup):
    import PFPNetR
    from odt_b200 import lib as L
    cfg = {"mode": "test", "data_format": "channels_last", "num_classes": 20, "weight_decay": 1e-4, "keep_prob": 0.5,
           "batch_size": 1, "nms_score_threshold": 0.5, "nms_max_boxes": 20, "nms_iou_threshold": 0.5,
           "pretraining_weight": None, "input_size": size, "bn_init": "trained", "precision": "fp16"}
    m = PFPNetR.PFPNetR(cfg, None)
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
    decode_ms = events_ms(lambda: tail.launch_decode(net, st), steps)
    nms_ms = events_ms(lambda: (tail.launch_decode(net, st), tail.launch_nms(net, st)), steps) - decode_ms
    gt = np.full((B, 60, 5), -1.0, np.float32)
    rng = np.random.default_rng(1)
    for b in range(B):
        n = 1 + b % 8
        gt[b, :n, 0:2] = rng.uniform(20, size - 20, (n, 2))
        gt[b, :n, 2:4] = rng.uniform(16, size / 2, (n, 2))
        gt[b, :n, 4] = rng.integers(0, 20, n)
    gtd = torch.from_numpy(gt).cuda()
    p = C.byref(tail.p)
    scratch = torch.zeros((net.lib.odt_pfpnet_loss_scratch_bytes(p, B) + 7) // 8, dtype=torch.int64, device="cuda")
    loss = torch.zeros(B, dtype=torch.float32, device="cuda")
    grad = torch.empty_like(net.head_buf)

    def loss_grad():
        L.check(net.lib.odt_pfpnet_loss_grad(net.head_buf.data_ptr(), p, B, gtd.data_ptr(), 60, scratch.data_ptr(),
                                             loss.data_ptr(), grad.data_ptr(), st), "pfpnet_loss_grad")
    for _ in range(warmup):
        loss_grad()
    loss_ms = events_ms(loss_grad, steps)
    achieved = flops * ips / 1e12
    return {"model": "PFPNetR", "size": size, "batch": B, "precision": "fp16", "images_per_s": round(ips, 1),
            "step_ms": round(step_ms, 3), "conv_gflop_per_image": round(flops / 1e9, 2),
            "achieved_conv_tflops": round(achieved, 1),
            "share_of_dense_fp16_datasheet": round(achieved / DENSE_FP16_TFLOPS, 3),
            "decode_ms": round(decode_ms, 4), "nms_ms": round(nms_ms, 4), "loss_grad_ms": round(loss_ms, 4),
            "launches": net.num_launches()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pfpnet_bench needs a GPU")
    name, power = card()
    for size, B in ((320, 64), (512, 16)):
        res = run(size, B, args.steps, args.warmup)
        res.update(card=name, power_limit_and_max_sm_clock=power)
        print(json.dumps(res))


if __name__ == "__main__":
    main()
