#!/usr/bin/env python
"""RetinaNet with basic-block ResNets (is_bottleneck=False, init_conv_filters=7) on one GPU, fp16:
  * detection at 800^2, B=16: images/s of the captured forward (convolutions, decode, NMS);
  * pretraining-mode inference at 224^2, B=256: images/s of the captured forward (convolutions, pooled logits);
  * the 7x7/2 stem of the detection engine alone (CUDA events): the packed-RGBX tensor-core stem (image pack +
    odt_conv2d_stem_rgbx, 16 computed outputs) against the fp32-gather stem (odt_conv2d_stem) on the same 7 outputs.
The card's name and power limit are read in the same run.  Prints one JSON line.
usage: basic_block_bench.py [--blocks 3,4,6,3] [--steps 30] [--warmup 5]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _odt_path  # noqa: F401,E402
from classify_bench import card, event_ms  # noqa: E402
from helpers import model_cfg  # noqa: E402


def model(blocks, size, pretraining):
    import RetinaNet
    return RetinaNet.RetinaNet(model_cfg("retinanet", is_bottleneck=False, init_conv_filters=7,
                                         residual_block_list=blocks, is_pretraining=pretraining,
                                         data_shape=[size, size, 3], precision="fp16"), None)


def forward_ms(blocks, size, batch, pretraining, steps, warmup):
    m = model(blocks, size, pretraining)
    net = m.engine(batch)
    img = np.random.default_rng(0).integers(0, 256, (batch, size, size, 3)).astype(np.float32)
    net.image_buf.copy_(torch.from_numpy(img))
    return net, event_ms(net.run, steps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", default="3,4,6,3")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "basic_block_bench.py measures on the GPU"
    from odt_b200 import lib as L
    blocks = [int(b) for b in a.blocks.split(",")]
    net, det_ms = forward_ms(blocks, 800, 16, False, a.steps, a.warmup)
    stem = net.ops[0]
    assert stem.is_image and stem.rgbx == 4, "the packed stem is expected on this shape"
    st = torch.cuda.current_stream().cuda_stream
    packed_ms = event_ms(lambda: stem.launch(net, st), a.steps * 4, a.warmup)
    # the fp32-gather stem on the same image, weights (first 7 of the 16 uploaded rows) and output
    p = L.ConvParams()
    C.memmove(C.byref(p), C.byref(stem.p), C.sizeof(p))
    p.in_ld, p.in_halo, p.Cout_pad = 3, 0, 7

    def gather():
        L.check(net.lib.odt_conv2d_stem(net.image_buf.data_ptr(), net.mean3, stem.wdev.data_ptr(), L.ODT_F16,
                                        C.byref(p), st), "stem")
    gather_ms = event_ms(gather, a.steps * 4, a.warmup)
    _, pre_ms = forward_ms(blocks, 224, 256, True, a.steps, a.warmup)
    name, limit = card()
    print(json.dumps({"workload": "retinanet_basic_block", "blocks": blocks, "precision": "fp16",
                      "detection_800_b16_images_per_s": round(16 * 1000.0 / det_ms, 1),
                      "detection_800_b16_forward_ms": round(det_ms, 4),
                      "pretraining_224_b256_images_per_s": round(256 * 1000.0 / pre_ms, 1),
                      "pretraining_224_b256_forward_ms": round(pre_ms, 4),
                      "stem_800_b16_packed_rgbx_ms": round(packed_ms, 4),
                      "stem_800_b16_fp32_gather_ms": round(gather_ms, 4),
                      "gpu": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
