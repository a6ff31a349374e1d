"""fp16 throughput of YOLOv3 (416², B = 64) at 1 to 9 priors per level and 20 / 80 classes: CUDA-graph replay images/s
of the whole forward (convolutions, decode, NMS), and the decode, NMS and training-loss forward kernels alone, timed
with CUDA events on the rows the network produced.  Prints the card name and power limit read in the same run, then one
JSON line per configuration.

    python scripts/prior_count_bench.py [--steps 20] [--warmup 5] [--priors 1 3 5 9] [--classes 20 80]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "object-detection-tensorflow_b200"), os.path.join(ROOT, "tests"),
          os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from class_count_bench import card, timed  # noqa: E402


def timed_after(setup, fn, steps, warmup):
    """Mean ms of fn() over `steps` calls, each preceded by setup() outside the timed window.  The NMS kernel retires
    the keys of its candidate lists in place, so every NMS launch needs the lists of a fresh decode, as in the graph."""
    for _ in range(warmup):
        setup()
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize()
    for a, b in ev:
        setup()
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in ev) / steps


def gt_boxes(rng, B, size, nc, n=16):
    """n GT boxes per image (of up to 32 slots, the rest padded with -1), sizes from 4 % of the image to all of it."""
    gt = np.full((B, 32, 5), -1.0, np.float32)
    gt[:, :n, 0:2] = rng.uniform(0.1 * size, 0.9 * size, (B, n, 2))
    gt[:, :n, 2:4] = rng.uniform(0.04 * size, 1.0 * size, (B, n, 2))
    gt[:, :n, 4] = rng.integers(0, nc, (B, n))
    return gt


def bench(A, nc, steps, warmup, thr):
    import YOLOv3
    import prior_count_ref as PR
    from helpers import model_cfg
    size, B = 416, 64
    m = YOLOv3.YOLOv3(model_cfg("yolov3", num_classes=nc, num_priors=A, priors=PR.priors_for(A), precision="fp16",
                                bn_init="trained", data_shape=[size, size, 3], nms_score_threshold=thr), None)
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (B, size, size, 3)).astype(np.float32)
    m.detect_batch(img)  # builds the engine and captures its graph
    net = m.engine(B)
    ms = timed(net.graph.replay, steps, warmup)
    st = torch.cuda.current_stream().cuda_stream
    t = net.tail
    dec = timed(lambda: t.launch_decode(net, st), steps, warmup)
    nms = timed_after(lambda: t.launch_decode(net, st), lambda: t.launch_nms(net, st), steps, warmup)
    # the training-loss forward on the same rows: scratch and GT on the device, the launches alone timed
    gt = torch.from_numpy(gt_boxes(rng, B, size, nc)).to(net.device)
    p = ctypes.byref(t.p)
    scratch = torch.zeros((net.lib.odt_yolo_loss_scratch_bytes(p, B) + 7) // 8, dtype=torch.int64, device=net.device)
    out = torch.zeros(B, dtype=torch.float32, device=net.device)

    def loss():
        rc = net.lib.odt_yolo_loss_fwd(net.head_buf.data_ptr(), p, B, gt.data_ptr(), gt.shape[1], 1.0, 1.0, 5.0, 1.0,
                                       scratch.data_ptr(), out.data_ptr(), st)
        assert rc == 0, net.lib.odt_last_error()
    lfwd = timed(loss, steps, warmup)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    cc = t.cand_count.cpu().numpy()
    return {"model": "yolov3", "priors": A, "classes": nc, "input": size, "batch": B, "rows_per_image": net.N,
            "score_threshold": thr, "graph_ms": round(ms, 3), "images_per_s": round(B / ms * 1e3, 1),
            "decode_ms": round(dec, 4), "nms_ms": round(nms, 4), "loss_fwd_ms": round(lfwd, 4),
            "candidates_per_class_mean": round(float(cc.mean()), 1), "detections": int(t.det_count.sum().item())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--priors", type=int, nargs="+", default=[1, 3, 5, 9])
    ap.add_argument("--classes", type=int, nargs="+", default=[20, 80])
    ap.add_argument("--thr", type=float, default=0.05)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    print(json.dumps({"card": card()}))
    for nc in a.classes:
        for A in a.priors:
            print(json.dumps(bench(A, nc, a.steps, a.warmup, a.thr)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
