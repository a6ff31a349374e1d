"""fp16 throughput of YOLOv3 (416², B = 64) and FCOS (1024², B = 16) at 20 and 80 classes: CUDA-graph replay
images/s of the whole forward (convolutions, decode, NMS), and the decode and NMS kernels alone, timed with CUDA events
on the rows the network produced.  Prints the card name and power limit read in the same run, then one JSON line per
configuration.

    python scripts/class_count_bench.py [--steps 20] [--warmup 5] [--classes 20 80]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "object-detection-tensorflow_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return {"name": name, "nvidia_smi": out}
    except (OSError, subprocess.SubprocessError):
        return {"name": name, "nvidia_smi": None}


def timed(fn, steps, warmup):
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


def bench(family, nc, steps, warmup, thr):
    import FCOS
    import YOLOv3
    from helpers import model_cfg
    size, B = (416, 64) if family == "yolov3" else (1024, 16)
    cls = YOLOv3.YOLOv3 if family == "yolov3" else FCOS.FCOS
    m = cls(model_cfg(family, num_classes=nc, precision="fp16", bn_init="trained", data_shape=[size, size, 3],
                      nms_score_threshold=thr), None)
    img = np.random.default_rng(0).integers(0, 256, (B, size, size, 3)).astype(np.float32)
    m.detect_batch(img)  # builds the engine and captures its graph
    net = m.engine(B)
    ms = timed(net.graph.replay, steps, warmup)
    st = torch.cuda.current_stream().cuda_stream
    t = net.tail
    dec = timed(lambda: t.launch_decode(net, st), steps, warmup)
    nms = timed(lambda: t.launch_nms(net, st), steps, warmup)  # the lists of the last decode, as in the graph
    torch.cuda.synchronize()
    cc = t.cand_count.cpu().numpy()
    return {"model": family, "classes": nc, "input": size, "batch": B, "score_threshold": thr, "graph_ms": round(ms, 3),
            "images_per_s": round(B / ms * 1e3, 1), "decode_ms": round(dec, 4), "nms_ms": round(nms, 4),
            "candidates_per_class_mean": round(float(cc.mean()), 1), "detections": int(t.det_count.sum().item())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--classes", type=int, nargs="+", default=[20, 80])
    ap.add_argument("--models", nargs="+", default=["yolov3", "fcos"])
    # random-init FCOS scores sit near sigmoid(-4.6)^2 = 1e-4 (the 'pi' bias init of both heads): a threshold of 5e-5
    # gives its NMS work, as 0.05 does for YOLOv3
    ap.add_argument("--thr", type=float, nargs=2, default=[0.05, 5e-5], metavar=("YOLO", "FCOS"))
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    for family in a.models:
        for nc in a.classes:
            thr = a.thr[0] if family == "yolov3" else a.thr[1]
            print(json.dumps(bench(family, nc, a.steps, a.warmup, thr)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
