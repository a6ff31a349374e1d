#!/usr/bin/env python
"""odt_groupnorm_act at the GroupNorm geometries of FCOS-1024 (B = 4 per GPU, fp16): CUDA-event time per launch pair,
and its accuracy / batch invariance at |mean|/sigma = 100 (fp32), optionally against a libodt_b200.so built from an
earlier commit (--baseline-lib; its odt_groupnorm_act takes B*groups*2 caller-zeroed doubles).  The two libraries are
timed in the same process, alternating rounds.  Also lists the GroupNorm ops of SSD300 / RetinaNet (none expected:
bench.py runs those two).
usage: gn_micro.py [--baseline-lib PATH] [--reps 200] [--rounds 5]"""
import argparse
import ctypes as C
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
from odt_b200 import lib as L  # noqa: E402
from odt_b200 import engine as E  # noqa: E402

EPS = 1e-6


def spec_ops(kind, B, precision="fp16"):
    import FCOS
    import RetinaNet
    import SSD300
    m = {"fcos": lambda: FCOS.FCOS(model_cfg("fcos", data_shape=[1024, 1024, 3]), None),
         "retinanet": lambda: RetinaNet.RetinaNet(model_cfg("retinanet", data_shape=[800, 800, 3]), None),
         "ssd300": lambda: SSD300.SSD300(model_cfg("ssd"), None)}[kind]()
    E.Net.spec_only = True
    try:
        net, _ = m._build(B, precision, True)
    finally:
        E.Net.spec_only = False
    return net.ops


class Impl:
    def __init__(self, name, lib, new):
        self.name, self.lib, self.new = name, lib, new

    def workspace(self, dt, B, hw, Cc, groups):
        n = (self.lib.odt_groupnorm_act_workspace_bytes(dt, B, hw, Cc, groups) + 7) // 8 if self.new else B * groups * 2
        return torch.zeros(max(n, 1), dtype=torch.float64, device="cuda")

    def run(self, x, y, ws, dt, B, hw, Cc, ld, groups, g, b, act=1):
        return self.lib.odt_groupnorm_act(x.data_ptr(), y.data_ptr(), ws.data_ptr(), dt, B, hw, Cc, ld, groups, EPS,
                                          g.data_ptr(), b.data_ptr(), act, torch.cuda.current_stream().cuda_stream)


def load_baseline(path):
    lib = C.CDLL(path)
    f = lib.odt_groupnorm_act
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_int,
                  C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    return lib


def accuracy(impls):
    """fp32, C = 256, groups = 8, B = 4, hw = 64^2, x = +-100 + N(0, 1): rstd-relative error of the output against
    float64 two-pass moments, and image 0 alone vs its slice of the batch."""
    B, H, W, Cc, groups = 4, 64, 64, 256, 8
    g = torch.Generator(device="cuda").manual_seed(0)
    sign = torch.tensor([1.0, -1.0, 1.0, -1.0], device="cuda").view(B, 1, 1, 1)
    x = torch.randn((B, H, W, Cc), generator=g, device="cuda") + 100.0 * sign
    gamma = torch.ones(Cc, device="cuda")
    beta = torch.zeros(Cc, device="cuda")
    xg = x.double().reshape(B, H * W, groups, -1)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(((xg - mean) ** 2).mean(dim=(1, 3), keepdim=True) + float(np.float32(EPS)))
    ref = ((xg - mean) * rstd).reshape(x.shape)
    for im in impls:
        y = torch.zeros_like(x)
        ws = im.workspace(L.ODT_F32, B, H * W, Cc, groups)
        L.check(im.run(x, y, ws, L.ODT_F32, B, H * W, Cc, Cc, groups, gamma, beta, act=0))
        y1 = torch.zeros_like(x[:1])
        ws1 = im.workspace(L.ODT_F32, 1, H * W, Cc, groups)
        x1 = x[:1].clone()
        L.check(im.run(x1, y1, ws1, L.ODT_F32, 1, H * W, Cc, Cc, groups, gamma, beta, act=0))
        torch.cuda.synchronize()
        err = float((y.double() - ref).abs().max())  # = rstd-relative error x |x - mean| / sigma, |x-mean| ~ 4 sigma
        print("accuracy %-8s fp32 |mean|/sigma=100: max|y - y_ref| = %.3g (fp32 bar in tests/test_gpu_glue.py: "
              "~2e-5 at |x - mean| = 4 sigma); image 0 alone == its slice of B=4: %s"
              % (im.name, err, bool(torch.equal(y1[0], y[0]))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    for kind, B in (("ssd300", 64), ("retinanet", 16)):
        n = sum(isinstance(op, E.GroupNormActOp) for op in spec_ops(kind, B))
        print("%s B=%d: %d GroupNormActOp" % (kind, B, n))
    assert torch.cuda.is_available(), "gn_micro.py times kernels on the GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q[0] if q else "n/a"))
    impls = [Impl("new", L.load(), True)]
    if a.baseline_lib:
        impls.insert(0, Impl("baseline", load_baseline(a.baseline_lib), False))
    accuracy(impls)

    geoms = {}
    for op in spec_ops("fcos", 4):
        if isinstance(op, E.GroupNormActOp):
            k = (op.x.B, op.x.H, op.x.W, op.x.C, op.x.ld, op.groups)
            geoms[k] = geoms.get(k, 0) + 1
    print("FCOS-1024 B=4 fp16: %d GroupNorm ops, %d geometries" % (sum(geoms.values()), len(geoms)))
    tot = {im.name: 0.0 for im in impls}
    for (B, H, W, Cc, ld, groups), count in sorted(geoms.items(), key=lambda kv: -kv[0][1] * kv[0][2] * kv[0][3]):
        hw = H * W
        x = (torch.randn((B, H, W, ld), device="cuda") + 3.0).half()
        y = torch.empty_like(x)
        gamma, beta = torch.rand(Cc, device="cuda") + 0.5, torch.randn(Cc, device="cuda")
        ws = {im.name: im.workspace(L.ODT_F16, B, hw, Cc, groups) for im in impls}
        times = {im.name: [] for im in impls}
        for im in impls:  # warm-up
            for _ in range(10):
                L.check(im.run(x, y, ws[im.name], L.ODT_F16, B, hw, Cc, ld, groups, gamma, beta))
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for im in impls:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    im.run(x, y, ws[im.name], L.ODT_F16, B, hw, Cc, ld, groups, gamma, beta)
                e1.record()
                e1.synchronize()
                times[im.name].append(e0.elapsed_time(e1) * 1e3 / a.reps)
        nbytes = 3 * B * hw * ld * 2  # the statistics read the tensor once, the apply reads and writes it
        line = "B=%d %4dx%-4d C=%4d groups=%d x%-2d" % (B, H, W, Cc, groups, count)
        for im in impls:
            t = float(np.median(times[im.name]))
            tot[im.name] += t * count
            line += " | %s %7.2f us (%4.0f GB/s, rounds %s)" % (im.name, t, nbytes / t / 1e3,
                                                               " ".join("%.1f" % v for v in times[im.name]))
        print(line)
    print("sum over the FCOS GroupNorm ops: " + ", ".join("%s %.1f us" % (k, v) for k, v in tot.items()))


if __name__ == "__main__":
    main()
