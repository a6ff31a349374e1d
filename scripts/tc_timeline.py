#!/usr/bin/env python
"""Per-warpgroup timeline of CTA 0 of conv_tc_kernel (debug build, -DODT_TC_TIMELINE): each consumer warpgroup's
mainloop (first MMA issue -> accumulators complete) and epilogue (-> last store issued), the mean clocks per K block
of the mainloops, and the share of the kernel during which no warpgroup has MMAs in flight, i.e. the exposed epilogue.
  --probe=feed  consumers wait for each stage and release it without MMAs: the rate the TMA feed alone sustains
  --probe=mma   the producer loads nothing and consumers do not wait: the rate of the MMAs alone (im2col mode)
Both probes compute wrong results by design.  ODT_TC_WIDE=0 / 2 pins the 128-wide / 256-wide tile of im2col layers.
conv_tc_swap.cu's kernel carries no stamps: a layer its planner takes is timed here with ODT_TC_SWAP=0 (forced below).
usage (on a GPU box): tc_timeline.py [--probe=feed|mma] B H W Cin Cout k stride [pool] [in_halo] [out_halo]
(conv_micro.py's arguments)"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
PKG = os.path.join(ROOT, "object-detection-tensorflow_b200")
sys.path.insert(0, ROOT)
sys.path.insert(0, PKG)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import __graft_entry__ as ge  # noqa: E402

EVENTS = ("mainloop start", "accumulators complete", "epilogue done")


PROBE_FLAGS = {None: [], "feed": ["-DODT_TC_PROBE_FEED"], "mma": ["-DODT_TC_PROBE_MMA"]}


def build_debug_lib(probe=None):
    ge.build()
    csrc = os.path.join(PKG, "csrc")
    obj = os.path.join(csrc, "conv_tc_tl.o")
    out = os.path.join(PKG, "odt_b200", "libodt_b200_tl.so")
    subprocess.check_call(["nvcc"] + ge.NVCC_FLAGS + ["-DODT_TC_TIMELINE"] + PROBE_FLAGS[probe] +
                          ["-c", "conv_tc.cu", "-o", obj], cwd=csrc)
    objs = [os.path.join(csrc, s[:-3] + ".o") for s in ge.SRCS if s != "conv_tc.cu"] + [obj]
    subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", out] + objs + ["-ldl"],
                          cwd=csrc)
    return out


def union_length(intervals):
    total, end = 0, None
    for a, b in sorted(intervals):
        if end is None or a > end:
            total += b - a
            end = b
        elif b > end:
            total += b - end
            end = b
    return total


def main():
    import ctypes as C
    from odt_b200 import lib as L
    argv = sys.argv[1:]
    probe = None
    if argv and argv[0].startswith("--probe="):
        probe = argv.pop(0).split("=", 1)[1]
    os.environ["ODT_TC_SWAP"] = "0"
    L.LIB_PATH = build_debug_lib(probe)
    L._lib = None  # __graft_entry__.build() has loaded the product library: bind the debug build instead
    import conv_micro
    args = [int(v) for v in argv]
    lib, launch, fl, _ = conv_micro.setup(args)
    lib.odt_debug_tc_timeline.restype = C.c_int
    lib.odt_debug_tc_timeline.argtypes = [C.c_void_p, C.c_int]
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    cap = 1 << 16
    buf = torch.zeros(2 * cap, dtype=torch.int64, device="cuda")
    L.check(lib.odt_debug_tc_timeline(buf.data_ptr(), cap), "timeline")
    launch()
    torch.cuda.synchronize()
    L.check(lib.odt_debug_tc_timeline(None, 0), "timeline off")
    raw = buf.cpu().numpy().view(np.uint64).reshape(-1, 2)
    raw = raw[raw[:, 0] != 0]
    clk = raw[:, 0].astype(np.int64)
    role = (raw[:, 1] >> np.uint64(56)).astype(int)
    ev = ((raw[:, 1] >> np.uint64(48)) & np.uint64(0xFF)).astype(int)
    tile = (raw[:, 1] & np.uint64(0xFFFFFFFF)).astype(int)
    t0, t1 = int(clk.min()), int(clk.max())
    B, H, W, Cin, Cout, k, stride = args[:7]
    kblocks = k * k * ((Cin + 63) // 64)  # im2col mode (the probes' mode)
    bn = lib.odt_conv_tc_pick_bn((Cout + 31) // 32 * 32, B * (-(-H // stride)) * (-(-W // stride)), kblocks)
    print("conv %s%s: BN %d (im2col plan), CTA 0, clocks since its first stamp; kernel span %d clk" % (
        args[:7], " probe=" + probe if probe else "", bn, t1 - t0))
    stamps = {}
    for c, r, e, t in zip(clk, role, ev, tile):
        stamps[(r, t, e)] = int(c) - t0
    busy, mains = [], []
    for g in (0, 1):
        tiles = sorted({t for (r, t, _) in stamps if r == 1 + g})
        print("-- warpgroup %d: %d tiles" % (g, len(tiles)))
        for t in tiles:
            a, b, c = (stamps.get((1 + g, t, e)) for e in range(3))
            print("tile %6d: mainloop %8s .. %8s (%6s clk)  epilogue .. %8s (%6s clk)" % (
                t, a, b, (b - a) if None not in (a, b) else "-", c, (c - b) if None not in (b, c) else "-"))
            if None not in (a, b):
                busy.append((a, b))
                mains.append(b - a)
    first = min(a for a, _ in busy) if busy else 0
    span = (t1 - t0) - first
    idle = span - union_length(busy)
    if mains:
        print("mainloop: mean %.0f clk per tile, %.0f clk per K block (%d K blocks)" % (
            np.mean(mains), np.mean(mains) / kblocks, kblocks))
    print("no warpgroup with MMAs in flight: %d of %d clk after the first mainloop start (%.1f %%)" % (
        idle, span, 100.0 * idle / max(span, 1)))


if __name__ == "__main__":
    main()
