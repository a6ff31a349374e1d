#!/usr/bin/env python
"""Per-round timeline of block (0, 0) of nms_per_class_kernel (debug build, -DODT_NMS_TIMELINE): where a greedy
round's latency goes (round top -> arg-max barrier -> suppression barrier), on one model's real head rows.
Also times the kernel (CUDA graph, 50 replays).
usage (on a GPU box): nms_timeline.py model batch"""
import ctypes as C
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


def build_debug_lib():
    ge.build()
    csrc = os.path.join(PKG, "csrc")
    obj = os.path.join(csrc, "tail_tl.o")
    out = os.path.join(PKG, "odt_b200", "libodt_b200_nmstl.so")
    subprocess.check_call(["nvcc"] + ge.NVCC_FLAGS + ["-DODT_NMS_TIMELINE", "-c", "tail.cu", "-o", obj], cwd=csrc)
    objs = [os.path.join(csrc, s[:-3] + ".o") for s in ge.SRCS if s != "tail.cu"] + [obj]
    subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", out] + objs + ["-ldl"],
                          cwd=csrc)
    return out


def main():
    from odt_b200 import lib as L
    L.LIB_PATH = build_debug_lib()
    L._lib = None  # __graft_entry__.build() has loaded the product library: bind the debug build instead
    lib = L.load()
    import tail_micro
    name, B = sys.argv[1], int(sys.argv[2])
    m, net = tail_micro.build_model(name, B)
    net.forward()
    torch.cuda.synchronize()
    t = net.tail
    st = torch.cuda.current_stream().cuda_stream

    def decode():
        L.check(lib.odt_decode_candidates(net.head_buf.data_ptr(), C.byref(t.p), net.batch, t.cand_keys.data_ptr(),
                                          t.cand_count.data_ptr(), torch.cuda.current_stream().cuda_stream))

    def nms():
        L.check(lib.odt_nms_per_class(net.head_buf.data_ptr(), C.byref(t.p), net.batch, t.cand_keys.data_ptr(),
                                      t.cand_count.data_ptr(), t.dets.data_ptr(), t.det_anchor.data_ptr(),
                                      t.det_count.data_ptr(), t.scratch.data_ptr(), t.work.data_ptr(),
                                      t.status.data_ptr(), t.box_pool.data_ptr() if t.box_pool is not None else None,
                                      t.pool_entries, t.rec.shape[1], torch.cuda.current_stream().cuda_stream))

    cnt = t.cand_count.cpu().numpy().reshape(B, -1)
    print("%s B=%d: candidates per list mean %.0f max %d ; list (0,0): %d" % (name, B, cnt.mean(), cnt.max(), cnt[0, 0]))
    lib.odt_debug_nms_timeline.restype = C.c_int
    lib.odt_debug_nms_timeline.argtypes = [C.c_void_p, C.c_int]
    cap = 4096
    for _ in range(3):
        decode(); nms()
    torch.cuda.synchronize()
    buf = torch.zeros(2 * cap, dtype=torch.int64, device="cuda")
    L.check(lib.odt_debug_nms_timeline(buf.data_ptr(), cap), "timeline")
    decode(); nms()
    torch.cuda.synchronize()
    L.check(lib.odt_debug_nms_timeline(None, 0), "timeline off")
    raw = buf.cpu().numpy().view(np.uint64).reshape(-1, 2)
    raw = raw[raw[:, 0] != 0]
    ev = (raw[:, 1] >> np.uint64(32)).astype(int)
    rnd = (raw[:, 1] & np.uint64(0xFFFFFFFF)).astype(int)
    t0 = int(raw[:, 0].min()) if len(raw) else 0
    print("-- block (0,0), clk since its first stamp (round top / after arg-max barrier / after suppression barrier)")
    rows = {}
    for (clk, _), e, r in zip(raw, ev, rnd):
        rows.setdefault((r, e), int(clk) - t0)
    rounds = sorted({r for r, _ in rows})
    prev = None
    for r in rounds:
        a, b, c = rows.get((r, 0)), rows.get((r, 1)), rows.get((r + 1, 2))
        line = "round %2d: top %7s  argmax +%5s  suppress +%5s" % (
            r, a, (b - a) if (a is not None and b is not None) else "-", (c - b) if (b is not None and c is not None) else "-")
        if prev is not None and a is not None:
            line += "   (round %d total %d clk)" % (r - 1, a - prev)
        prev = a
        print(line)
    # warm graph timing of the NMS launch alone
    g = torch.cuda.CUDAGraph()
    decode()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        for _ in range(50):
            nms()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); e1.record()
    torch.cuda.synchronize()
    print("   nms (2 memsets + kernel), graph of 50: %.2f us per launch" % (e0.elapsed_time(e1) / 50 * 1e3))


if __name__ == "__main__":
    main()
