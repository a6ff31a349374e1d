#!/usr/bin/env python
"""One tensor-core conv in isolation (for A-B timing with CUDA events).
usage: conv_micro.py B H W Cin Cout k stride [pool] [in_halo] [out_halo] [reps]"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "object-detection-tensorflow_b200"))
from odt_b200 import lib as L  # noqa: E402
from odt_b200.engine import same_pad  # noqa: E402


def main():
    a = [int(v) for v in sys.argv[1:]]
    B, H, W, Cin, Cout, k, stride = a[:7]
    pool = a[7] if len(a) > 7 else 0
    ih = a[8] if len(a) > 8 else 1
    oh = a[9] if len(a) > 9 else 1
    reps = a[10] if len(a) > 10 else 20
    lib = L.load()
    ld = (Cin + 63) // 64 * 64
    old = (Cout + 63) // 64 * 64
    cpad = (Cout + 31) // 32 * 32
    OH, pt, _ = same_pad(H, k, stride)
    OW, pl, _ = same_pad(W, k, stride)
    x = torch.zeros((B, H + 2 * ih, W + 2 * ih, ld), dtype=torch.float16, device="cuda")
    x[:, ih:ih + H, ih:ih + W, :Cin] = torch.randn((B, H, W, Cin), device="cuda").half()
    w = torch.zeros((cpad, k, k, ld), dtype=torch.float16, device="cuda")
    w[:Cout, :, :, :Cin] = (torch.randn((Cout, k, k, Cin), device="cuda") * (2.0 / (k * k * Cin)) ** 0.5).half()
    yh, yw = (OH // 2, OW // 2) if pool else (OH, OW)
    y = torch.zeros((B, yh + 2 * oh, yw + 2 * oh, old), dtype=torch.float16, device="cuda")
    shift = torch.zeros(Cout, device="cuda")
    p = L.ConvParams()
    p.B, p.H, p.W, p.Cin, p.in_ld = B, H, W, Cin, ld
    p.OH, p.OW, p.Cout = OH, OW, Cout
    p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = k, k, stride, 1, pt, pl
    p.w_ld, p.Cout_pad = ld, cpad
    p.shift, p.act = shift.data_ptr(), 1
    p.out0, p.out0_dtype = y.data_ptr(), L.ODT_F16
    p.out0_img_stride, p.out0_pix_stride = (yh + 2 * oh) * (yw + 2 * oh) * old, old
    p.in_halo, p.out0_halo, p.out0_pool = ih, oh, pool
    # ODT_MICRO_EXTRA = "r" (residual) / "1" (second output) / "2" (third output) / "n" (no out0), any combination:
    # the epilogue variants of RetinaNet's bottleneck 1x1 convolutions
    extra = os.environ.get("ODT_MICRO_EXTRA", "")
    keep = []
    if "r" in extra:
        keep.append(torch.randn(y.shape, device="cuda").half())
        p.residual = keep[-1].data_ptr()
    for tag, pre in (("1", "1"), ("2", "2")):
        if tag in extra:
            t = torch.zeros((B, OH, OW, old), dtype=torch.float16, device="cuda")
            sc, sh = torch.ones(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
            keep += [t, sc, sh]
            if pre == "1":
                p.scale2, p.shift2, p.act2 = sc.data_ptr(), sh.data_ptr(), 1
                p.out1, p.out1_img_stride, p.out1_pix_stride = t.data_ptr(), OH * OW * old, old
            else:
                p.scale3, p.shift3, p.act3 = sc.data_ptr(), sh.data_ptr(), 1
                p.out2, p.out2_img_stride, p.out2_pix_stride = t.data_ptr(), OH * OW * old, old
    if "n" in extra:
        p.out0 = None
    st = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        L.check(lib.odt_conv2d_f16_tc(x.data_ptr(), w.data_ptr(), C.byref(p), st), "conv")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        L.check(lib.odt_conv2d_f16_tc(x.data_ptr(), w.data_ptr(), C.byref(p), st), "conv")
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    fl = 2.0 * B * OH * OW * Cout * k * k * Cin
    print("conv %s pool=%d halo=%d/%d extra=%r thin/tapn launches %d/%d: %.4f ms  %.1f TFLOP/s" % (
        a[:7], pool, ih, oh, extra, lib.odt_debug_thin_launches(), lib.odt_debug_tapn_launches(), ms, fl / ms / 1e9))


if __name__ == "__main__":
    main()
