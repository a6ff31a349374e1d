"""The thin-layer kernel's OWN source (csrc/conv_thin.cu: thin_fill / thin_pixel are __host__ __device__) executed
on the CPU through a test-only harness (tests/native/thin_host.cu, built here with nvcc) and compared with the
oracle's TF-SAME convolution + the epilogue chain of epilogue.cuh: index arithmetic (halo / no halo, stride 2),
fp16 rounding order, residual, the two extra pre-activated outputs, untouched padding lanes and halo ring.
The device launch itself still needs an H100 (tests/test_gpu_conv.py::test_conv_thin_matches_reference)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import tfops as T

HERE = os.path.dirname(os.path.abspath(__file__))


def build_host_harness(name, kernel_src, entry):
    """nvcc-build tests/native/<name>.cu (which #includes the kernel source) and bind its entry point."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(HERE, "native", name + ".cu")
    out_dir = os.path.join(HERE, "native", "_build")
    os.makedirs(out_dir, exist_ok=True)
    out = os.path.join(out_dir, "lib%s.so" % name)
    csrc = os.path.join(HERE, "..", "object-detection-tensorflow_b200", "csrc")
    deps = [src, os.path.join(csrc, kernel_src), os.path.join(csrc, "epilogue.cuh"), os.path.join(csrc, "common.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(f) > os.path.getmtime(out) for f in deps):
        # -fno-strict-aliasing: the kernel reinterprets uint4 registers as __half2 (fine for nvcc's device code,
        # undefined behaviour for the host compiler's optimiser)
        subprocess.check_call([nvcc, "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler",
                               "-fPIC,-fno-strict-aliasing", "-shared", "-o", out, src])
    from odt_b200 import lib as L
    lib = C.CDLL(out)
    fn = getattr(lib, entry)
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(L.ConvParams), C.c_int]
    lib.run = fn
    return lib, L


@pytest.fixture(scope="module")
def host():
    return build_host_harness("thin_host", "conv_thin.cu", "odt_test_thin_host")


def _act(v, act):
    return np.maximum(v, 0) if act == 1 else (np.maximum(v, np.float32(0.1) * v) if act == 2 else v)


def _run(host, B, H, W, Cin, Cout, ks, stride, act=1, residual=False, pre=False, pre2=False, in_halo=0, out_halo=0,
         no_out0=False, force=1, seed=0, aux_halo=0):
    lib, L = host
    rng = np.random.default_rng(seed)
    f16 = np.float16
    ld, old, cpad = (Cin + 63) // 64 * 64, (Cout + 63) // 64 * 64, (Cout + 31) // 32 * 32
    x = rng.standard_normal((B, H, W, Cin)).astype(f16)
    w = (rng.standard_normal((ks, ks, Cin, Cout)) * np.sqrt(2.0 / (ks * ks * Cin))).astype(f16)
    scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    shift = (rng.standard_normal(Cout) * 0.2).astype(np.float32)
    OH, pt, _ = T.same_pad(H, ks, stride)
    OW, pl, _ = T.same_pad(W, ks, stride)
    ih, oh, ah = in_halo, out_halo, aux_halo
    xd = np.zeros((B, H + 2 * ih, W + 2 * ih, ld), f16)
    xd[:, ih:ih + H, ih:ih + W, :Cin] = x
    wd = np.zeros((cpad, ks, ks, ld), f16)
    wd[:Cout, :, :, :Cin] = np.transpose(w, (3, 0, 1, 2))
    yd = np.zeros((B, OH + 2 * oh, OW + 2 * oh, old), f16)
    keep = [xd, wd, yd, scale, shift]
    p = L.ConvParams()
    p.B, p.H, p.W, p.Cin, p.in_ld = B, H, W, Cin, ld
    p.OH, p.OW, p.Cout = OH, OW, Cout
    p.R, p.S, p.stride, p.dil, p.pad_t, p.pad_l = ks, ks, stride, 1, pt, pl
    p.w_ld, p.Cout_pad = ld, cpad
    p.scale, p.shift, p.act = scale.ctypes.data, shift.ctypes.data, act
    p.out0, p.out0_dtype = (None if no_out0 else yd.ctypes.data), L.ODT_F16
    p.out0_img_stride, p.out0_pix_stride = (OH + 2 * oh) * (OW + 2 * oh) * old, old
    p.in_halo, p.out0_halo, p.out0_pool = ih, oh, 0
    res = None
    if residual:
        res = rng.standard_normal((B, OH, OW, Cout)).astype(f16)
        rd = np.zeros_like(yd)
        rd[:, oh:oh + OH, oh:oh + OW, :Cout] = res
        p.residual = rd.ctypes.data
        keep.append(rd)
    if pre:
        s2, h2 = rng.uniform(0.5, 1.5, Cout).astype(np.float32), (rng.standard_normal(Cout) * 0.2).astype(np.float32)
        y1 = np.zeros((B, OH + 2 * ah, OW + 2 * ah, old), f16)
        p.scale2, p.shift2, p.act2 = s2.ctypes.data, h2.ctypes.data, 1
        p.out1, p.out1_img_stride, p.out1_pix_stride = y1.ctypes.data, (OH + 2 * ah) * (OW + 2 * ah) * old, old
        p.out1_halo = ah
        keep += [s2, h2, y1]
    if pre2:
        s3, h3 = rng.uniform(0.5, 1.5, Cout).astype(np.float32), (rng.standard_normal(Cout) * 0.2).astype(np.float32)
        y2 = np.zeros((B, OH + 2 * ah, OW + 2 * ah, old), f16)
        p.scale3, p.shift3, p.act3 = s3.ctypes.data, h3.ctypes.data, 2
        p.out2, p.out2_img_stride, p.out2_pix_stride = y2.ctypes.data, (OH + 2 * ah) * (OW + 2 * ah) * old, old
        p.out2_halo = ah
        keep += [s3, h3, y2]
    rc = lib.run(xd.ctypes.data, wd.ctypes.data, C.byref(p), force)
    if rc != 0:
        return rc, None
    ref = T.conv2d_same(x.astype(np.float32), w.astype(np.float32), None, stride) * scale + shift
    ref = _act(ref, act)
    if residual:
        ref = ref + res.astype(np.float32)
    out = {"ref": ref}
    tol = 2e-3 * max(np.abs(ref).max(), 1.0)
    got = yd[:, oh:oh + OH, oh:oh + OW, :Cout].astype(np.float32)
    if not no_out0:
        assert np.abs(got - ref).max() <= tol
        assert float(np.abs(yd[..., Cout:].astype(np.float32)).max()) == 0.0          # padding lanes stay zero
        if oh:                                                                        # and so does the halo ring
            full = yd.astype(np.float32)
            assert np.abs(full[:, 0]).max() == 0 and np.abs(full[:, -1]).max() == 0
            assert np.abs(full[:, :, 0]).max() == 0 and np.abs(full[:, :, -1]).max() == 0
    base = ref.astype(f16).astype(np.float32) if no_out0 else got      # the consumer sees the ROUNDED out0 value
    if pre:
        want = np.maximum(base * s2 + h2, 0)
        g1 = y1[:, ah:ah + OH, ah:ah + OW, :Cout].astype(np.float32)
        lim = (3 * tol) if no_out0 else 1.5e-3 * max(np.abs(want).max(), 1.0)
        assert np.abs(g1 - want).max() <= lim
        assert float(np.abs(y1[..., Cout:].astype(np.float32)).max()) == 0.0
        if ah:
            full = y1.astype(np.float32)
            assert max(np.abs(full[:, 0]).max(), np.abs(full[:, -1]).max(), np.abs(full[:, :, 0]).max(),
                       np.abs(full[:, :, -1]).max()) == 0
    if pre2:
        t = base * s3 + h3
        want = np.maximum(t, 0.1 * t)
        g2 = y2[:, ah:ah + OH, ah:ah + OW, :Cout].astype(np.float32)
        assert np.abs(g2 - want).max() <= 1.5e-3 * max(np.abs(want).max(), 1.0)
    return 0, out


@pytest.mark.parametrize("shape,kw", [
    ((2, 12, 13, 7, 7, 3, 1), {"in_halo": 1, "out_halo": 1}),
    ((2, 11, 9, 7, 7, 3, 1), {}),
    ((2, 10, 10, 16, 7, 1, 1), {"pre": True}),
    ((2, 10, 10, 7, 28, 1, 1), {"residual": True, "pre": True, "pre2": True, "out_halo": 1}),
    ((2, 10, 10, 28, 14, 1, 1), {"in_halo": 1, "act": 2}),
    ((2, 13, 11, 14, 14, 3, 2), {"in_halo": 1}),
    ((2, 12, 12, 14, 14, 3, 2), {"out_halo": 1, "act": 0}),
    ((1, 8, 8, 32, 32, 1, 1), {"no_out0": True, "pre": True}),
    ((1, 9, 9, 9, 16, 3, 1), {"in_halo": 1, "residual": True}),
])
def test_thin_kernel_source_on_the_cpu(host, shape, kw):
    rc, _ = _run(host, *shape, seed=sum(shape), **kw)
    assert rc == 0


def test_thin_plan_declines_what_the_kernel_cannot_do(host):
    unsupported = -3
    assert _run(host, 1, 8, 8, 40, 8, 1, 1)[0] == unsupported          # Cin > 32
    assert _run(host, 1, 8, 8, 8, 40, 1, 1)[0] == unsupported          # Cout > 32
    assert _run(host, 1, 8, 8, 24, 8, 3, 1)[0] == unsupported          # 3x3 with Cin > 16
    assert _run(host, 1, 8, 8, 16, 16, 3, 1, force=0)[0] == unsupported  # 2 304 multiply-adds per pixel: mode 1 declines
    assert _run(host, 1, 8, 8, 16, 16, 3, 1, force=1)[0] == 0
    assert _run(host, 1, 8, 8, 8, 16, 3, 1, force=0)[0] == unsupported  # mode 1 takes 1x1 layers only (round-2 A/B:
    assert _run(host, 1, 8, 8, 8, 16, 3, 1, force=1)[0] == 0            # every 3x3 is faster through taps-as-N)
    assert _run(host, 1, 8, 8, 16, 8, 1, 1, force=0)[0] == 0            # 1x1, 128 multiply-adds per pixel: taken
