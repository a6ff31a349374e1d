"""The staged pointwise kernel's OWN source (csrc/conv_pw.cu: every phase is a __host__ __device__ function of the
thread id) executed on the CPU, block by block, warp by warp and phase by phase, through a test-only harness
(tests/native/pw_host.cu) and compared with the oracle's convolution + the epilogue chain of epilogue.cuh:
staging indices (halo / dense inputs, ragged last group), the round-robin of pixel groups over warps, the
output-channel passes, fp16 rounding order, residual, the two extra pre-activated outputs (dense and halo layouts), untouched
padding lanes and halo rings.  The device launch itself needs an H100 (tests/test_gpu_conv.py::test_conv_pw_*)."""
import ctypes as C

import pytest

from test_thin_host import _run, build_host_harness


@pytest.fixture(scope="module")
def host():
    lib, L = build_host_harness("pw_host", "conv_pw.cu", "odt_test_pw_host")
    lib.odt_test_pw_plan.restype = C.c_int
    lib.odt_test_pw_plan.argtypes = [C.c_void_p, C.POINTER(L.ConvParams), C.c_int] + [C.POINTER(C.c_int)] * 3
    return lib, L


@pytest.mark.parametrize("shape,kw", [
    ((2, 10, 10, 16, 7, 1, 1), {"pre": True}),                                           # reduce, COT 8
    ((2, 13, 11, 28, 7, 1, 1), {"in_halo": 1, "out_halo": 1}),                            # halo in / out, ragged block
    ((2, 10, 10, 7, 28, 1, 1), {"residual": True, "pre": True, "pre2": True, "out_halo": 1, "aux_halo": 1}),
    ((2, 10, 10, 7, 28, 1, 1), {"residual": True, "pre": True, "pre2": True, "no_out0": True, "aux_halo": 1}),
    ((1, 17, 19, 14, 56, 1, 1), {"residual": True, "pre": True, "pre2": True, "aux_halo": 1}),     # 2 passes
    ((1, 9, 9, 28, 112, 1, 1), {"residual": True, "pre": True, "pre2": True, "no_out0": True}),      # 4 passes
    ((1, 7, 6, 56, 224, 1, 1), {"residual": True, "pre": True, "aux_halo": 1, "in_halo": 1}),        # 7 passes
    ((1, 12, 12, 112, 28, 1, 1), {"act": 2}),                                                         # wide K
    ((1, 8, 8, 56, 14, 1, 1), {"act": 0, "in_halo": 1}),                                              # COT 16
    ((3, 5, 5, 9, 9, 1, 1), {"pre2": True}),                                                          # odd widths
])
def test_pw_kernel_source_on_the_cpu(host, shape, kw):
    rc, _ = _run(host, *shape, seed=sum(shape), **kw)
    assert rc == 0


def test_pw_plan(host):
    lib, L = host
    unsupported = -3
    assert _run(host, 1, 8, 8, 16, 8, 3, 1)[0] == unsupported            # 3x3
    assert _run(host, 1, 8, 8, 16, 8, 1, 2)[0] == unsupported            # stride 2
    assert _run(host, 1, 8, 8, 136, 8, 1, 1)[0] == unsupported           # Cin > 128
    assert _run(host, 1, 8, 8, 8, 264, 1, 1)[0] == unsupported           # Cout > 256
    assert _run(host, 1, 8, 8, 56, 224, 1, 1, force=0)[0] == unsupported   # 14 336 multiply-adds per pixel: tensor-core work
    assert _run(host, 1, 8, 8, 56, 224, 1, 1, force=1)[0] == 0
    # default planner: only where the round-2 A/B showed a gain (8-channel-input expand layers of large maps)
    assert _run(host, 1, 8, 8, 28, 112, 1, 1, force=0)[0] == unsupported
    assert _run(host, 1, 8, 8, 7, 28, 1, 1, force=0)[0] == unsupported      # 64 pixels: not worth a launch of its own
    assert _run(host, 1, 512, 512, 7, 28, 1, 1, force=0)[0] == 0
