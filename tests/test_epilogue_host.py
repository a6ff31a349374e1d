"""The fused fp16 output step of csrc/epilogue.cuh, on the CPU through a test-only harness (tests/native/epilogue_host.cu):
the vector step epi_store_f16<1> / <4> (what conv_tc, conv_tapn, conv_thin and conv_pw store) must be bit-identical,
element by element, to the scalar epi_store_one<__half> (what conv_direct stores).  Covers every activation triple,
residual / out0 / out1 / out2 on and off, dense and halo extra outputs, missing scale / shift pointers, a run that
straddles Cout (its pad channels take epi_param's identity parameters), fp16 rounding ties and overflow."""
import ctypes as C
import itertools

import numpy as np
import pytest

from test_thin_host import build_host_harness

B, OH, OW = 2, 3, 5


@pytest.fixture(scope="module")
def host():
    lib, L = build_host_harness("epilogue_host", "epilogue.cuh", "odt_test_epilogue_host")
    lib.run.argtypes = [C.POINTER(L.ConvParams), C.c_void_p, C.c_int, C.c_int, C.c_int]
    return lib, L


def _act(v, act):
    return np.maximum(v, 0) if act == 1 else (np.maximum(v, np.float32(0.1) * v) if act == 2 else v)


def _inputs(rng, cout, cpad):
    acc = (rng.standard_normal((B, OH * OW, cpad)) * 4).astype(np.float32)
    # channels 0..3 have scale 1 / shift 0: the accumulator reaches the fp16 rounding unchanged (without a residual)
    ties = np.array([1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 2049, -2051, 65520, 65504, 70000, -1e6], np.float32)
    acc[:, :, :4] = ties[rng.integers(0, len(ties), (B, OH * OW, 4))]
    prm = {}
    for k in ("scale", "scale2", "scale3"):
        prm[k] = rng.uniform(-1.5, 1.5, cout).astype(np.float32)
    for k in ("shift", "shift2", "shift3"):
        prm[k] = (rng.standard_normal(cout) * 0.5).astype(np.float32)
    prm["scale"][:4], prm["shift"][:4] = 1, 0
    res = rng.standard_normal((B, OH * OW, cpad + 8)).astype(np.float16)
    return acc, prm, res


def _run(host, nv, cout, acts, residual, out0, out1, out2, halo, nullp, seed):
    lib, L = host
    cpad = (cout + 8 * nv - 1) // (8 * nv) * (8 * nv)
    ld = cpad + 8  # one sector past the last run: must stay untouched
    acc, prm, res = _inputs(np.random.default_rng(seed), cout, cpad)
    ah = 1 if halo else 0
    aux_shape = (B, (OH + 2 * ah) * (OW + 2 * ah), ld)

    def params(bufs):
        p = L.ConvParams()
        p.B, p.H, p.W, p.OH, p.OW, p.Cout, p.Cout_pad = B, OH, OW, OH, OW, cout, cpad
        p.act, p.act2, p.act3 = acts
        for k in ("scale", "shift", "scale2", "shift2", "scale3", "shift3"):
            setattr(p, k, prm[k].ctypes.data)
        if nullp:  # missing pointers on both the first affine step and one extra output
            p.scale, p.shift, p.shift3 = None, None, None
        p.out0_dtype = L.ODT_F16
        p.out0_img_stride, p.out0_pix_stride = OH * OW * ld, ld
        p.out1_img_stride = p.out2_img_stride = aux_shape[1] * ld
        p.out1_pix_stride = p.out2_pix_stride = ld
        p.out1_halo = p.out2_halo = ah
        if residual:
            p.residual = res.ctypes.data
        if out0:
            p.out0 = bufs[0].ctypes.data
        if out1:
            p.out1 = bufs[1].ctypes.data
        if out2:
            p.out2 = bufs[2].ctypes.data
        return p

    got = [np.zeros((B, OH * OW, ld), np.float16), np.zeros(aux_shape, np.float16), np.zeros(aux_shape, np.float16)]
    want = [np.zeros_like(b) for b in got]
    assert lib.run(C.byref(params(got)), acc.ctypes.data, cpad, nv, 1) == 0
    assert lib.run(C.byref(params(want)), acc.ctypes.data, cpad, nv, 0) == 0
    for i, on in enumerate((out0, out1, out2)):
        if on:
            assert np.array_equal(got[i].view(np.uint16), want[i].view(np.uint16)), "output %d differs" % i
        else:
            assert not got[i].view(np.uint16).any(), "output %d written although disabled" % i
            assert not want[i].view(np.uint16).any(), "scalar output %d written although disabled" % i
        assert not got[i][..., cpad:].view(np.uint16).any()
    if out0:
        # channels past Cout: scale 1 / shift 0 whatever the pointers say
        v = _act(acc[..., cout:cpad], acts[0])
        if residual:
            v = v + res[..., cout:cpad].astype(np.float32)
        assert np.array_equal(got[0][..., cout:cpad].view(np.uint16), v.astype(np.float16).view(np.uint16))


@pytest.mark.parametrize("nv,cout", [(1, 21), (4, 45)])
@pytest.mark.parametrize("acts", list(itertools.product(range(3), repeat=3)))
def test_vector_step_matches_scalar_epilogue(host, nv, cout, acts):
    for opts in itertools.product((False, True), repeat=6):
        residual, out0, out1, out2, halo, nullp = opts
        if not (out0 or out1 or out2):
            continue
        _run(host, nv, cout, acts, residual, out0, out1, out2, halo, nullp, seed=sum(acts) + 7 * sum(opts))
