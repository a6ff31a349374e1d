"""Shared pieces of the GPU kernel tests: sentinel-guarded output buffers, the halo / channel masks a kernel must not
write, the names of the library kernels a call launches (from a torch.profiler trace, or the library's record of its
last convolution launch), and the network constructor of the in-situ checks."""
import re

import numpy as np
import torch

SENT = -12345.0  # exactly representable in fp16 and fp32


class Guarded:
    """A tensor of `shape` placed `off` elements into a sentinel-filled buffer with `guard` elements on either side;
    `fill` (optional) gives the tensor's initial contents."""

    def __init__(self, shape, dt, off=0, guard=2048, fill=None):
        n = int(np.prod(shape))
        self.buf = torch.full((n + 2 * guard + off,), SENT, dtype=dt, device="cuda")
        self.lo, self.n = guard + off, n
        self.t = self.buf[self.lo:self.lo + n].view(shape)
        if fill is not None:
            self.t.copy_(fill)
        self.before = self.buf.clone()

    def ptr(self):
        return self.t.data_ptr()

    def initial(self):
        """The tensor's contents before the call under test."""
        return self.before[self.lo:self.lo + self.n].view(self.t.shape)

    def assert_outside_untouched(self):
        b, a = self.buf, self.before
        assert torch.equal(b[:self.lo], a[:self.lo]), "write before the tensor"
        assert torch.equal(b[self.lo + self.n:], a[self.lo + self.n:]), "write past the tensor"

    def assert_untouched(self, region, what):
        """`region` (a boolean mask over the tensor) kept its initial contents."""
        now, was = self.t[region], self.initial()[region]
        assert torch.equal(now, was), "%s written" % what


def mask(shape, halo=0, c=None):
    """True at the positions a kernel must not write: the 1-pixel halo and the channels >= c."""
    m = torch.zeros(shape, dtype=torch.bool, device="cuda")
    if halo:
        m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = True, True, True, True
    if c is not None:
        m[..., c:] = True
    return m


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def assert_slice_writes(now, was, c0, cout, end, what):
    """The write rules of a channel slice [c0, c0 + cout) of a wider tensor (Net.concat's parts): every element of the
    slice written; channels [c0 + cout, end) untouched or +0 (the pad lanes of a producer that stores whole chunks);
    every other channel keeps its initial bits.  Returns how many channels past the slice were written (with +0)."""
    assert not bool((now[..., c0:c0 + cout] == SENT).any()), "%s: a slice element left unwritten" % what
    pad = now[..., c0 + cout:end]
    wrote = _bits(pad) != _bits(was[..., c0 + cout:end])
    assert bool((~wrote | (_bits(pad) == 0)).all()), "%s: channels [c0 + Cout, %d) hold neither +0 nor the initial " \
                                                     "contents" % (what, end)
    assert torch.equal(_bits(now[..., :c0]), _bits(was[..., :c0])), "%s: channels below the slice written" % what
    assert torch.equal(_bits(now[..., end:]), _bits(was[..., end:])), "%s: channels >= %d written" % (what, end)
    if wrote.shape[-1] == 0:
        return 0
    cols = wrote.reshape(-1, wrote.shape[-1]).any(dim=0).nonzero()
    return int(cols.max()) + 1 if cols.numel() else 0


def interior(t, halo):
    return t[:, halo:t.shape[1] - halo, halo:t.shape[2] - halo] if halo else t


def kernels_launched(fn, tries=3):
    """(fn(), names with whitespace removed of the library's kernels fn launches), from a torch.profiler trace.  A short
    trace can come back without some of its device activity, so fn runs between two torch marker kernels and the trace
    counts only when both markers are in it (fn is re-run otherwise: every call here is idempotent)."""
    from torch.profiler import ProfilerActivity, profile
    marker = torch.zeros(1, device="cuda")
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            marker.add_(1)
            out = fn()
            marker.add_(1)
            torch.cuda.synchronize()
        names = [re.sub(r"\s+", "", e.name) for e in prof.events()
                 if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
                 and "Memset" not in e.name]
        if len([n for n in names if "odt::" not in n]) == 2:
            return out, [n for n in names if "odt::" in n]
    raise AssertionError("%d profiler traces in a row lost device activity" % tries)


def last_conv_kernel():
    """Name of the convolution kernel the library's last odt_conv2d_* call launched, e.g. "conv_tc_kernel<128,true>"
    (the names nm -C gives the instantiations, without whitespace).  It needs no profiler trace, which late in a long
    test process can come back without device activity."""
    import ctypes
    from odt_b200 import lib as L
    f = L.load().odt_debug_last_conv_kernel
    f.restype = ctypes.c_char_p
    return f().decode()


def model(kind, precision, **over):
    """One of the six detectors with trained-style BN statistics (helpers.model_cfg), no checkpoint."""
    from helpers import model_cfg
    import FCOS
    import RetinaNet
    import SSD300
    import SSD512
    import YOLOv3
    if kind == "ssd300":
        return SSD300.SSD300(model_cfg("ssd", precision=precision, bn_init="trained", **over), None)
    if kind == "ssd512":
        return SSD512.SSD512(model_cfg("ssd", precision=precision, bn_init="trained", **over), None)
    if kind == "retinanet":
        return RetinaNet.RetinaNet(model_cfg("retinanet", precision=precision, bn_init="trained", **over), None)
    if kind == "yolov3":
        return YOLOv3.YOLOv3(model_cfg("yolov3", precision=precision, bn_init="trained", **over), None)
    if kind == "yolov2":  # `over` takes _cfg's A (priors), nc (classes) and size as well
        import YOLOv2
        from test_gpu_yolov2 import _cfg
        return YOLOv2.YOLOv2(_cfg(precision=precision, bn_init="trained", **over), None)
    return FCOS.FCOS(model_cfg("fcos", precision=precision, bn_init="trained", **over), None)
