"""The training-image augmentation kernels (csrc/augment.cu, odt_augment_batch) behind
`BatchIterator.get_next(device)`: tfrecord.augment_pixels for a whole batch on the GPU.

The host side is what tfrecord.plan_augment decided per image (AugmentPlan) plus the uint8 sources.  They go through
one reused pinned staging buffer and one host-to-device copy; the launches run on the device's current stream."""
import ctypes as C

import numpy as np
import torch

from . import lib as L

_MODES = {"bilinear": L.AUG_BILINEAR, "nearest": L.AUG_NEAREST, "bicubic": L.AUG_BICUBIC, "pad": L.AUG_PAD,
          "legacy": L.AUG_LEGACY}


def kernel_params(plan, src_offset=0):
    """odt_augment_params of one AugmentPlan: the float32 scalars are numpy's own (np.float32 of each draw,
    np.float32(delta) * np.float32(6) for hue, the rotation's cos / sin / offsets)."""
    p = L.AugmentParams()
    p.src_offset, p.h, p.w, p.mode = int(src_offset), plan.h, plan.w, _MODES[plan.mode]
    p.zh, p.zw, p.rh, p.rw, p.cval = plan.zh, plan.zw, plan.rh, plan.rw, float(plan.cval)
    p.crop_y, p.crop_x = plan.crop if plan.crop is not None else (0, 0)
    p.flip_y, p.flip_x = int(plan.flip_y), int(plan.flip_x)
    if plan.brightness is not None:
        p.brightness_on, p.brightness = 1, float(np.float32(plan.brightness))
    if plan.contrast is not None:
        p.contrast_on, p.contrast = 1, float(np.float32(plan.contrast))
    if plan.hue is not None:
        p.hue_on, p.hue6 = 1, float(np.float32(plan.hue) * np.float32(6))
    if plan.angle is not None:
        p.rotate_on = 1
        p.rot_c, p.rot_s, p.rot_x_off, p.rot_y_off = (float(v) for v in plan.rotation)
    p.oh, p.ow = plan.oh, plan.ow
    p.layout = L.AUG_NCHW if plan.channels_first else L.AUG_NHWC
    return p


class GpuAugmentor:
    """Reusable buffers of the device path: a pinned staging buffer for the sources, their device copy and the
    kernels' scratch, grown on demand and reallocated when a call names another device.  The staging buffer is
    refilled only once its previous copy has left."""

    def __init__(self):
        self._pinned = self._src = self._scratch = None
        self._copied = None

    @staticmethod
    def _grow(buf, n, device, **kw):
        if buf is None or buf.numel() < n or buf.device != device:
            return torch.empty(max(n, 1), dtype=torch.uint8, device=device, **kw)
        return buf

    def __call__(self, items, device, means_out=None):
        """items: [(uint8 [h, w, 3] source, AugmentPlan, ...)] -> float32 [B, oh, ow, 3] (or [B, 3, oh, ow]) on
        `device`.  means_out: optional float32 [B, 3] CUDA tensor for the contrast means."""
        lib = L.load()
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError("the augmentation kernels run on a CUDA device, not %s" % device)
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        B = len(items)
        srcs = [np.ascontiguousarray(i[0], np.uint8) for i in items]
        for s in srcs:
            if s.ndim != 3 or s.shape[2] != 3:
                raise ValueError("the augmentation kernels take RGB uint8 [h, w, 3] sources, not %s" % (s.shape,))
        offsets = np.concatenate([[0], np.cumsum([s.nbytes for s in srcs])]).astype(np.int64)
        params = (L.AugmentParams * B)(*[kernel_params(i[1], o) for i, o in zip(items, offsets[:-1])])
        need = int(lib.odt_augment_scratch_bytes(params, B))
        if need < 0:
            raise ValueError("augmentation plan rejected: %s" % lib.odt_last_error().decode())
        total = int(offsets[-1])
        with torch.cuda.device(device):
            if self._copied is not None:
                self._copied.synchronize()          # the previous batch's copy has read the staging buffer
            self._pinned = self._grow(self._pinned, total, torch.device("cpu"), pin_memory=True)
            self._src = self._grow(self._src, total, device)
            self._scratch = self._grow(self._scratch, need, device)
            staging = self._pinned.numpy()
            for s, o in zip(srcs, offsets[:-1]):
                staging[o:o + s.nbytes] = s.reshape(-1)
            stream = torch.cuda.current_stream(device)
            self._src[:total].copy_(self._pinned[:total], non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record(stream)
            plan = items[0][1]
            shape = (B, 3, plan.oh, plan.ow) if plan.channels_first else (B, plan.oh, plan.ow, 3)
            out = torch.empty(shape, dtype=torch.float32, device=device)
            if means_out is not None:
                assert means_out.shape == (B, 3) and means_out.dtype == torch.float32 and means_out.device == device
            L.check(lib.odt_augment_batch(self._src.data_ptr(), params, B, out.data_ptr(),
                                          means_out.data_ptr() if means_out is not None else None,
                                          self._scratch.data_ptr(), stream.cuda_stream), "odt_augment_batch")
        return out
