"""TFRecord + tf.train.Example reader / writer and the VOC record schema of the reference's
input pipeline (utils/tfrecord_voc_utils.py:30-113), without TensorFlow.  Host-side IO for
SURVEY section 8(f) row 3.  The augmentation's pixel step also runs as CUDA kernels (odt_b200/augment.py,
`BatchIterator.get_next(device)`); everything else here is host-side.

* TFRecord framing: u64 length | u32 masked crc32c(length) | payload | u32 masked crc32c(payload).
* tf.train.Example: Example{1: Features{1: map<string, Feature>}}, Feature = oneof
  {1: BytesList{1: bytes...}, 2: FloatList{1: packed float}, 3: Int64List{1: packed varint}}.
* VOC schema written by `xml_to_example` (:30-62): 'image' = JPEG bytes, 'shape' = int32[3]
  (h, w, c) as bytes, 'ground_truth' = float32[n,5] rows (ymin, ymax, xmin, xmax, class id).
* `preprocess` restates `image_augmentor` (utils/image_augmentor.py:7-264): align_corners bilinear /
  nearest resize (optionally aspect-preserving + constant padding) to `zoom_size`/`output_shape`, centre or
  random crop, top-down / left-right flips (with the reference's `- 1` offsets), colour jitter (brightness,
  contrast, hue as TF's adjust_* ops define them), small-angle rotation with the box re-fit of
  `rotate_helper`, box clamping, the centre-inside filter, the "no box left" fallback of
  `gt_checker_helper`, (y_centre, x_centre, h, w, id) rows padded with -1 to `pad_truth_to`; randomness
  from a seeded numpy generator.  BICUBIC resampling restates TF 1.13's table-driven ResizeBicubic kernel.
  (The reference returns the UNaugmented `image_copy` when `pad_truth_to` is set, :229 -- an upstream slip
  that would defeat batching; the augmented image is returned here.  It also concatenates the UNfiltered box
  centres with the filtered sizes / ids (:211-220), a shape error whenever a box is dropped; the filtered
  centres are used here.)
PARITY UNPINNED: no TensorFlow and no TF-written record here; JPEG decoding goes through
OpenCV (libjpeg-turbo), TF uses libjpeg -- pixels can differ by a few levels.
"""
import struct
import sys

import numpy as np

from .tf_checkpoint import (CheckpointError, _get_varint, _pb_bytes, _pb_fields, _put_varint, crc32c,
                            mask_crc)


class RecordError(CheckpointError):
    pass


# ---------------------------------------------------------------- framing ---
def write_records(path, payloads):
    with open(path, "wb") as f:
        for p in payloads:
            head = struct.pack("<Q", len(p))
            f.write(head)
            f.write(struct.pack("<I", mask_crc(crc32c(head))))
            f.write(p)
            f.write(struct.pack("<I", mask_crc(crc32c(p))))


def read_records(path, verify=True):
    import os
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        while True:
            head = f.read(8)
            if not head:
                return
            if len(head) != 8:
                raise RecordError("%s: truncated record header" % path)
            (n,) = struct.unpack("<Q", head)
            hc = f.read(4)
            if len(hc) != 4:
                raise RecordError("%s: truncated record header" % path)
            if verify and mask_crc(crc32c(head)) != struct.unpack("<I", hc)[0]:
                raise RecordError("%s: record length checksum mismatch" % path)
            if n > size - f.tell():      # also keeps a corrupt length from turning into a huge allocation
                raise RecordError("%s: truncated record" % path)
            data = f.read(n)
            tail = f.read(4)
            if len(data) != n or len(tail) != 4:
                raise RecordError("%s: truncated record" % path)
            if verify and mask_crc(crc32c(data)) != struct.unpack("<I", tail)[0]:
                raise RecordError("%s: record payload checksum mismatch" % path)
            yield data


# ---------------------------------------------------------------- Example ---
def encode_example(features):
    """features: {name: bytes | list of bytes | float array | int array}."""
    fmap = bytearray()
    for key in sorted(features):
        v = features[key]
        feat = bytearray()
        if isinstance(v, (bytes, bytearray)):
            v = [bytes(v)]
        if isinstance(v, (list, tuple)) and v and isinstance(v[0], (bytes, bytearray)):
            bl = bytearray()
            for b in v:
                _pb_bytes(bl, 1, bytes(b))
            _pb_bytes(feat, 1, bl)
        else:
            a = np.asarray(v)
            inner = bytearray()
            if a.dtype.kind == "f":
                _pb_bytes(inner, 1, a.astype("<f4").tobytes())
                _pb_bytes(feat, 2, inner)
            else:
                packed = bytearray()
                for x in a.reshape(-1).tolist():
                    _put_varint(packed, int(x))
                _pb_bytes(inner, 1, packed)
                _pb_bytes(feat, 3, inner)
        entry = bytearray()
        _pb_bytes(entry, 1, key.encode("utf-8"))
        _pb_bytes(entry, 2, feat)
        _pb_bytes(fmap, 1, entry)
    out = bytearray()
    _pb_bytes(out, 1, fmap)
    return bytes(out)


def parse_example(data):
    """-> {name: list of bytes | float32 array | int64 array}."""
    out = {}
    for f, _, features in _pb_fields(data):
        if f != 1:
            continue
        for f2, _, entry in _pb_fields(features):
            if f2 != 1:
                continue
            key, feat = None, b""
            for f3, wt3, v in _pb_fields(entry):
                if wt3 != 2:
                    raise RecordError("Example: map entry field %d is not length-delimited" % f3)
                if f3 == 1:
                    try:
                        key = v.decode("utf-8")
                    except UnicodeDecodeError:
                        raise RecordError("Example: feature name is not UTF-8") from None
                elif f3 == 2:
                    feat = v
            val = []
            for kind, wtk, lst in _pb_fields(feat):
                if wtk != 2:
                    raise RecordError("Example: Feature field %d is not length-delimited" % kind)
                if kind == 1:
                    val = []
                    for f4, wt, v in _pb_fields(lst):
                        if f4 == 1:
                            if wt != 2:
                                raise RecordError("Example: BytesList value is not length-delimited")
                            val.append(v)
                elif kind == 2:
                    parts = []
                    for f4, wt, v in _pb_fields(lst):
                        if f4 == 1:
                            if wt == 2 and len(v) % 4 == 0:
                                parts.append(np.frombuffer(v, "<f4"))
                            elif wt == 5:
                                parts.append(np.frombuffer(struct.pack("<I", v), "<f4"))
                            else:
                                raise RecordError("Example: malformed FloatList")
                    val = np.concatenate(parts).astype(np.float32) if parts else np.zeros(0, np.float32)
                elif kind == 3:
                    ints = []
                    for f4, wt, v in _pb_fields(lst):
                        if f4 != 1:
                            continue
                        if wt == 2:
                            pos = 0
                            while pos < len(v):
                                x, pos = _get_varint(v, pos)
                                ints.append(x - (1 << 64) if x >= (1 << 63) else x)
                        elif wt == 0:
                            ints.append(v - (1 << 64) if v >= (1 << 63) else v)
                        else:
                            raise RecordError("Example: malformed Int64List")
                    val = np.asarray(ints, np.int64)
            if key is not None:
                out[key] = val
    return out


# ------------------------------------------------------------- VOC schema ---
def encode_voc_example(jpeg_bytes, shape, ground_truth):
    return encode_example({"image": jpeg_bytes, "shape": np.asarray(shape, "<i4").tobytes(),
                           "ground_truth": np.asarray(ground_truth, "<f4").tobytes()})


def decode_voc_example(data):
    """-> (image uint8 [H,W,3] RGB, ground_truth float32 [n,5] = (ymin, ymax, xmin, xmax, id))."""
    ex = parse_example(data)
    for k in ("image", "shape", "ground_truth"):
        if k not in ex or len(ex[k]) == 0:
            raise RecordError("record lacks the %r feature" % k)
    for k in ("image", "shape", "ground_truth"):
        if not isinstance(ex[k], list):
            raise RecordError("feature %r is not a bytes list" % k)
    if len(ex["shape"][0]) != 12 or len(ex["ground_truth"][0]) % 20:
        raise RecordError("'shape' must hold 3 int32 and 'ground_truth' rows of 5 float32")
    gt = np.frombuffer(ex["ground_truth"][0], "<f4").reshape(-1, 5).astype(np.float32)
    return _decode_image(ex), gt


# -------------------------------------------------------- ImageNet schema ---
def encode_imagenet_example(jpeg_bytes, shape, label):
    """utils/tfrecord_imagenet_utils.py:83-93: 'image' = JPEG bytes, 'shape' = int32[3] (h, w, c) as bytes,
    'label' = int64 class id."""
    return encode_example({"image": jpeg_bytes, "shape": np.asarray(shape, "<i4").tobytes(),
                           "label": np.asarray([label], np.int64)})


def decode_imagenet_example(data):
    """-> (image uint8 [H,W,3] RGB, label int64) (parse_function, utils/tfrecord_imagenet_utils.py:100-115)."""
    ex = parse_example(data)
    for k in ("image", "shape", "label"):
        if k not in ex or len(ex[k]) == 0:
            raise RecordError("record lacks the %r feature" % k)
    for k in ("image", "shape"):
        if not isinstance(ex[k], list):
            raise RecordError("feature %r is not a bytes list" % k)
    if isinstance(ex["label"], list) or ex["label"].dtype != np.int64 or len(ex["label"]) != 1:
        raise RecordError("'label' must be one int64")
    if len(ex["shape"][0]) != 12:
        raise RecordError("'shape' must hold 3 int32")
    return _decode_image(ex), np.int64(ex["label"][0])


def _decode_image(ex):
    """The 'image' JPEG of a parsed record, RGB, checked against its 'shape' feature."""
    import cv2
    shape = np.frombuffer(ex["shape"][0], "<i4")
    img = cv2.imdecode(np.frombuffer(ex["image"][0], np.uint8), cv2.IMREAD_COLOR)
    if img is None:
        raise RecordError("image bytes are not decodable")
    img = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
    if tuple(img.shape) != tuple(int(x) for x in shape):
        raise RecordError("decoded image %s does not match the stored shape %s" % (img.shape, shape.tolist()))
    return img


def _resize_bilinear_aligned(img, oh, ow):
    """tf.image.resize_images(..., BILINEAR, align_corners=True) as image_augmentor calls it (:103-106,:124-127):
    src = dst * (in - 1) / (out - 1)."""
    h, w = img.shape[:2]
    x = img.astype(np.float32)
    sy = np.float32((h - 1) / (oh - 1)) if oh > 1 else np.float32(0)
    sx = np.float32((w - 1) / (ow - 1)) if ow > 1 else np.float32(0)
    ys = np.arange(oh, dtype=np.float32) * sy
    xs = np.arange(ow, dtype=np.float32) * sx
    y0 = np.floor(ys).astype(np.int64)
    x0 = np.floor(xs).astype(np.int64)
    y1 = np.minimum(y0 + 1, h - 1)
    x1 = np.minimum(x0 + 1, w - 1)
    wy = (ys - y0).astype(np.float32).reshape(-1, 1, 1)
    wx = (xs - x0).astype(np.float32).reshape(1, -1, 1)
    top = x[y0][:, x0] * (1 - wx) + x[y0][:, x1] * wx
    bot = x[y1][:, x0] * (1 - wx) + x[y1][:, x1] * wx
    return (top * (1 - wy) + bot * wy).astype(np.float32)


_BICUBIC_TABLE = None


def _bicubic_table():
    """TF's ResizeBicubic weight table (resize_bicubic_op.cc, TF 1.13): 1024 + 1 entries of the Keys kernel with
    A = -0.75, float32: [i*2] = weight of a tap at distance x = i/1024 (|x| <= 1), [i*2+1] = at distance x + 1."""
    global _BICUBIC_TABLE
    if _BICUBIC_TABLE is None:
        a = np.float32(-0.75)
        x = (np.arange(1025, dtype=np.float32) * np.float32(1.0 / 1024)).astype(np.float32)
        t = np.empty(2 * 1025, np.float32)
        t[0::2] = ((a + 2) * x - (a + 3)) * x * x + 1
        x1 = x + np.float32(1.0)
        t[1::2] = ((a * x1 - 5 * a) * x1 + 8 * a) * x1 - 4 * a
        _BICUBIC_TABLE = t
    return _BICUBIC_TABLE


def _bicubic_axis(n_in, n_out):
    """Per output coordinate: four clamped source indices and their table weights (GetWeightsAndIndices with
    align_corners=True: src = dst * (in - 1)/(out - 1), no half-pixel centres; offset = lrintf(frac * 1024))."""
    scale = np.float32((n_in - 1) / (n_out - 1)) if n_out > 1 else np.float32(0)
    loc = (np.arange(n_out, dtype=np.float32) * scale).astype(np.float32)
    fl = np.floor(loc)
    off = np.rint((loc - fl) * np.float32(1024)).astype(np.int64)   # lrintf: round half to even, like numpy
    base = fl.astype(np.int64)
    t = _bicubic_table()
    w = np.stack([t[off * 2 + 1], t[off * 2], t[(1024 - off) * 2], t[(1024 - off) * 2 + 1]], axis=1)
    idx = np.clip(np.stack([base - 1, base, base + 1, base + 2], axis=1), 0, n_in - 1)
    return idx, w.astype(np.float32)


def _resize_bicubic_aligned(img, oh, ow):
    """tf.image.resize_images(..., BICUBIC, align_corners=True) of image_augmentor (:103-106,:121-127): TF 1.13's
    ResizeBicubic kernel -- table-driven Keys cubic (A = -0.75), taps clamped at the border, float32, interpolating
    along x first and then along y.  [TF-sem: restated from the kernel's source, unverifiable here]"""
    x = img.astype(np.float32)
    h, w = x.shape[:2]
    yi, yw = _bicubic_axis(h, oh)
    xi, xw = _bicubic_axis(w, ow)
    rows = sum(x[:, xi[:, k]] * xw[:, k].reshape(1, -1, 1) for k in range(4)).astype(np.float32)   # [h, ow, c]
    return sum(rows[yi[:, k]] * yw[:, k].reshape(-1, 1, 1) for k in range(4)).astype(np.float32)


def _resize_nearest_aligned(img, oh, ow):
    """ResizeNearestNeighbor with align_corners=True (TF 1.13): src = min(round(dst * (in-1)/(out-1)), in-1)."""
    h, w = img.shape[:2]
    sy = np.float32((h - 1) / (oh - 1)) if oh > 1 else np.float32(0)
    sx = np.float32((w - 1) / (ow - 1)) if ow > 1 else np.float32(0)
    ys = np.minimum(np.floor(np.arange(oh, dtype=np.float32) * sy + np.float32(0.5)).astype(np.int64), h - 1)
    xs = np.minimum(np.floor(np.arange(ow, dtype=np.float32) * sx + np.float32(0.5)).astype(np.int64), w - 1)
    return img[ys][:, xs].astype(np.float32)


def _resize_bilinear_legacy(img, oh, ow):
    """tf.image.resize(image, size) of gt_checker_helper (:260): TF1 bilinear, align_corners=False, no
    half-pixel centres: src = dst * in/out, hi = min(lo + 1, in - 1)."""
    h, w = img.shape[:2]
    x = img.astype(np.float32)
    ys = np.arange(oh, dtype=np.float32) * np.float32(h / oh)
    xs = np.arange(ow, dtype=np.float32) * np.float32(w / ow)
    y0 = np.minimum(np.floor(ys).astype(np.int64), h - 1)
    x0 = np.minimum(np.floor(xs).astype(np.int64), w - 1)
    y1 = np.minimum(y0 + 1, h - 1)
    x1 = np.minimum(x0 + 1, w - 1)
    wy = (ys - y0).astype(np.float32).reshape(-1, 1, 1)
    wx = (xs - x0).astype(np.float32).reshape(1, -1, 1)
    top = x[y0][:, x0] * (1 - wx) + x[y0][:, x1] * wx
    bot = x[y1][:, x0] * (1 - wx) + x[y1][:, x1] * wx
    return (top * (1 - wy) + bot * wy).astype(np.float32)


def adjust_brightness(img, delta):
    """tf.image.adjust_brightness on a float image: image + delta (no rescale, no clipping)."""
    return (img + np.float32(delta)).astype(np.float32)


def adjust_contrast(img, factor, mean=None):
    """tf.image.adjust_contrast: (x - mean) * factor + mean with the mean of each channel over H, W.  `mean` (3
    float32) replaces numpy's own float32 mean, so that a mean computed elsewhere can be applied bit for bit."""
    if mean is None:
        mean = img.mean(axis=(0, 1), keepdims=True, dtype=np.float32)
    else:
        mean = np.asarray(mean, np.float32).reshape(1, 1, -1)
    return ((img - mean) * np.float32(factor) + mean).astype(np.float32)


def adjust_hue(img, delta):
    """tf.image.adjust_hue (AdjustHue kernel): RGB -> (hue in [0,6), min, max), hue += 6*delta (wrapped),
    back to RGB.  The (min, max) pair is kept, so the result is independent of the value range."""
    x = img.astype(np.float32)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    vmax = np.maximum(np.maximum(r, g), b)
    vmin = np.minimum(np.minimum(r, g), b)
    rng_ = vmax - vmin
    safe = np.where(rng_ > 0, rng_, np.float32(1))
    # sector of the hue hexagon and the position inside it (all six orderings of r, g, b; ties as the kernel)
    cat = np.select([(r < g) & (b < r), (r < g) & (b > g), (r < g), (b < g), (b > r)], [1, 3, 2, 0, 4], 5)
    vmid = r + g + b - vmax - vmin
    ratio = (vmid - vmin) / safe
    inc = (cat % 2) == 0
    h = np.where(rng_ > 0, cat + np.where(inc, ratio, 1 - ratio), np.float32(0)).astype(np.float32)
    h = np.mod(h + np.float32(delta) * np.float32(6), np.float32(6)).astype(np.float32)
    cat2 = np.minimum(h.astype(np.int64), 5)
    frac = h - cat2
    frac = np.where((cat2 % 2) == 0, frac, 1 - frac)
    mid = vmin + frac * rng_
    r2 = np.select([cat2 == 0, cat2 == 1, cat2 == 2, cat2 == 3, cat2 == 4], [vmax, mid, vmin, vmin, mid], vmax)
    g2 = np.select([cat2 == 0, cat2 == 1, cat2 == 2, cat2 == 3, cat2 == 4], [mid, vmax, vmax, mid, vmin], vmin)
    b2 = np.select([cat2 == 0, cat2 == 1, cat2 == 2, cat2 == 3, cat2 == 4], [vmin, vmin, mid, vmax, vmax], mid)
    return np.stack([r2, g2, b2], -1).astype(np.float32)


def rotation_coefficients(angle, h, w):
    """(cos, sin, x_off, y_off) of `rotate_bilinear` on an h x w image, float32 as numpy computes them."""
    c, s = np.float32(np.cos(angle)), np.float32(np.sin(angle))
    x_off = np.float32(((w - 1) - (c * (w - 1) - s * (h - 1))) / 2.0)
    y_off = np.float32(((h - 1) - (s * (w - 1) + c * (h - 1))) / 2.0)
    return c, s, x_off, y_off


def rotate_bilinear(img, angle):
    """tf.contrib.image.rotate(img, angle, 'BILINEAR'): counter-clockwise by `angle` (radians) about the
    image centre; output pixel (x, y) samples input (cos*x - sin*y + x_off, sin*x + cos*y + y_off) with the
    offsets of angles_to_projective_transforms; neighbours outside the image read 0."""
    h, w = img.shape[:2]
    c, s, x_off, y_off = rotation_coefficients(angle, h, w)
    xs, ys = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32))
    sx = c * xs - s * ys + x_off
    sy = s * xs + c * ys + y_off
    x0, y0 = np.floor(sx), np.floor(sy)
    wx, wy = (sx - x0)[..., None], (sy - y0)[..., None]
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    src = img.astype(np.float32)

    def read(yy, xx):
        ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        return np.where(ok[..., None], src[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)], np.float32(0))

    top = read(y0, x0) * (1 - wx) + read(y0, x0 + 1) * wx
    bot = read(y0 + 1, x0) * (1 - wx) + read(y0 + 1, x0 + 1) * wx
    return (top * (1 - wy) + bot * wy).astype(np.float32)


def rotate_boxes(angle, ymin, xmin, ymax, xmax, oh, ow):
    """Box re-fit of rotate_helper (:236-256): the four corners rotated by -angle about
    ((ow-1)/2, (oh-1)/2), then their axis-aligned hull."""
    a = np.float32(-angle)
    c, s = np.float32(np.cos(a)), np.float32(np.sin(a))
    cx, cy = np.float32((ow - 1.0) / 2.0), np.float32((oh - 1.0) / 2.0)
    off_x = cx * (1 - c) + cy * s
    off_y = cy * (1 - c) - cx * s
    px = [x * c - y * s + off_x for x, y in ((xmin, ymin), (xmax, ymax), (xmin, ymax), (xmax, ymin))]
    py = [x * s + y * c + off_y for x, y in ((xmin, ymin), (xmax, ymax), (xmin, ymax), (xmax, ymin))]
    return (np.minimum.reduce(py).astype(np.float32), np.minimum.reduce(px).astype(np.float32),
            np.maximum.reduce(py).astype(np.float32), np.maximum.reduce(px).astype(np.float32))


class AugmentPlan:
    """Everything `preprocess` decides for one image without touching its pixels: the resize mode and geometry, the
    crop, the flips and the drawn jitter / rotation values (the raw draws for the numpy step, and the float32
    scalars numpy derives from them for the CUDA kernels of odt_b200/augment.py).

      mode       'bilinear' | 'nearest' | 'bicubic': resize the source to the inner rh x rw rectangle at the
                 top-left of a zh x zw canvas of `cval` (rh, rw = zh, zw unless the aspect ratio is kept);
                 'pad': the CONSTANT fill mode, the source copied into that corner as it is, rh, rw = min(h, zh),
                 min(w, zw); 'legacy': the `gt_checker_helper` fallback, the original image through TF1's
                 half-pixel-free bilinear resize to oh x ow, nothing else applied.
      crop       (ch, cw) window of oh x ow on the canvas, or None without `zoom_size` (the canvas is oh x ow)
      brightness, contrast, hue, angle: the drawn value, or None where the step did not fire."""
    __slots__ = ("h", "w", "mode", "zh", "zw", "rh", "rw", "cval", "crop", "oh", "ow", "flip_y", "flip_x",
                 "brightness", "contrast", "hue", "angle", "channels_first")

    def __init__(self, **kw):
        for k in self.__slots__:
            setattr(self, k, kw.pop(k, None))
        assert not kw, kw

    def __repr__(self):
        return "AugmentPlan(%s)" % ", ".join("%s=%r" % (k, getattr(self, k)) for k in self.__slots__)

    @property
    def rotation(self):
        """(cos, sin, x_off, y_off) float32 of the rotation, or None."""
        return None if self.angle is None else rotation_coefficients(self.angle, self.oh, self.ow)


_RESIZE = {"NEAREST_NEIGHBOR": "nearest", "BICUBIC": "bicubic"}


def plan_augment(h, w, gt, config, rng=None):
    """The pixel-free half of `preprocess` for an h x w source: argument checks, every random draw (same order, same
    conditions), the box arithmetic, the fallback decision and `pad_truth_to`.  -> (AugmentPlan, boxes), boxes None
    when gt is None.  `augment_pixels(img, plan)` then gives preprocess's image bit for bit."""
    no_boxes = gt is None
    if no_boxes:
        gt = np.zeros((0, 5), np.float32)
    oh, ow = config["output_shape"]
    rot = config.get("rotate")
    if rot is not None:                       # argument checks of :50-59
        if len(rot) != 3:
            raise ValueError('please provide "rotate" parameter as [rotate_prob, min_angle, max_angle]!')
        if not 0.0 <= rot[0] <= 1.0 or not rot[1] <= rot[2]:
            raise ValueError("rotate: prob must be in [0, 1] and min_angle <= max_angle")
    cj = config.get("color_jitter_prob")
    if cj is not None and not 0.0 <= cj <= 1.0:
        raise ValueError("color_jitter_prob can't be less than 0.0 or greater than 1.0")
    gt_copy = gt
    zoom = config.get("zoom_size")
    zh, zw = (zoom if zoom is not None else (oh, ow))
    ymin, ymax, xmin, xmax = [gt[:, i].astype(np.float32) for i in range(4)]
    fill = config.get("fill_mode", "BILINEAR")
    keep = bool(config.get("keep_aspect_ratios")) or fill == "CONSTANT"
    p = AugmentPlan(h=h, w=w, mode=_RESIZE.get(fill, "bilinear"), zh=zh, zw=zw, rh=zh, rw=zw, oh=oh, ow=ow,
                    cval=np.float32(config.get("constant_values") or 0.0), flip_y=False, flip_x=False,
                    channels_first=config.get("data_format") == "channels_first")
    if keep and fill != "CONSTANT":           # :93-114
        ratio = np.float32(min(zh / h, zw / w))
        p.rh, p.rw = (zh, int(np.float32(w) * ratio)) if zh / h < zw / w else (int(np.float32(h) * ratio), zw)
        ymin, ymax, xmin, xmax = ymin * ratio, ymax * ratio, xmin * ratio, xmax * ratio
    elif keep:                                # CONSTANT: pad only (:115-119)
        p.mode, p.rh, p.rw = "pad", min(h, zh), min(w, zw)
    else:                                     # :121-131
        ry, rx = np.float32(zh / h), np.float32(zw / w)
        ymin, ymax, xmin, xmax = ymin * ry, ymax * ry, xmin * rx, xmax * rx
    if zoom is not None:                      # :133-147
        if config.get("crop_method") == "random" and rng is not None:
            ch = int(rng.integers(0, zh - oh)) if zh > oh else 0
            cw = int(rng.integers(0, zw - ow)) if zw > ow else 0
        else:
            ch, cw = (zh - oh) // 2, (zw - ow) // 2
        p.crop = (ch, cw)
        ymin, ymax, xmin, xmax = ymin - ch, ymax - ch, xmin - cw, xmax - cw
    flip = config.get("flip_prob")
    if flip is not None and rng is not None:  # :149-173 (note the reference's "- 1." offsets)
        if rng.random() < flip[0]:
            p.flip_y = True
            ymax, ymin = oh - ymin - 1.0, oh - ymax - 1.0
        if rng.random() < flip[1]:
            p.flip_x = True
            xmax, xmin = ow - xmin - 1.0, ow - xmax - 1.0
    if cj is not None and rng is not None:    # :174-187 (deltas drawn only when the step fires, like tf.cond)
        bcs = rng.random(3)
        if bcs[0] < cj:
            p.brightness = rng.uniform(0.0, 0.3)
        if bcs[1] < cj:
            p.contrast = rng.uniform(0.8, 1.2)
        if bcs[2] < cj:
            p.hue = rng.uniform(-0.1, 0.1)
    if rot is not None and rng is not None:   # :189-196
        if rng.random() < rot[0]:
            p.angle = np.float32(rng.uniform(rot[1], rot[2]) * 3.1415926 / 180.0)
            ymin, xmin, ymax, xmax = rotate_boxes(p.angle, ymin, xmin, ymax, xmax, float(oh), float(ow))
    lim_y, lim_x = np.float32(oh - 1), np.float32(ow - 1)   # :199-218
    ymin, ymax = np.clip(ymin, 0, lim_y), np.clip(ymax, 0, lim_y)
    xmin, xmax = np.clip(xmin, 0, lim_x), np.clip(xmax, 0, lim_x)
    yc, xc = (ymin + ymax) / 2, (xmin + xmax) / 2
    m = (yc > 0) & (yc < lim_y) & (xc > 0) & (xc < lim_x)
    box = np.stack([yc[m], xc[m], (ymax - ymin)[m], (xmax - xmin)[m], gt[:, 4][m]], -1).astype(np.float32)
    if len(box) == 0 and len(gt_copy):        # gt_checker_helper (:220-225,:259-264): plain resize of the original
        p.mode, p.zh, p.zw, p.rh, p.rw, p.crop, p.flip_y, p.flip_x = "legacy", oh, ow, oh, ow, None, False, False
        p.brightness = p.contrast = p.hue = p.angle = None
        fy, fx = np.float32(oh) / np.float32(h), np.float32(ow) / np.float32(w)
        g = gt_copy.astype(np.float32)
        box = np.stack([(g[:, 0] / 2 + g[:, 1] / 2) * fy, (g[:, 2] / 2 + g[:, 3] / 2) * fx,
                        (g[:, 1] - g[:, 0]) * fy, (g[:, 3] - g[:, 2]) * fx, g[:, 4]], -1).astype(np.float32)
    pad = config.get("pad_truth_to")
    if pad:
        full = np.full((int(pad), 5), -1.0, np.float32)
        n = min(len(box), int(pad))
        full[:n] = box[:n]
        box = full
    return p, (None if no_boxes else box)


_RESIZE_FN = {"bilinear": _resize_bilinear_aligned, "nearest": _resize_nearest_aligned,
              "bicubic": _resize_bicubic_aligned}


def augment_pixels(img, plan, means=None):
    """The pixel half of `preprocess`: `img` (uint8 or float [h, w, c]) through `plan`.  `means` (3 float32) stands
    in for numpy's own channel means in the contrast step, e.g. the means the CUDA kernels computed."""
    p = plan
    if p.mode == "legacy":
        out = _resize_bilinear_legacy(img, p.oh, p.ow)
    else:
        if p.mode == "pad":
            out = np.full((p.zh, p.zw, img.shape[2]), p.cval, np.float32)
            out[:p.rh, :p.rw] = img[:p.zh, :p.zw]
        elif (p.rh, p.rw) == (p.zh, p.zw):
            out = _RESIZE_FN[p.mode](img, p.zh, p.zw)
        else:
            out = np.full((p.zh, p.zw, img.shape[2]), p.cval, np.float32)
            out[:p.rh, :p.rw] = _RESIZE_FN[p.mode](img, p.rh, p.rw)
        if p.crop is not None:
            ch, cw = p.crop
            out = out[ch:ch + p.oh, cw:cw + p.ow]
        if p.flip_y:
            out = out[::-1]
        if p.flip_x:
            out = out[:, ::-1]
        if p.brightness is not None:
            out = adjust_brightness(out, p.brightness)
        if p.contrast is not None:
            out = adjust_contrast(out, p.contrast, means)
        if p.hue is not None:
            out = adjust_hue(out, p.hue)
        if p.angle is not None:
            out = rotate_bilinear(out, p.angle)
    if p.channels_first:
        out = np.transpose(out, (2, 0, 1))
    return np.ascontiguousarray(out, np.float32)


def preprocess(img, gt, config, rng=None):
    """image_augmentor (utils/image_augmentor.py:7-233): resize (or aspect-preserving resize + constant padding) to
    `zoom_size` / `output_shape`, centre or random crop, top-down / left-right flips, colour jitter, rotation, box
    clamping and the centre-inside filter, conversion to (y_c, x_c, h, w, id), `pad_truth_to`.  Randomness comes
    from the seeded numpy generator `rng` (TF's generator is not reproducible outside TF); without one the
    random steps are skipped.  gt=None (`image_augmentor(ground_truth=None)`, the ImageNet path) returns the
    image alone.  = `plan_augment` (no pixels) + `augment_pixels`."""
    plan, box = plan_augment(img.shape[0], img.shape[1], gt, config, rng)
    out = augment_pixels(img, plan)
    return out if gt is None else (out, box)


preprocess._warned = {}


DECODE_THREADS = 4   # JPEG decoding ahead of the consumer (cv2.imdecode releases the GIL)
DECODE_AHEAD = 16    # records in flight


class BatchIterator:
    """`iterator.get_next()` of `get_generator` (utils/tfrecord_voc_utils.py:115-120): endless batches
    (images float32 [B,...], ground_truth float32 [B,pad,5]); drop_remainder, shuffle buffer, repeat.

    Records are decoded ahead on DECODE_THREADS threads and consumed in record order; the random draws (plan_augment
    per example, then the shuffle buffer's pick) happen in the consumer, in the order `preprocess` made them.  The
    shuffle buffer holds (uint8 source, AugmentPlan, boxes); the pixels are made when a batch is taken:
    `get_next()` with numpy, `get_next(device)` with the CUDA kernels of odt_b200/augment.py (the same batch, the
    images a float32 CUDA tensor in the configured layout).  The decoding threads end with the iterator (`close()`,
    a new `initialize()`, or garbage collection)."""

    def __init__(self, tfrecords, batch_size, buffer_size, config, seed=0):
        self.files = [tfrecords] if isinstance(tfrecords, str) else list(tfrecords)
        self.batch_size, self.buffer_size, self.config = int(batch_size), max(int(buffer_size), 1), dict(config)
        self.rng = np.random.default_rng(seed)
        self._it = None
        self._gpu = None

    def initialize(self):
        self.close()
        self._it = self._batches()

    def close(self):
        """Stop the decoding threads (the next get_next() starts a fresh stream, like initialize())."""
        if self._it is not None:
            self._it.close()
            self._it = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # The stream is a chain of module-level generators that hold the files, config and generator but not the
    # iterator itself, so that dropping the iterator closes the chain (and its decoding threads) at once.
    def _examples(self):
        return _voc_examples(self.files, self.config, self.rng)

    def _batches(self):
        return _batches(_shuffled(self._examples(), self.buffer_size, self.rng), self.batch_size)

    def _next_items(self):
        if self._it is None:
            self.initialize()
        return next(self._it)

    def _images(self, items, device):
        if device is None:
            return np.stack([augment_pixels(i[0], i[1]) for i in items])
        if self._gpu is None:
            from .augment import GpuAugmentor
            self._gpu = GpuAugmentor()
        return self._gpu(items, device)

    def get_next(self, device=None):
        """The next batch.  device=None: numpy images; a CUDA device: the same images as a float32 tensor there,
        made by the augmentation kernels on that device's current stream (the truth stays numpy)."""
        items = self._next_items()
        return self._images(items, device), np.stack([i[2] for i in items])


class ImageNetBatchIterator(BatchIterator):
    """`iterator.get_next()` of utils/tfrecord_imagenet_utils.py:118-123: endless batches (images float32 [B,...],
    labels int64 [B]) of ImageNet records, each image through `preprocess` without boxes."""

    def _examples(self):
        return _imagenet_examples(self.files, self.config, self.rng)


def _records(files):
    while True:  # .repeat()
        n = 0
        for path in files:
            for rec in read_records(path):
                n += 1
                yield rec
        if n == 0:
            raise RecordError("no records in %r" % (files,))


def _decoded(files, decode):
    """decode(record) of every record in order, DECODE_AHEAD records ahead on a small thread pool.  An error of the
    record stream or of a decode is raised where that record's example would have been."""
    import collections
    from concurrent.futures import ThreadPoolExecutor
    from sys import is_finalizing     # a local: module globals may be gone when the generator is finalised at exit
    src = _records(files)
    window = collections.deque()
    pool = ThreadPoolExecutor(DECODE_THREADS, thread_name_prefix="odt-decode")
    failed = False
    try:
        while True:
            while not failed and len(window) < DECODE_AHEAD:
                try:
                    rec = next(src)
                except Exception as e:          # framing error / no records: at its place in the stream
                    window.append(e)
                    failed = True
                    break
                window.append(pool.submit(decode, rec))
            item = window.popleft()
            if isinstance(item, BaseException):
                raise item
            yield item.result()
    finally:
        if not is_finalizing():     # at interpreter exit concurrent.futures has joined its workers already
            pool.shutdown(wait=True, cancel_futures=True)


def _voc_examples(files, config, rng):
    for img, gt in _decoded(files, decode_voc_example):
        yield (img,) + plan_augment(img.shape[0], img.shape[1], gt, config, rng)


def _imagenet_examples(files, config, rng):
    for img, label in _decoded(files, decode_imagenet_example):
        yield img, plan_augment(img.shape[0], img.shape[1], None, config, rng)[0], label


def _shuffled(examples, buffer_size, rng):
    buf = []
    for ex in examples:
        buf.append(ex)
        if len(buf) >= buffer_size:
            yield buf.pop(int(rng.integers(len(buf))))


def _batches(src, batch_size):
    while True:
        yield [next(src) for _ in range(batch_size)]
