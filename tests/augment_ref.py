"""The input pipeline as it was before tfrecord.preprocess was split into plan_augment + augment_pixels and the
batch iterators started to hold (uint8 source, plan, boxes): one piece of numpy per image, preprocessed as each record
was read.  tests/test_augment.py checks that the split changed nothing, bit for bit, random stream included."""
import numpy as np

from odt_b200 import tfrecord as T


def preprocess(img, gt, config, rng=None):
    """image_augmentor (utils/image_augmentor.py:7-233): resize (or aspect-preserving resize + constant padding) to
    `zoom_size` / `output_shape`, centre or random crop, top-down / left-right flips, colour jitter, rotation, box
    clamping and the centre-inside filter, conversion to (y_c, x_c, h, w, id), `pad_truth_to`.  Randomness comes
    from the seeded numpy generator `rng` (TF's generator is not reproducible outside TF); without one the
    random steps are skipped.  gt=None (`image_augmentor(ground_truth=None)`, the ImageNet path) returns the
    image alone."""
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
    img_copy, gt_copy = img, gt
    zoom = config.get("zoom_size")
    zh, zw = (zoom if zoom is not None else (oh, ow))
    h, w = img.shape[:2]
    ymin, ymax, xmin, xmax = [gt[:, i].astype(np.float32) for i in range(4)]
    fill = config.get("fill_mode", "BILINEAR")
    keep = bool(config.get("keep_aspect_ratios")) or fill == "CONSTANT"
    resize = {"NEAREST_NEIGHBOR": T._resize_nearest_aligned, "BICUBIC": T._resize_bicubic_aligned}.get(
        fill, T._resize_bilinear_aligned)
    cval = np.float32(config.get("constant_values") or 0.0)
    if keep and fill != "CONSTANT":           # :93-114
        ratio = np.float32(min(zh / h, zw / w))
        rh, rw = (zh, int(np.float32(w) * ratio)) if zh / h < zw / w else (int(np.float32(h) * ratio), zw)
        out = np.full((zh, zw, img.shape[2]), cval, np.float32)
        out[:rh, :rw] = resize(img, rh, rw)
        ymin, ymax, xmin, xmax = ymin * ratio, ymax * ratio, xmin * ratio, xmax * ratio
    elif keep:                                # CONSTANT: pad only (:115-119)
        out = np.full((zh, zw, img.shape[2]), cval, np.float32)
        out[:min(h, zh), :min(w, zw)] = img[:zh, :zw]
    else:                                     # :121-131
        out = resize(img, zh, zw)
        ry, rx = np.float32(zh / h), np.float32(zw / w)
        ymin, ymax, xmin, xmax = ymin * ry, ymax * ry, xmin * rx, xmax * rx
    if zoom is not None:                      # :133-147
        if config.get("crop_method") == "random" and rng is not None:
            ch = int(rng.integers(0, zh - oh)) if zh > oh else 0
            cw = int(rng.integers(0, zw - ow)) if zw > ow else 0
        else:
            ch, cw = (zh - oh) // 2, (zw - ow) // 2
        out = out[ch:ch + oh, cw:cw + ow]
        ymin, ymax, xmin, xmax = ymin - ch, ymax - ch, xmin - cw, xmax - cw
    flip = config.get("flip_prob")
    if flip is not None and rng is not None:  # :149-173 (note the reference's "- 1." offsets)
        if rng.random() < flip[0]:
            out = out[::-1]
            ymax, ymin = oh - ymin - 1.0, oh - ymax - 1.0
        if rng.random() < flip[1]:
            out = out[:, ::-1]
            xmax, xmin = ow - xmin - 1.0, ow - xmax - 1.0
    if cj is not None and rng is not None:    # :174-187 (deltas drawn only when the step fires, like tf.cond)
        bcs = rng.random(3)
        if bcs[0] < cj:
            out = T.adjust_brightness(out, rng.uniform(0.0, 0.3))
        if bcs[1] < cj:
            out = T.adjust_contrast(out, rng.uniform(0.8, 1.2))
        if bcs[2] < cj:
            out = T.adjust_hue(out, rng.uniform(-0.1, 0.1))
    if rot is not None and rng is not None:   # :189-196
        if rng.random() < rot[0]:
            ang = np.float32(rng.uniform(rot[1], rot[2]) * 3.1415926 / 180.0)
            out = T.rotate_bilinear(out, ang)
            ymin, xmin, ymax, xmax = T.rotate_boxes(ang, ymin, xmin, ymax, xmax, float(oh), float(ow))
    lim_y, lim_x = np.float32(oh - 1), np.float32(ow - 1)   # :199-218
    ymin, ymax = np.clip(ymin, 0, lim_y), np.clip(ymax, 0, lim_y)
    xmin, xmax = np.clip(xmin, 0, lim_x), np.clip(xmax, 0, lim_x)
    yc, xc = (ymin + ymax) / 2, (xmin + xmax) / 2
    m = (yc > 0) & (yc < lim_y) & (xc > 0) & (xc < lim_x)
    box = np.stack([yc[m], xc[m], (ymax - ymin)[m], (xmax - xmin)[m], gt[:, 4][m]], -1).astype(np.float32)
    if len(box) == 0 and len(gt_copy):        # gt_checker_helper (:220-225,:259-264): plain resize of the original
        out = T._resize_bilinear_legacy(img_copy, oh, ow)
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
    if config.get("data_format") == "channels_first":
        out = np.transpose(out, (2, 0, 1))
    if no_boxes:
        return np.ascontiguousarray(out, np.float32)
    return np.ascontiguousarray(out, np.float32), box


class BatchIterator:
    """`iterator.get_next()` of `get_generator` (utils/tfrecord_voc_utils.py:115-120): endless batches
    (images float32 [B,...], ground_truth float32 [B,pad,5]); drop_remainder, shuffle buffer, repeat."""

    def __init__(self, tfrecords, batch_size, buffer_size, config, seed=0):
        self.files = [tfrecords] if isinstance(tfrecords, str) else list(tfrecords)
        self.batch_size, self.buffer_size, self.config = int(batch_size), max(int(buffer_size), 1), dict(config)
        self.rng = np.random.default_rng(seed)
        self._it = None

    def initialize(self):
        self._it = self._batches()

    def _examples(self):
        while True:  # .repeat()
            n = 0
            for path in self.files:
                for rec in T.read_records(path):
                    n += 1
                    yield preprocess(*T.decode_voc_example(rec), self.config, self.rng)
            if n == 0:
                raise T.RecordError("no records in %r" % (self.files,))

    def _shuffled(self):
        buf = []
        for ex in self._examples():
            buf.append(ex)
            if len(buf) >= self.buffer_size:
                yield buf.pop(int(self.rng.integers(len(buf))))

    def _batches(self):
        src = self._shuffled()
        while True:
            items = [next(src) for _ in range(self.batch_size)]
            yield np.stack([i[0] for i in items]), np.stack([i[1] for i in items])

    def get_next(self):
        if self._it is None:
            self.initialize()
        return next(self._it)


class ImageNetBatchIterator(BatchIterator):
    """`iterator.get_next()` of utils/tfrecord_imagenet_utils.py:118-123: endless batches (images float32 [B,...],
    labels int64 [B]) of ImageNet records, each image through `preprocess` without boxes."""

    def _examples(self):
        while True:
            n = 0
            for path in self.files:
                for rec in T.read_records(path):
                    n += 1
                    img, label = T.decode_imagenet_example(rec)
                    yield preprocess(img, None, self.config, self.rng), label
            if n == 0:
                raise T.RecordError("no records in %r" % (self.files,))
