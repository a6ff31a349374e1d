"""`utils.tfrecord_imagenet_utils` of the reference, TensorFlow-free (ref utils/tfrecord_imagenet_utils.py): the input
pipeline of RetinaNet's ImageNet-pretraining mode.

`get_generator(tfrecords, batch_size, buffer_size, image_preprocess_config)` returns the reference's
`(init_op, iterator)` pair (:118-123); `iterator.get_next()` yields `(images float32 [B,H,W,3] or [B,3,H,W],
labels int64 [B])` read from TFRecord files with odt_b200.tfrecord (record framing, tf.train.Example, OpenCV JPEG
decoding, image_augmentor's geometry without boxes).  `dataset2tfrecord` (:45-97) converts a directory of class
sub-directories into `<name>_%05d-of-%05d.tfrecord` shards of (image, shape, label) records.
"""
import os
import sys

_PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "object-detection-tensorflow_b200")
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)


def get_generator(tfrecords, batch_size, buffer_size, image_preprocess_config):
    from odt_b200.tfrecord import ImageNetBatchIterator
    it = ImageNetBatchIterator(tfrecords, batch_size, buffer_size, image_preprocess_config)
    return it.initialize, it


def dataset2tfrecord(img_dir, output_dir, name, total_shards=50, seed=None):
    """ref :45-97: every file of every class sub-directory of `img_dir`, shuffled (`seed` makes the order
    reproducible), as `<name>_%05d-of-%05d.tfrecord` shards (the reference's shard arithmetic is kept).

    Class ids are the positions of the sub-directory names in sorted order.  The reference looks them up in its
    `imagenet_classname_encoder` table, which is the sorted list of the 1000 ILSVRC-2012 synsets, so the ids agree
    when `img_dir` holds exactly that set; the table itself is not shipped here.  Returns the list of shard paths."""
    import math
    import random

    import cv2
    import numpy as np
    from odt_b200.tfrecord import encode_imagenet_example, write_records
    os.makedirs(output_dir, exist_ok=True)
    classes = sorted(f for f in os.listdir(img_dir) if os.path.isdir(os.path.join(img_dir, f)))
    imglist = [(os.path.join(img_dir, c, f), cid) for cid, c in enumerate(classes)
               for f in sorted(os.listdir(os.path.join(img_dir, c)))]
    random.Random(seed).shuffle(imglist)
    num_per_shard = int(math.ceil(len(imglist)) / float(total_shards))

    def example(path, cid):
        with open(path, "rb") as f:
            data = f.read()
        img = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)   # decode_jpeg(channels=3) (:16-30)
        if img is None or img.ndim != 3 or img.shape[2] != 3:
            raise ValueError("%s is not a 3-channel image" % path)
        return encode_imagenet_example(data, img.shape, cid)

    outputfiles = []
    for shard_id in range(total_shards):
        out = os.path.join(output_dir, "%s_%05d-of-%05d.tfrecord" % (name, shard_id + 1, total_shards))
        outputfiles.append(out)
        lo, hi = shard_id * num_per_shard, min((shard_id + 1) * num_per_shard, len(imglist))
        write_records(out, (example(*imglist[i]) for i in range(lo, hi)))
    return outputfiles
