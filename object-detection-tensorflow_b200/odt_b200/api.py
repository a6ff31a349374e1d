"""The reference's public model surface on the H100 engine.

Same class names, constructor signature `(config, data_provider)`, config keys,
asserts and method names as the reference model scripts, so its test*.py
drivers run unchanged (SURVEY.md section 8b):
    SSD300.py:11-50,473-504   SSD512.py   RetinaNet.py:11-79,505-539
    YOLOv3.py:11-60,444-483   YOLOv2.py:11-54,305-343   FCOS.py:11-49,401-436
    PFPNetR.py:11-53,615-661  CenterNet.py:11-48,272-324
Inference (`test_one_image`) runs entirely on the hand-written GPU kernels; there is no CPU
fallback.  `train_one_epoch` runs the training step of odt_b200/train.py (PyTorch autograd over the
engine's layer list + the reference's losses + Momentum: the first stage of SURVEY 8f row 2; RetinaNet's
ImageNet-pretraining mode: the same step with the pooled-logit cross-entropy).  Extensions: `test_one_image`
accepts [B,H,W,3] (returns a list per image for B > 1), `detect_batch` / `detect_stream` / `detect_*_sharded`
expose the batched, pipelined and multi-GPU paths.
"""
import os
import sys

import numpy as np
import torch

from . import nets, tf_checkpoint
from .engine import Net, check_class_labels, init_weights

# VGG-16 classification checkpoint scope -> (kernel variable, bias variable) as the reference
# names them, typos included (SSD300.py:195-301: 'kenrel_conv2_1', 'bias_conv_3_1')
VGG16_CKPT_NAMES = {
    "conv%d/conv%d_%d" % (blk, blk, i): ("feature_extractor/" + kv, "feature_extractor/" + bv)
    for (blk, i, kv, bv) in [
        (int(e[0][4]), int(e[0][6]), e[1], e[2]) for e in nets._VGG if isinstance(e, tuple)]
}


def _as_host_tensor(images):
    """numpy / array-like / torch CPU tensor -> contiguous float32 torch tensor (no copy if possible)."""
    if isinstance(images, torch.Tensor):
        return images.to(torch.float32).contiguous()
    return torch.from_numpy(np.ascontiguousarray(images, dtype=np.float32))


def _next_batch(iterator, tr, data_format):
    """The next training batch, NHWC.  A tfrecord BatchIterator feeding a CUDA trainer augments on the trainer's
    device (get_next(device): the same batch, made by the augmentation kernels); any other iterator, and a CPU
    trainer, take the numpy batch."""
    from .tfrecord import BatchIterator
    if isinstance(iterator, BatchIterator) and tr.device.type == "cuda":
        images, truth = iterator.get_next(tr.device)
        if data_format == "channels_first":
            images = images.permute(0, 2, 3, 1)
        return images, truth
    images, truth = iterator.get_next()
    if data_format == "channels_first":
        images = np.transpose(np.asarray(images), (0, 2, 3, 1))
    return images, truth


def _precision(config):
    return config.get("precision", os.environ.get("ODT_PRECISION", "fp16"))


class _Detector:
    name = "detector"
    seed = 1

    def _common_init(self, config, data_provider):
        self._base_init(config, data_provider)
        self.nms_score_threshold = config["nms_score_threshold"]
        self.nms_max_boxes = config["nms_max_boxes"]
        self.nms_iou_threshold = config["nms_iou_threshold"]

    def _base_init(self, config, data_provider):
        assert config["mode"] in ["train", "test"]
        assert config["data_format"] in ["channels_first", "channels_last"]
        self.config = config
        self.data_provider = data_provider
        self.mode = config["mode"]
        self.data_format = config["data_format"]
        self.weight_decay = config["weight_decay"]
        self.prob = 1.0 - config["keep_prob"]
        self.batch_size = config["batch_size"] if config["mode"] == "train" else 1
        if self.mode == "train":
            self.num_train = data_provider["num_train"]
            self.num_val = data_provider["num_val"]
            self.train_generator = data_provider["train_generator"]
            self.train_initializer, self.train_iterator = self.train_generator
            if data_provider["val_generator"] is not None:
                self.val_generator = data_provider["val_generator"]
                self.val_initializer, self.val_iterator = self.val_generator
        self.precision = _precision(config)
        self.global_step = 0
        self._engines = {}
        self._weights = None
        self._bn_mode = config.get("bn_init", "tf_init")
        self.device = config.get("device", "cuda")

    # ---- engine management -------------------------------------------------
    def _build(self, batch, precision, allow_tc=True):
        raise NotImplementedError

    def engine(self, batch=1, precision=None, graph=True, allow_tc=True):
        """Build (once) the network for a fixed batch size: buffers, weights on
        the device, kernel parameter blocks, CUDA graph."""
        precision = precision or self.precision
        key = (batch, precision, allow_tc)
        if key in self._engines:
            return self._engines[key]
        net, tail = self._build(batch, precision, allow_tc)
        if self._weights is None:
            self._weights = self._initial_weights(net.vars)
        net.finalize(self._weights, tail)
        if graph:
            net.capture()
        self._engines[key] = net
        return net

    def variables(self):
        """name -> (shape, init kind) without touching the GPU."""
        return self._build_spec().vars

    def _build_spec(self):
        from .engine import Net
        Net.spec_only = True
        try:
            net, tail = self._build(1, "fp32", False)
        finally:
            Net.spec_only = False
        net.tail = tail  # never prepared: it describes the head rows (Tail.row) for the training step
        return net

    def _initial_weights(self, variables):
        w = init_weights(variables, seed=self.seed, bn_mode=self._bn_mode)
        path = self.config.get("pretraining_weight")
        if path and os.path.exists(path) and path.endswith(".npz"):
            self._load_npz_into(w, path)
        elif path and tf_checkpoint.is_checkpoint(path):
            self._load_bundle_into(w, path)
        elif path:
            # the reference throws inside NewCheckpointReader (SSD300.py:31).  BASELINE config 0 runs the driver's
            # own config (pretraining_weight './vgg_16.ckpt') with random-init VGG-16: that needs the explicit
            # opt-in config['allow_random_init'] = True or ODT_ALLOW_RANDOM_INIT=1.
            if not (self.config.get("allow_random_init") or os.environ.get("ODT_ALLOW_RANDOM_INIT") == "1"):
                raise FileNotFoundError(
                    "pretraining_weight %r is neither a TF checkpoint (V2 bundle / V1 file) nor an .npz; set "
                    "config['allow_random_init'] = True (or ODT_ALLOW_RANDOM_INIT=1) to run on the seeded random "
                    "initialisation instead" % (path,))
            sys.stderr.write("[odt_b200] pretraining weight %r not found; using the seeded random init (opt-in)\n"
                             % (path,))
        return w

    @staticmethod
    def _load_bundle_into(w, prefix, require=None):
        """Variables by their own names (checkpoints written by save_weight / the reference's
        Saver), plus the VGG-16 classification names the SSD constructors read
        (`vgg_16/convN/convN_M/{weights,biases}`, SSD300.py:195-301).  `require`: names that must be
        in the file -- `Saver.restore` fails with NotFoundError on the first variable of its list
        that the checkpoint lacks; here every missing name is reported at once."""
        r = tf_checkpoint.open_checkpoint(prefix)  # V2 bundle or V1 single file (the slim vgg_16.ckpt)
        if require is not None:
            missing = [k for k in require if not r.has_tensor(k)]
            if missing:
                raise tf_checkpoint.CheckpointError(
                    "%s lacks %d of the %d variables to restore (first: %s)" % (prefix, len(missing), len(require),
                                                                             ", ".join(missing[:3])))
            # same names, other shapes: a checkpoint of the other ResNet unit (RetinaNet's is_bottleneck) -- refused
            # before anything is restored
            shapes = r.get_variable_to_shape_map()
            wrong = [k for k in require if tuple(shapes[k]) != tuple(w[k].shape)]
            if wrong:
                raise tf_checkpoint.CheckpointError(
                    "%s holds %d of the %d variables to restore with another shape (first: %s %s, expected %s)"
                    % (prefix, len(wrong), len(require), wrong[0], tuple(shapes[wrong[0]]), tuple(w[wrong[0]].shape)))
        n = 0
        for k in (w if require is None else require):
            if r.has_tensor(k):
                t = r.get_tensor(k)
                assert tuple(t.shape) == tuple(w[k].shape), (k, t.shape, w[k].shape)
                w[k] = t.astype(np.float32)
                n += 1
        for ck_name, (kvar, bvar) in VGG16_CKPT_NAMES.items():
            for src, dst in (("vgg_16/%s/weights" % ck_name, kvar), ("vgg_16/%s/biases" % ck_name, bvar)):
                if dst in w and r.has_tensor(src):
                    t = r.get_tensor(src)
                    assert tuple(t.shape) == tuple(w[dst].shape), (src, t.shape, w[dst].shape)
                    w[dst] = t.astype(np.float32)
                    n += 1
        if n == 0:
            raise tf_checkpoint.CheckpointError("%s holds none of this model's variables" % prefix)
        return n

    @staticmethod
    def _load_npz_into(w, path):
        data = np.load(path)
        for k in data.files:
            if k in w:
                assert w[k].shape == data[k].shape, (k, w[k].shape, data[k].shape)
                w[k] = data[k].astype(np.float32)

    def set_weights(self, weights):
        """Replace all variables (dict name -> array in TF layout); rebuilds engines."""
        self._weights = {k: np.asarray(v, np.float32) for k, v in weights.items()}
        self._engines = {}

    def get_weights(self):
        if self._weights is None:
            self._weights = self._initial_weights(self.variables())
        return self._weights

    # ---- inference -----------------------------------------------------------
    def detect_batch(self, images, precision=None):
        """images: array-like [B,H,W,3] float (RGB, 0..255).  Returns a sequence of
        [scores, bbox(y1,x1,y2,x2), class_id] per image."""
        images = _as_host_tensor(images)
        assert images.dim() == 4 and images.shape[3] == 3, "expected [B,H,W,3]"
        net = self.engine(images.shape[0], precision)
        assert tuple(images.shape[1:3]) == (net.in_h, net.in_w), (images.shape, net.in_h, net.in_w)
        net.image_buf.copy_(images, non_blocking=True)  # H2D (async when the source is pinned)
        net.run()
        return net.tail.results()

    def detect_stream(self, batches, precision=None, sharded=False, consumer=None):
        """Pipelined inference over an iterable of host batches [B,H,W,3].  Per step, on the GPU's main
        stream: device copy of the staged images -> the captured forward graph (convs, decode, NMS; the NMS
        kernel writes the packed per-image records); on a side stream behind it: (sharded: ONE all-gather of the
        records) -> ONE asynchronous D2H of the records into pinned host memory.  The H2D copy of batch i+1 runs on a copy
        stream under the kernels of batch i, and the host only waits for / unpacks batch i AFTER batch i+1
        has been queued, so neither the D2H latency nor the Python work idles the GPU.  Results are yielded
        in order (the generator simply runs one batch ahead of what it yields); pinned sources make the
        H2D copies truly asynchronous.
        sharded: `batches` are this rank's image shards (one process per GPU, torch.distributed);
        consumer=None: every rank reads back and yields all ranks' detections; consumer=r: only rank r
        reads back the gathered records (the others yield their own shard's) -- the D2H volume of the job
        then grows with N, not N^2."""
        from . import dist
        from .engine import unpack_records
        it = iter(batches)
        try:
            cur = _as_host_tensor(next(it))
        except StopIteration:
            return
        net = self.engine(cur.shape[0], precision)
        assert tuple(cur.shape[1:]) == tuple(net.image_buf.shape[1:]), (cur.shape, net.image_buf.shape)
        if not hasattr(net, "_stage"):
            net._stage = [torch.empty_like(net.image_buf) for _ in range(2)]
            net._copy_stream = torch.cuda.Stream()
            net._h2d = [torch.cuda.Event() for _ in range(2)]
            net._used = [torch.cuda.Event() for _ in range(2)]
        world = dist.dist.get_world_size() if (sharded and dist.dist.is_initialized()) else 1
        rank = dist.dist.get_rank() if world > 1 else 0
        read_all = world > 1 and (consumer is None or consumer == rank)
        tail = net.tail
        rec_shape = ((world if read_all else 1) * cur.shape[0], tail.rec.shape[1])
        if getattr(net, "_rec_host", None) is None or tuple(net._rec_host[0].shape) != rec_shape:
            net._rec_host = [torch.empty(rec_shape, dtype=torch.float32).pin_memory() for _ in range(2)]
            net._rec_done = [torch.cuda.Event() for _ in range(2)]
        if world > 1 and (getattr(net, "_gathered", None) is None or net._gathered.shape[0] != world * cur.shape[0]):
            net._gathered = torch.empty((world * cur.shape[0], tail.rec.shape[1]), dtype=torch.float32,
                                        device=tail.rec.device)
        main = torch.cuda.current_stream()
        cs = net._copy_stream
        if getattr(net, "_rec_stream", None) is None:
            net._rec_stream = torch.cuda.Stream()
            net._ran, net._snapped = torch.cuda.Event(), torch.cuda.Event()
            net._rec_snap = [torch.empty_like(tail.rec) for _ in range(2)]
        rs = net._rec_stream

        def prefetch(t, slot):
            cs.wait_event(net._used[slot])
            with torch.cuda.stream(cs):
                net._stage[slot].copy_(t, non_blocking=True)
                net._h2d[slot].record(cs)

        def complete(slot):
            net._rec_done[slot].synchronize()
            return unpack_records(net._rec_host[slot].numpy().copy(), tail.p.cap)

        for ev in net._used:
            ev.record(main)
        prefetch(cur, 0)
        i, pending = 0, None
        # ODT_PIPELINE=0: one graph per batch (bench.py reads the same switch for its own loop)
        pipelined = net.graph is not None and os.environ.get("ODT_PIPELINE", "1") != "0"
        if pipelined:
            # two-stage pipeline (engine.Net.run_pipelined): decode + NMS + gather + read-back of batch i on the tail
            # stream under the first convolutions of batch i+1; the records are double-buffered by pipeline slot, so no
            # snapshot copy is needed and the body of batch i+2 waits for the read-back of batch i only
            net.capture_pipelined()

            def after_tail(t, slot_=None):
                src = t.rec
                if world > 1:
                    dist.gather_records(t.rec, out=net._gathered)
                    if read_all:
                        src = net._gathered
                net._rec_host[slot_].copy_(src, non_blocking=True)
                net._rec_done[slot_].record(torch.cuda.current_stream())

            while cur is not None:
                slot = i & 1
                main.wait_event(net._h2d[slot])
                net.image_buf.copy_(net._stage[slot], non_blocking=True)  # device-to-device
                net._used[slot].record(main)
                try:
                    nxt = _as_host_tensor(next(it))
                    assert nxt.shape == cur.shape, "all batches of a stream must share a shape"
                    prefetch(nxt, slot ^ 1)
                except StopIteration:
                    nxt = None
                net.run_pipelined(slot, lambda t, s_=slot: after_tail(t, s_))
                if pending is not None:
                    yield complete(pending)  # host work of batch i-1 while batch i runs
                pending = slot
                cur = nxt
                i += 1
            if pending is not None:
                yield complete(pending)
            return
        while cur is not None:
            slot = i & 1
            main.wait_event(net._h2d[slot])
            net.image_buf.copy_(net._stage[slot], non_blocking=True)  # device-to-device
            net._used[slot].record(main)
            try:
                nxt = _as_host_tensor(next(it))
                assert nxt.shape == cur.shape, "all batches of a stream must share a shape"
                prefetch(nxt, slot ^ 1)  # overlaps the launches below
            except StopIteration:
                nxt = None
            if pending is not None:
                main.wait_event(net._snapped)     # the previous records have been copied out of tail.rec (a ~5 us copy)
            net.run()
            net._ran.record(main)
            # snapshot + all-gather + read-back on a side stream: the next batch's kernels do not queue behind the
            # collective (which waits for the slowest rank) or the D2H copy, only behind the 0.6 MB snapshot
            rs.wait_event(net._ran)
            with torch.cuda.stream(rs):
                snap = net._rec_snap[slot]
                snap.copy_(tail.rec, non_blocking=True)
                net._snapped.record(rs)
                src = snap
                if world > 1:
                    dist.gather_records(snap, out=net._gathered)
                    if read_all:
                        src = net._gathered
                net._rec_host[slot].copy_(src, non_blocking=True)
                net._rec_done[slot].record(rs)
            if pending is not None:
                yield complete(pending)  # host work of batch i-1 while batch i runs
            pending = slot
            cur = nxt
            i += 1
        if pending is not None:
            yield complete(pending)

    detect_stream_deferred = detect_stream  # round-1 name of the deferred read-back variant

    def test_one_image(self, images):
        """ref SSD300.py:486-488: returns [scores, bbox, class_id]."""
        if self.data_format == "channels_first":
            images = np.transpose(np.asarray(images), (0, 2, 3, 1))
        res = self.detect_batch(images)
        return res[0] if len(res) == 1 else list(res)

    def detect_batch_sharded(self, images_local, consumer=None):
        """Batch-parallel multi-GPU inference: each rank runs its image shard,
        one NCCL all-gather of the fixed-size detection records follows."""
        from . import dist
        return dist.detect_sharded(self, images_local, consumer)

    def detect_stream_sharded(self, batches_local, precision=None, consumer=None):
        """detect_stream over this rank's image shards (see detect_stream)."""
        return self.detect_stream(batches_local, precision, sharded=True, consumer=consumer)

    # ---- training / checkpoints (API surface; SURVEY 8f) --------------------
    loss_kind = None  # the family's training loss: 'ssd' | 'retina' | 'yolo' | 'yolo2' | 'fcos' (engine.Tail.loss)

    def _loss_scalars(self):
        """The family's loss scalars from config, as keywords of engine.Tail.loss."""
        return {}

    def loss_forward(self, images, ground_truth, precision=None, return_info=False):
        """Forward of the per-image training loss on the head rows the inference tail reads (what it computes:
        the class's `loss_kind`).  ground_truth: [B,G,5] (y,x,h,w,id) padded with -1.  Returns float32 [B]; for
        the SSD models with return_info=True also int32 [B,3] = (#positives, #negatives, #mined negatives)."""
        images = _as_host_tensor(images)
        net = self.engine(images.shape[0], precision)
        net.image_buf.copy_(images)
        net.run()
        return net.tail.loss(net, self.loss_kind, ground_truth, return_info, **self._loss_scalars())

    def trainer(self):
        """The training state (variables as tensors, Momentum slots, BN moving statistics), created on first use."""
        if getattr(self, "_trainer", None) is None:
            from .train import GraphTrainer
            self._trainer = GraphTrainer(self, self.device if torch.cuda.is_available() else "cpu")
        return self._trainer

    def train_one_epoch(self, lr):
        """ref SSD300.py:473-484 (same loop in RetinaNet.py:476-486, YOLOv3.py:444-456, FCOS.py:401-412):
        `num_train // batch_size` steps of [train_op, loss] on the train generator; returns the mean loss.  The step
        itself is odt_b200/train.py (training-mode forward of the engine's layer list, the family's loss, backward,
        Momentum 0.9 + L2); afterwards the inference engines are rebuilt from the updated variables."""
        assert self.mode == "train", "construct the model with mode='train'"
        tr = self.trainer()
        self.train_initializer()
        num_iters = self.num_train // self.batch_size
        mean_loss = []
        for i in range(num_iters):
            images, gt = _next_batch(self.train_iterator, tr, self.data_format)
            loss = tr.step(images, gt, lr)
            sys.stdout.write("\r>> iters %d/%d loss %s" % (i, num_iters, loss))
            sys.stdout.flush()
            mean_loss.append(loss)
        sys.stdout.write("\n")
        self._weights = tr.export()
        self._engines = {}
        self.global_step = tr.global_step
        return float(np.mean(mean_loss)) if mean_loss else float("nan")

    def save_weight(self, mode, path):
        assert mode in ["latest", "best"]
        d = os.path.dirname(path)
        if d and not os.path.exists(d):
            os.makedirs(d)
            print(d, "does not exist, create it done")
        # `saver.save(sess, path, global_step=...)` (SSD300.py:499): a V2 bundle `<path>-<step>`
        out = "%s-%d" % (path, self.global_step)
        tensors = dict(self.get_weights())
        # int32 like the reference's variable (tf.get_variable('global_step', initializer=tf.constant(0)),
        # SSD300.py:43): Saver.restore does not cast, an int64 entry would fail its dtype check
        tensors["global_step"] = np.asarray(self.global_step, np.int32)
        tf_checkpoint.write_checkpoint(out, tensors)
        print("save", mode, "model in", out, "successfully")
        return out

    def load_weight(self, path):
        """`saver.restore(sess, path)` with `tf.train.Saver()` over every variable (SSD300.py:464-466,503):
        a TF checkpoint that holds ALL of this model's variables (or an .npz of any subset)."""
        w = dict(self.get_weights())
        if path.endswith(".npz"):
            self._load_npz_into(w, path)
        else:
            self._load_bundle_into(w, path, require=list(w))
            r = tf_checkpoint.open_checkpoint(path)
            if r.has_tensor("global_step"):
                self.global_step = int(r.get_tensor("global_step"))
        self.set_weights(w)
        print("load weight", path, "successfully")

    # scope whose TRAINABLE variables the backbone saver covers (YOLOv3.py:376-378 and FCOS.py:390-392:
    # 'backone'; RetinaNet.py:553-557: 'feature_extractor')
    backbone_scope = "feature_extractor"

    def pretraining_variables(self):
        """`tf.trainable_variables(scope)`: kernels, biases, gamma / beta of the backbone -- the moving
        statistics of batch normalisation are not trainable and are NOT in that saver."""
        return [k for k in self.get_weights()
                if k.startswith(self.backbone_scope + "/") and not k.endswith(("moving_mean", "moving_variance"))]

    def load_pretraining_weight(self, path):
        """`pretraining_weight_saver.restore` (YOLOv3.py:481-483, RetinaNet.py:537-539, FCOS.py:434-436):
        only the backbone's trainable variables, all of which must be in the checkpoint."""
        w = dict(self.get_weights())
        names = self.pretraining_variables()
        if path.endswith(".npz"):
            self._load_npz_into(w, path)
        else:
            self._load_bundle_into(w, path, require=names)
        self.set_weights(w)
        print("load pretraining weight", path, "successfully")

    load_pretrained_weight = load_pretraining_weight  # FCOS spelling (FCOS.py:434)


class SSD300(_Detector):
    name, input_size = "SSD300", 300
    # matching, cross-entropy, smooth-L1, hard-negative mining by NMS over the negative anchors: ref SSD300.py:345-453
    loss_kind = "ssd"

    def __init__(self, config, data_provider):
        self._common_init(config, data_provider)
        nets.check_num_classes(config)
        self.num_classes = config["num_classes"] + 1
        s = self.input_size
        self.data_shape = [s, s, 3] if config["data_format"] == "channels_last" else [3, s, s]

    def _build(self, batch, precision, allow_tc=True):
        return nets.build_ssd(self.input_size, batch, self.config, precision, self.device, allow_tc)


class SSD512(SSD300):
    name, input_size = "SSD512", 512


class RetinaNet(_Detector):
    name = "RetinaNet"
    loss_kind = "retina"  # matching + softmax focal + smooth-L1: ref RetinaNet.py:357-474

    def __init__(self, config, data_provider):
        assert len(config["data_shape"]) == 3
        self._common_init(config, data_provider)
        self.is_pretraining = bool(config["is_pretraining"])
        self.is_bottleneck = config["is_bottleneck"]
        self.block_list = config["residual_block_list"]
        self.data_shape = config["data_shape"]
        # the basic unit's first shortcut adds pool1 (init_conv_filters channels) to a 7-channel branch
        # (RetinaNet.py:277-279,621-632): TF's shape check builds that graph only for 7 (or the broadcast 1, which this
        # path does not reproduce: DESIGN.md section 1)
        if not self.is_bottleneck and config["init_conv_filters"] != 7:
            raise ValueError("is_bottleneck=False: block1_unit1 adds pool1 (init_conv_filters = %r channels) to its "
                             "7-channel conv branch; init_conv_filters must be 7" % (config["init_conv_filters"],))
        # ImageNet-pretraining mode (RetinaNet.py:61-69,120-135) classifies into num_logits classes; the configured
        # num_classes is unused there
        if not self.is_pretraining:
            nets.check_num_classes(config)
        self.num_classes = config["num_classes"] + 1
        self.gamma, self.alpha = config["gamma"], config["alpha"]

    def _build(self, batch, precision, allow_tc=True):
        if self.is_pretraining:
            return nets.build_retinanet_backbone(batch, self.config, precision, self.device, allow_tc)
        return nets.build_retinanet(batch, self.config, precision, self.device, allow_tc)

    def _loss_scalars(self):
        return {"alpha": self.alpha, "gamma": self.gamma}

    # ---- ImageNet-pretraining mode (ref RetinaNet.py:476-519) -------------------------------------------------------
    @property
    def num_logits(self):
        """Width of the pretraining-mode logits, the last unit's output channels with filters = 7 * 2^i
        (RetinaNet.py:27): 4 * filters[-1] for the bottleneck variant, filters[-1] for the basic one."""
        return (4 if self.is_bottleneck else 1) * 7 * 2 ** (len(self.block_list) - 1)

    def test_one_image(self, images):
        """Detection: [scores, bbox, class_id] (ref RetinaNet.py:505-507).  Pretraining mode: int64 [B] = the first
        maximum of the pooled logits (ref :501-503); [B,H,W,3] batches run as one engine batch."""
        if not self.is_pretraining:
            return _Detector.test_one_image(self, images)
        if self.data_format == "channels_first":
            images = np.transpose(np.asarray(images), (0, 2, 3, 1))
        net = self._classify(images)
        return net.tail.results()

    def _classify(self, images, precision=None):
        images = _as_host_tensor(images)
        assert images.dim() == 4 and images.shape[3] == 3, "expected [B,H,W,3]"
        net = self.engine(images.shape[0], precision)
        assert tuple(images.shape[1:3]) == (net.in_h, net.in_w), (images.shape, net.in_h, net.in_w)
        net.image_buf.copy_(images, non_blocking=True)
        net.run()
        return net

    def loss_forward(self, images, ground_truth, precision=None, return_info=False):
        """Detection: the focal + smooth-L1 loss per image (see _Detector.loss_forward).  Pretraining mode:
        `ground_truth` is the label vector [B] and the result is the per-image sparse softmax cross-entropy of the
        pooled logits, float32 [B], on the GPU kernel (labels outside [0, C) raise ValueError before any launch)."""
        if not self.is_pretraining:
            return _Detector.loss_forward(self, images, ground_truth, precision, return_info)
        labels = check_class_labels(ground_truth, _as_host_tensor(images).shape[0], self.num_logits)
        net = self._classify(images, precision)
        return net.tail.loss(net, labels)

    def train_one_epoch(self, lr):
        """Detection: the mean loss (see _Detector.train_one_epoch).  Pretraining mode (ref RetinaNet.py:476-486):
        (mean loss, mean accuracy) over `num_train // batch_size` steps on (images, labels) batches."""
        if not self.is_pretraining:
            return _Detector.train_one_epoch(self, lr)
        assert self.mode == "train", "construct the model with mode='train'"
        tr = self.trainer()
        self.train_initializer()
        num_iters = self.num_train // self.batch_size
        losses, accs = [], []
        for i in range(num_iters):
            images, labels = _next_batch(self.train_iterator, tr, self.data_format)
            loss, acc = tr.step(images, labels, lr)
            losses.append(loss)
            accs.append(acc)
        self._weights = tr.export()
        self._engines = {}
        self.global_step = tr.global_step
        if not losses:
            return float("nan"), float("nan")
        return float(np.mean(losses)), float(np.mean(accs))

    def save_weight(self, mode, path):
        """Detection: every variable + global_step.  Pretraining mode (ref RetinaNet.py:509-519,548-551):
        `Saver(trainable feature_extractor variables).save(path, global_step)` -> `<path>-<step>` holding those
        variables only (no BN moving statistics, no global_step)."""
        if not self.is_pretraining:
            return _Detector.save_weight(self, mode, path)
        assert mode in ["latest", "best"]
        d = os.path.dirname(path)
        if d and not os.path.exists(d):
            os.makedirs(d)
            print(d, "does not exist, create it done")
        out = "%s-%d" % (path, self.global_step)
        w = self.get_weights()
        tf_checkpoint.write_checkpoint(out, {k: w[k] for k in self.pretraining_variables()})
        print("save", mode, "model in", out, "successfully")
        return out

    def load_weight(self, path):
        """Pretraining mode: `saver.restore` with the pretraining saver -- every trainable variable must be in the
        checkpoint; the BN moving statistics keep their values."""
        if not self.is_pretraining:
            return _Detector.load_weight(self, path)
        w = dict(self.get_weights())
        if path.endswith(".npz"):
            self._load_npz_into(w, path)
        else:
            self._load_bundle_into(w, path, require=self.pretraining_variables())
        self.set_weights(w)
        print("load weight", path, "successfully")

    def load_pretraining_weight(self, path):
        """`pretraining_weight_saver.restore` (RetinaNet.py:537-539,553-555): the trainable 'feature_extractor'
        variables.  The ResNet's must all be in the checkpoint -- they are what pretraining-mode `save_weight` writes;
        the pyramid convolutions, which the reference's saver also lists but no pretraining checkpoint holds, are
        restored when present."""
        if self.is_pretraining:  # the reference builds no pretraining_weight_saver in this mode (:61-69)
            raise AttributeError("RetinaNet in the ImageNet-pretraining mode has no load_pretraining_weight; "
                                 "use load_weight")
        if path.endswith(".npz"):
            return _Detector.load_pretraining_weight(self, path)
        Net.spec_only = True
        try:
            backbone, _ = nets.build_retinanet_backbone(1, self.config, "fp32", self.device, False)
        finally:
            Net.spec_only = False
        resnet = [k for k, (_, kind) in backbone.vars.items() if kind not in ("bn_mean", "bn_var")]
        w = dict(self.get_weights())
        self._load_bundle_into(w, path, require=resnet)
        r = tf_checkpoint.open_checkpoint(path)
        for k in set(self.pretraining_variables()) - set(resnet):
            if r.has_tensor(k):
                t = r.get_tensor(k)
                assert tuple(t.shape) == tuple(w[k].shape), (k, t.shape, w[k].shape)
                w[k] = t.astype(np.float32)
        self.set_weights(w)
        print("load pretraining weight", path, "successfully")


class YOLOv3(_Detector):
    name = "YOLOv3"
    backbone_scope = "backone"  # sic: the reference's scope name (YOLOv3.py:377)
    # level / prior assignment, sigmoid-CE centre, class and objectness terms, squared log-size term, no-object
    # term: ref YOLOv3.py:115-318
    loss_kind = "yolo"

    def __init__(self, config, data_provider):
        assert len(config["data_shape"]) == 3
        nets.check_sigmoid_num_classes(config)
        nets.check_yolo_priors(config)
        self._common_init(config, data_provider)
        self.data_shape = config["data_shape"]
        self.num_classes = config["num_classes"]
        self.coord_sacle = config["coord_scale"]
        self.noobj_scale = config["noobj_scale"]
        self.obj_scale = config["obj_scale"]
        self.class_scale = config["class_scale"]
        self.num_priors = config["num_priors"]

    def _build(self, batch, precision, allow_tc=True):
        return nets.build_yolov3(batch, self.config, precision, self.device, allow_tc)

    def _loss_scalars(self):
        return {"coord_scale": self.coord_sacle, "noobj_scale": self.noobj_scale, "obj_scale": self.obj_scale,
                "class_scale": self.class_scale}


class YOLOv2(_Detector):
    name = "YOLOv2"
    backbone_scope = "backone"  # sic: the reference's scope name (YOLOv2.py:76,220)
    # YOLOv3's loss on one level, no-object IoU <= 0.6, not divided by the GT count: ref YOLOv2.py:103-181
    loss_kind = "yolo2"

    def __init__(self, config, data_provider):
        assert len(config["data_shape"]) == 3
        nets.check_yolo2_config(config)
        self._common_init(config, data_provider)
        self.data_shape = config["data_shape"]
        self.num_classes = config["num_classes"]
        self.coord_sacle = config["coord_scale"]
        self.noobj_scale = config["noobj_scale"]
        self.obj_scale = config["obj_scale"]
        self.class_scale = config["class_scale"]
        self.rescore_confidence = config["rescore_confidence"]  # read and unused, as in the reference
        self.num_priors = len(config["priors"])

    def _build(self, batch, precision, allow_tc=True):
        return nets.build_yolov2(batch, self.config, precision, self.device, allow_tc)

    def _loss_scalars(self):
        return {"coord_scale": self.coord_sacle, "noobj_scale": self.noobj_scale, "obj_scale": self.obj_scale,
                "class_scale": self.class_scale}


class FCOS(_Detector):
    name = "FCOS"
    backbone_scope = "backone"  # sic (FCOS.py:391)
    # level assignment, IoU loss, centre-ness BCE, sigmoid focal loss: ref FCOS.py:153-187,266-348
    loss_kind = "fcos"

    def __init__(self, config, data_provider):
        nets.check_sigmoid_num_classes(config)
        self._common_init(config, data_provider)
        self.data_shape = config["data_shape"]
        self.num_classes = config["num_classes"]

    def _build(self, batch, precision, allow_tc=True):
        return nets.build_fcos(batch, self.config, precision, self.device, allow_tc,
                               share_heads=self.config.get("share_heads", True))


class PFPNetR(_Detector):
    """PFPNet-R (ref PFPNetR.py): VGG-16 to conv4_3, a parallel pyramid of bilinear resizes, transposed convolutions
    and average pools, ARM / TCB / ODM heads and the two-step decode."""
    name = "PFPNetR"
    # matching in the 0.5 / 0.4 band, ARM cross-entropy with NMS hard-negative mining, ODM negatives on the raw ARM
    # logit, smooth-L1 against the anchor (ARM) and the decoded ARM box (ODM): ref PFPNetR.py:469-610
    loss_kind = "pfpnet"

    def __init__(self, config, data_provider):
        nets.check_pfpnet_config(config)
        self._common_init(config, data_provider)
        self.input_size = config["input_size"]
        self.num_classes = config["num_classes"] + 1
        s = self.input_size
        self.data_shape = [s, s, 3] if config["data_format"] == "channels_last" else [3, s, s]
        self.anchor_ratios = list(nets.PFPNET_RATIOS)
        self.num_anchors = len(self.anchor_ratios)

    def _build(self, batch, precision, allow_tc=True):
        return nets.build_pfpnet(batch, self.config, precision, self.device, allow_tc)


class CenterNet(_Detector):
    """CenterNet (ref CenterNet.py): a DLA backbone with pooled stage joins, three transposed-convolution upsampling
    paths summed at stride 4, keypoint / offset / size heads, a peak + top-k tail; trained with Adam."""
    name = "CenterNet"
    backbone_scope = "backone"  # sic (CenterNet.py:73,279)
    # Gaussian-heatmap focal loss with one sigma per image, L1 offset and size at the centre cells:
    # ref CenterNet.py:187-270
    loss_kind = "centernet"

    def __init__(self, config, data_provider):
        nets.check_centernet_config(config)
        self._base_init(config, data_provider)  # the config has no nms_* keys
        self.input_size = config["input_size"]
        s = self.input_size
        self.data_shape = [s, s, 3] if config["data_format"] == "channels_last" else [3, s, s]
        self.num_classes = config["num_classes"]
        if self.mode == "test":
            self.score_threshold = config["score_threshold"]
            self.top_k_results_output = config["top_k_results_output"]

    def _build(self, batch, precision, allow_tc=True):
        return nets.build_centernet(batch, self.config, precision, self.device, allow_tc)
