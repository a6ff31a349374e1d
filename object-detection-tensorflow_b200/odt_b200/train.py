"""Training step of SSD300 / SSD512 (SURVEY.md 8f row 2, first stage): forward in training mode, the reference's
per-image loss, backward, Momentum(0.9) + L2 weight decay -- what `train_one_epoch` runs per batch
(SSD300.py:129-155,345-453,473-484).

Scope and honesty: this is the "PyTorch autograd first" stage the survey plans.  The forward / backward convolutions
here are PyTorch's (library kernels), in fp32; the hand-written sm_90a kernels of this repository cover the
inference hot path and the loss FORWARD (csrc/loss.cu: the same value this module computes, used as a cross-check).
dgrad / wgrad kernels are the next stage.  Restated from the reference, not copied:

* graph: VGG-16 conv+bias+ReLU (no BN), conv6..conv11_2 / pred convs = conv -> BN -> (ReLU), BN in TRAINING mode
  (`tf.layers.batch_normalization(training=True)`: batch moments, eps 1e-3; moving statistics updated with momentum
  0.99 through UPDATE_OPS, the variance with Bessel's correction as the fused TF kernel reports it  [TF-sem]);
* loss per image (`_compute_one_image_loss`): every GT's arg-max anchor is positive, other anchors with best IoU > 0.5
  are positive, the rest negative; hard-negative mining = NonMaxSuppression over the negative ANCHOR boxes scored by
  their background cross-entropy (IoU 0.7, at most 3 x #positives, gradients flow through the selected scores only);
  loss = mean CE(positives) + mean CE(mined negatives) + mean smooth-L1(positives); batch mean over images;
* + weight_decay * sum(l2_loss(v)) over ALL trainable variables (kernels, biases, BN gamma / beta, the L2-norm scale),
  l2_loss(v) = sum(v^2) / 2;
* `tf.train.MomentumOptimizer(lr, 0.9)`: accum = 0.9 * accum + grad; v -= lr * accum.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import nets

BN_EPS = 1e-3
BN_MOMENTUM = 0.99
ADAM_BETA1, ADAM_BETA2, ADAM_EPS = 0.9, 0.999, 1e-8  # tf.train.AdamOptimizer defaults


def _same_pad(size, k, stride, dil=1):
    out = -(-size // stride)
    total = max((out - 1) * stride + (k - 1) * dil + 1 - size, 0)
    return total // 2, total - total // 2


def conv_same(x, kernel_hwio, bias, stride=1, dil=1):
    """tf.layers.conv2d / tf.nn.conv2d with SAME padding on NCHW activations; kernel stored HWIO like TF."""
    kh, kw = kernel_hwio.shape[0], kernel_hwio.shape[1]
    pt, pb = _same_pad(x.shape[2], kh, stride, dil)
    pl, pr = _same_pad(x.shape[3], kw, stride, dil)
    if pt or pb or pl or pr:
        x = F.pad(x, (pl, pr, pt, pb))
    return F.conv2d(x, kernel_hwio.permute(3, 2, 0, 1), bias, stride=stride, dilation=dil)


def max_pool_same(x, k, stride):
    pt, pb = _same_pad(x.shape[2], k, stride)
    pl, pr = _same_pad(x.shape[3], k, stride)
    if pt or pb or pl or pr:
        x = F.pad(x, (pl, pr, pt, pb), value=float("-inf"))
    return F.max_pool2d(x, k, stride)


class SSDTrainer:
    """Holds the trainable variables of one SSD model as torch tensors (TF layout / names), the BN moving statistics
    and the Momentum slots.  `step(images, gt, lr)` = one `sess.run([train_op, loss])`."""

    def __init__(self, model, device=None, dtype=torch.float32):
        self.model = model
        self.size = model.input_size
        self.cfg = model.config
        self.weight_decay = float(model.weight_decay)
        self.device = torch.device(device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu"))
        self.dtype = dtype
        w = model.get_weights()
        self.params, self.buffers, self.slots = {}, {}, {}
        for name, arr in w.items():
            t = torch.tensor(np.asarray(arr, np.float32), device=self.device, dtype=dtype)
            if name.endswith(("moving_mean", "moving_variance")):
                self.buffers[name] = t
            else:
                self.params[name] = t.requires_grad_(True)
                self.slots[name] = torch.zeros_like(t)
        self._anchors = None
        self.global_step = int(getattr(model, "global_step", 0))

    # ------------------------------------------------------------------ graph --
    def _bn_train(self, x, scope, stats):
        g, b = self.params[scope + "/gamma"], self.params[scope + "/beta"]
        mean = x.mean(dim=(0, 2, 3))
        var = x.var(dim=(0, 2, 3), unbiased=False)
        n = x.shape[0] * x.shape[2] * x.shape[3]
        stats.append((scope, mean.detach(), (var * (n / max(n - 1, 1))).detach()))
        inv = torch.rsqrt(var + BN_EPS) * g
        return x * inv.view(1, -1, 1, 1) + (b - mean * inv).view(1, -1, 1, 1)

    def forward_rows(self, images, stats=None):
        """images [B,H,W,3] float (RGB 0..255) -> candidate rows [B,N,25] (21 logits, ty, tx, th, tw), training-mode
        BN.  Layer / variable order follows nets.build_ssd (same names as the reference's checkpoints)."""
        P = self.params
        stats = [] if stats is None else stats
        x = torch.as_tensor(images, device=self.device, dtype=self.dtype)
        mean = torch.tensor([123.68, 116.779, 103.979], device=self.device, dtype=self.dtype)
        x = (x - mean).permute(0, 3, 1, 2)
        conv4_3 = None
        for item in nets._VGG:
            if item == "pool":
                x = max_pool_same(x, 2, 2)
                continue
            lname, kn, bnm, _ = item
            x = F.relu(conv_same(x, P["feature_extractor/" + kn], P["feature_extractor/" + bnm]))
            if lname == "conv4_3":
                conv4_3 = x
        x = max_pool_same(x, 3, 1)
        bn_idx = [0]

        def bn_scope(prefix):
            k = bn_idx[0]
            bn_idx[0] += 1
            return prefix + ("/batch_normalization" if k == 0 else "/batch_normalization_%d" % k)

        def cl(x, k, s, name, dil=1, act=True, prefix="feature_extractor"):
            y = conv_same(x, P["%s/%s/kernel" % (prefix, name)], P["%s/%s/bias" % (prefix, name)], s, dil)
            y = self._bn_train(y, bn_scope(prefix), stats)
            return F.relu(y) if act else y

        conv6 = cl(x, 3, 1, "conv6", dil=2)
        conv7 = cl(conv6, 1, 1, "conv7")
        conv8_2 = cl(cl(conv7, 1, 1, "conv8_1"), 3, 2, "conv8_2")
        conv9_2 = cl(cl(conv8_2, 1, 1, "conv9_1"), 3, 2, "conv9_2")
        conv10_2 = cl(cl(conv9_2, 1, 1, "conv10_1"), 3, 1, "conv10_2")
        conv11_2 = cl(cl(conv10_2, 1, 1, "conv11_1"), 3, 2, "conv11_2")
        feats = [conv4_3, conv7, conv8_2, conv9_2, conv10_2, conv11_2]
        if self.size == 512:
            feats.append(cl(cl(conv11_2, 1, 1, "conv12_1"), 3, 2, "conv12_2"))
        # conv4_3: x * rsqrt(max(sum_c x^2, 1e-12)) * gamma  (SSD300.py:74-83)
        f0 = feats[0]
        f0 = f0 * torch.rsqrt(torch.clamp((f0 * f0).sum(dim=1, keepdim=True), min=1e-12))
        feats[0] = f0 * P["feature_extractor/l2_norm_factor"].view(1, 1, 1, 1)
        bn_idx[0] = 0
        rows = []
        for i, f in enumerate(feats):
            p = cl(f, 3, 1, "pred%d" % (i + 1), act=False, prefix="regressor")   # conv -> BN, no activation
            B, C, H, W = p.shape
            rows.append(p.permute(0, 2, 3, 1).reshape(B, H * W * (C // 25), 25))
        self._shapes = [(f.shape[2], f.shape[3]) for f in feats]
        return torch.cat(rows, dim=1)

    def anchors(self):
        if self._anchors is None:
            scales, ratios = nets.ssd_scales(self.size), nets.ssd_ratios(self.size)
            y1x1, y2x2 = [], []
            for (h, w), s, ar in zip(self._shapes, scales, ratios):
                pri = [[s[0], s[0]], [s[1], s[1]]] + [[s[0] * (a ** 0.5), s[0] / (a ** 0.5)] for a in ar]
                pri = torch.tensor(pri, dtype=torch.float32).view(1, 1, -1, 2)
                cy = (torch.arange(h, dtype=torch.float32) + 0.5) * float(self.size) / float(h)
                cx = (torch.arange(w, dtype=torch.float32) + 0.5) * float(self.size) / float(w)
                yx = torch.stack(torch.meshgrid(cy, cx, indexing="ij"), dim=-1).view(h, w, 1, 2)
                y1x1.append((yx - pri / 2.0).reshape(-1, 2))
                y2x2.append((yx + pri / 2.0).reshape(-1, 2))
            a1 = torch.cat(y1x1).to(self.device, self.dtype)
            a2 = torch.cat(y2x2).to(self.device, self.dtype)
            self._anchors = (a1, a2, a1 / 2.0 + a2 / 2.0, a2 - a1)
        return self._anchors

    # ------------------------------------------------------------------- loss --
    @staticmethod
    def _smooth_l1(x):
        ax = x.abs()
        return torch.where(ax < 1.0, 0.5 * x * x, ax - 0.5)

    def image_loss(self, row, gt):
        """One image: row [N,25], gt [G,5] (y, x, h, w, id) padded with -1.  Returns (loss, #pos, #neg, #mined)."""
        from torchvision.ops import nms
        a1, a2, ayx, ahw = self.anchors()
        gt = torch.as_tensor(gt, device=self.device, dtype=self.dtype)
        cnt = int(torch.argmin(gt[:, 0]).item())              # first padded row (SSD300.py:347-348)
        g = gt[:cnt]
        gyx, ghw, label = g[:, 0:2], g[:, 2:4], g[:, 4].long()
        g1, g2 = gyx - ghw / 2.0, gyx + ghw / 2.0
        pconf, pyx, phw = row[:, :21], row[:, 21:23], row[:, 23:25]
        with torch.no_grad():
            i1 = torch.maximum(a1[None], g1[:, None])
            i2 = torch.minimum(a2[None], g2[:, None])
            inter = torch.clamp(i2 - i1, min=0).prod(dim=-1)
            iou = inter / (ahw.prod(dim=-1)[None] + ghw.prod(dim=-1)[:, None] - inter)
            best = torch.argmax(iou, dim=1)
            other = torch.ones(iou.shape[1], dtype=torch.bool, device=self.device)
            other[best] = False
            o_idx = torch.nonzero(other).squeeze(1)
            o_best, rg = iou[:, o_idx].max(dim=0)
            pos = o_best > 0.5
            pos_idx = torch.cat([best, o_idx[pos]])
            pos_g = torch.cat([torch.arange(cnt, device=self.device), rg[pos]])
            neg_idx = o_idx[~pos]
        num_pos, num_neg = int(pos_idx.numel()), int(neg_idx.numel())
        chosen = 3 * num_pos if num_neg > 3 * num_pos else num_neg
        neg_l = F.cross_entropy(pconf[neg_idx], torch.full((num_neg,), 20, device=self.device, dtype=torch.long),
                                reduction="none")
        with torch.no_grad():
            nbox = torch.cat([ayx[neg_idx] - ahw[neg_idx] / 2.0, ayx[neg_idx] + ahw[neg_idx] / 2.0], dim=1)
            sel = nms(nbox.float(), neg_l.detach().float(), 0.7)[:chosen]
        neg_loss = neg_l[sel].mean()
        pos_loss = F.cross_entropy(pconf[pos_idx], label[pos_g], reduction="none").mean()
        tyx = (gyx[pos_g] - ayx[pos_idx]) / ahw[pos_idx]
        thw = torch.log(ghw[pos_g] / ahw[pos_idx])
        coord = (self._smooth_l1(pyx[pos_idx] - tyx).sum(-1) + self._smooth_l1(phw[pos_idx] - thw).sum(-1)).mean()
        return neg_loss + pos_loss + coord, num_pos, num_neg, int(sel.numel())

    def total_loss(self, rows, ground_truth):
        per = [self.image_loss(rows[b], ground_truth[b])[0] for b in range(rows.shape[0])]
        data = torch.stack(per).sum() / rows.shape[0]
        l2 = sum((p * p).sum() for p in self.params.values()) * 0.5
        return data + self.weight_decay * l2, data

    # ------------------------------------------------------------------- step --
    def step(self, images, ground_truth, lr):
        stats = []
        rows = self.forward_rows(images, stats)
        loss, _ = self.total_loss(rows, ground_truth)
        grads = torch.autograd.grad(loss, list(self.params.values()))
        with torch.no_grad():
            for (name, p), gr in zip(self.params.items(), grads):
                acc = self.slots[name]
                acc.mul_(0.9).add_(gr)
                p.sub_(acc, alpha=float(lr))
            for scope, mean, var in stats:          # UPDATE_OPS: moving = moving * 0.99 + batch * 0.01
                self.buffers[scope + "/moving_mean"].mul_(BN_MOMENTUM).add_(mean, alpha=1 - BN_MOMENTUM)
                self.buffers[scope + "/moving_variance"].mul_(BN_MOMENTUM).add_(var, alpha=1 - BN_MOMENTUM)
        self.global_step += 1
        return float(loss.detach())

    def export(self):
        """name -> float32 ndarray of every variable (TF layout), for save_weight / the inference engines."""
        out = {k: v.detach().float().cpu().numpy() for k, v in self.params.items()}
        out.update({k: v.detach().float().cpu().numpy() for k, v in self.buffers.items()})
        return out


# ======================================================================================================================
# All four families through ONE graph executor: the layer list that nets.build_* describes for the inference engine
# (engine.Net in spec mode: ConvOp / PoolOp / AffineActOp (= BN + activation) / GroupNormActOp / UpsampleAddOp /
# NearestConcatOp / L2NormOp, with the reference's variable names) is replayed with differentiable torch operations.
# `training=True` normalises with batch moments (and collects them for the moving-average update), `False` with the
# moving statistics -- the latter is checked against the independent oracle restatement (oracle/nets.py) in the tests,
# which pins the executor itself.
# ======================================================================================================================
def _act(x, act):
    if act == "relu":
        return F.relu(x)
    if act == "leaky":
        return torch.maximum(x, 0.1 * x)       # YOLOv3.py:506
    return x


def tf_minimum(x, y):
    """min(x, y) with TF's Minimum gradient: a tie sends the whole gradient to x (torch.minimum splits it 0.5 / 0.5).
    FCOS.py:315-316 writes tf.minimum(GT distance, predicted distance), so at a tie the prediction gets none."""
    return torch.where(x <= y, x, y)


class GraphTrainer:
    """Training state + step of SSD300 / SSD512 / RetinaNet / YOLOv3 / YOLOv2 / FCOS (reference: SSD300.py:129-155,
    RetinaNet.py:193-222, YOLOv3.py:115-318, YOLOv2.py:103-181, FCOS.py:153-195).  Same interface as SSDTrainer."""

    def __init__(self, model, device=None, dtype=torch.float32):
        from . import engine as E
        self.model, self.cfg, self.E = model, model.config, E
        self.kind = {"SSD300": "ssd", "SSD512": "ssd", "RetinaNet": "retina", "YOLOv3": "yolo", "YOLOv2": "yolo2",
                     "FCOS": "fcos", "PFPNetR": "pfpnet", "CenterNet": "centernet"}[model.name]
        if getattr(model, "is_pretraining", False):
            self.kind = "classify"                # RetinaNet's ImageNet-pretraining mode
        self.weight_decay = float(model.weight_decay)
        self.device = torch.device(device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu"))
        self.dtype = dtype
        self.net = model._build_spec()            # unfused op list, no CUDA
        self.features = self.net.ops[-1].y        # the last tensor of the list (forward_features)
        self.row = getattr(self.net.tail, "row", None)  # floats per candidate row (engine.Tail.row)
        w = model.get_weights()
        self.params, self.buffers, self.slots = {}, {}, {}
        for name, arr in w.items():
            t = torch.tensor(np.asarray(arr, np.float32), device=self.device, dtype=dtype)
            if name.endswith(("moving_mean", "moving_variance")):
                self.buffers[name] = t
            else:
                self.params[name] = t.requires_grad_(True)
                self.slots[name] = torch.zeros_like(t)
        self.global_step = int(getattr(model, "global_step", 0))
        self._anchor_cache = None
        # CenterNet trains with tf.train.AdamOptimizer (CenterNet.py:154): its slots `<var>/Adam` (m) and `<var>/Adam_1`
        # (v) and the non-slot accumulators beta1_power / beta2_power, which start at beta1 / beta2
        self.adam = self.kind == "centernet"
        if self.adam:
            self.slots = {k + "/Adam": torch.zeros_like(v) for k, v in self.params.items()}
            self.slots.update({k + "/Adam_1": torch.zeros_like(v) for k, v in self.params.items()})
            self.beta1_power, self.beta2_power = ADAM_BETA1, ADAM_BETA2
        # CUDA, fp32 rows: the data term is the family's loss-gradient kernel (csrc/loss.cu) behind one autograd
        # Function; the CPU (and float64) keep the restatement below, which the kernels are tested against
        self._loss_kernels = None
        if self.kind in ("ssd", "retina", "yolo", "yolo2", "fcos", "pfpnet", "centernet") and self.device.type == "cuda" \
                and dtype == torch.float32:
            self._loss_kernels = LossKernels(self)
        if self.kind == "ssd":
            self._ssd = SSDTrainer.__new__(SSDTrainer)   # borrows the SSD loss / anchors
            self._ssd.device, self._ssd.dtype, self._ssd.size, self._ssd._anchors = self.device, dtype, model.input_size, None
            self._ssd._shapes = [(h, w) for h, w, _ in self.net.levels]

    # ------------------------------------------------------------------ graph --
    def _bn(self, x, scope, training, stats):
        g, b = self.params[scope + "/gamma"], self.params[scope + "/beta"]
        if training:
            mean = x.mean(dim=(0, 2, 3))
            var = x.var(dim=(0, 2, 3), unbiased=False)
            n = x.shape[0] * x.shape[2] * x.shape[3]
            stats.append((scope, mean.detach(), (var * (n / max(n - 1, 1))).detach()))
        else:
            mean, var = self.buffers[scope + "/moving_mean"], self.buffers[scope + "/moving_variance"]
        inv = torch.rsqrt(var + BN_EPS) * g
        return x * inv.view(1, -1, 1, 1) + (b - mean * inv).view(1, -1, 1, 1)

    def forward_rows(self, images, training=True, stats=None):
        """images [B,H,W,3] -> candidate rows [B,N,row] in the layout of DESIGN.md section 2."""
        _, rows = self._replay(images, training, stats)
        return rows.view(rows.shape[0], rows.shape[1] // self.row, self.row)

    def forward_features(self, images, training=True, stats=None):
        """images [B,H,W,3] -> the last tensor of the layer list, NCHW (pretraining mode: the last bottleneck's
        conv + shortcut sum that the classification tail pools)."""
        val, _ = self._replay(images, training, stats)
        return val[id(self.features)]

    def _replay(self, images, training, stats):
        """The layer list with torch ops -> ({id(Act): NCHW value}, head rows [B, N*row])."""
        E, P = self.E, self.params
        stats = [] if stats is None else stats
        x0 = torch.as_tensor(images, device=self.device, dtype=self.dtype)
        if self.kind == "centernet":               # (x / 255 - mean) / std, CenterNet.py:53-67
            from . import nets as NN
            mean = torch.tensor(NN.CENTERNET_MEAN, device=self.device, dtype=self.dtype)
            std = torch.tensor(NN.CENTERNET_STD, device=self.device, dtype=self.dtype)
            x0 = ((x0 / 255.0 - mean) / std).permute(0, 3, 1, 2)
        else:
            mean = torch.tensor([123.68, 116.779, 103.979], device=self.device, dtype=self.dtype)
            x0 = (x0 - mean).permute(0, 3, 1, 2)
        B = x0.shape[0]
        N = sum(h * w * a for h, w, a in self.net.levels)
        rows = torch.zeros((B, N * (self.row or 0)), device=self.device, dtype=self.dtype)
        val = {}
        for op in self.net.ops:
            if isinstance(op, E.PhaseConvOp):          # tf.layers.conv2d_transpose(4, 2, 'same') + BN
                k = P[op.kernel].permute(3, 2, 0, 1)   # [4, 4, out, in] -> [in, out, 4, 4]
                y = F.conv_transpose2d(val[id(op.x)], k, P[op.bias], stride=2, padding=1)
                val[id(op.y)] = _act(self._bn(y, op.bn, training, stats), op.act)
            elif isinstance(op, E.ConvOp):
                if op.is_image:
                    x = x0
                elif op.x.parts:                    # engine.Net.concat: the slices in channel order
                    x = torch.cat([val[id(v)] for v in op.x.parts], dim=1)
                else:
                    x = val[id(op.x)]
                y = conv_same(x, P[op.kernel], P[op.bias] if op.bias else None, op.stride, op.dil)
                if op.bn:
                    y = self._bn(y, op.bn, training, stats)
                y = _act(y, op.act)
                if op.residual is not None:
                    y = y + val[id(op.residual)]
                if op.head is None:
                    val[id(op.y)] = y
                    continue
                lvl_off, col, group, gstride, A = op.head
                Bc, C, H, W = y.shape
                n = torch.arange(C, device=self.device)
                ch = (n // group) * gstride + (n % group) if group > 0 else n
                pix = torch.arange(H * W, device=self.device)
                idx = ((lvl_off + pix * A) * self.row + col).view(-1, 1) + ch.view(1, -1)
                rows = rows.index_add(1, idx.reshape(-1), y.permute(0, 2, 3, 1).reshape(Bc, -1))
            elif isinstance(op, E.PoolOp):
                val[id(op.y)] = max_pool_same(val[id(op.x)], op.k, op.stride)
            elif isinstance(op, E.AffineActOp):
                x = val[id(op.x)]
                val[id(op.y)] = _act(x if op.bn is None else self._bn(x, op.bn, training, stats), op.act)
            elif isinstance(op, E.GroupNormActOp):
                x = val[id(op.x)]
                y = F.group_norm(x, op.groups, P[op.gn + "/gamma"], P[op.gn + "/beta"], eps=E.GN_EPS)
                val[id(op.y)] = _act(y, op.act)
            elif isinstance(op, E.L2NormOp):
                x = torch.cat([val[id(v)] for v in op.x.parts], dim=1) if op.x.parts else val[id(op.x)]
                x = x * torch.rsqrt(torch.clamp((x * x).sum(dim=1, keepdim=True), min=1e-12))
                val[id(op.y)] = x * P[op.var].view(1, 1, 1, 1)
            elif isinstance(op, E.UpsampleAddOp):
                top, a = val[id(op.top)], val[id(op.a)]
                val[id(op.y)] = a + _resize_bilinear_legacy(top, a.shape[2], a.shape[3])
            elif isinstance(op, E.NearestConcatOp):
                a, b = val[id(op.a)], val[id(op.b)]
                val[id(op.y)] = torch.cat([a, _resize_nearest_legacy(b, a.shape[2], a.shape[3])], dim=1)
            elif isinstance(op, E.PixelShuffleOp):     # the transposed convolution (+ lateral) (+ ReLU)
                y = val[id(op.x)]
                if op.residual is not None:
                    y = y + val[id(op.residual)]
                val[id(op.y)] = _act(y, op.act)
            elif isinstance(op, E.ResizeOp):           # resize_bilinear(align_corners=True): (in-1)/(out-1) scale
                y = F.interpolate(val[id(op.x)], size=(op.y.H, op.y.W), mode="bilinear", align_corners=True)
                val[id(op.y)] = y
                if op.out2 is not None:
                    val[id(op.out2)] = y
            elif isinstance(op, E.AvgPoolOp):          # 2x2/2 SAME: partial windows divided by their cells inside
                val[id(op.y)] = F.avg_pool2d(val[id(op.x)], 2, 2, ceil_mode=True, count_include_pad=False)
            elif isinstance(op, E.DlaJoinOp):          # a + b, or max_pool(a) + avg_pool(b), 2x2/2 SAME
                a, b = val[id(op.a)], val[id(op.b)]
                if op.pooled:
                    a = max_pool_same(a, 2, 2)
                    b = F.avg_pool2d(b, 2, 2, ceil_mode=True, count_include_pad=False)
                val[id(op.y)] = a + b
            else:
                raise TypeError(type(op))
        return val, rows

    # ------------------------------------------------------------------ losses --
    def _softmax_anchors(self):
        if self._anchor_cache is None:
            if self.kind == "ssd":
                self._anchor_cache = self._ssd.anchors()
            else:
                from . import nets as NN
                sizes = [32, 64, 128, 256, 512]
                Wd = self.cfg["data_shape"][1]
                y1x1, y2x2 = [], []
                for (h, w, _), size in zip(self.net.levels, sizes):
                    rate = float(np.float32(np.float32(Wd) / np.float32(h)))
                    pri = [[s * size * (r ** 0.5), s * size / (r ** 0.5)] for r in [1, 1 / 2, 2]
                           for s in [2 ** 0, 2 ** (1 / 3), 2 ** (2 / 3)]]
                    pri = torch.tensor(pri, dtype=torch.float32).view(1, 1, -1, 2)
                    cy = (torch.arange(h, dtype=torch.float32) + 0.5) * rate
                    cx = (torch.arange(w, dtype=torch.float32) + 0.5) * rate
                    yx = torch.stack(torch.meshgrid(cy, cx, indexing="ij"), dim=-1).view(h, w, 1, 2)
                    y1x1.append((yx - pri / 2.0).reshape(-1, 2))
                    y2x2.append((yx + pri / 2.0).reshape(-1, 2))
                a1 = torch.cat(y1x1).to(self.device, self.dtype)
                a2 = torch.cat(y2x2).to(self.device, self.dtype)
                self._anchor_cache = (a1, a2, a1 / 2.0 + a2 / 2.0, a2 - a1)
        return self._anchor_cache

    def retina_image_loss(self, row, gt):
        """RetinaNet.py:357-474: per-GT arg-max anchors + IoU > 0.5 positive, < 0.4 negative, between ignored; softmax
        focal loss (alpha 0.25 for both, p clipped to [1e-8, 1]) summed / #positives + mean smooth-L1."""
        a1, a2, ayx, ahw = self._softmax_anchors()
        alpha, gamma = float(self.cfg["alpha"]), float(self.cfg["gamma"])
        gt = torch.as_tensor(gt, device=self.device, dtype=self.dtype)
        cnt = int(torch.argmin(gt[:, 0]).item())
        g = gt[:cnt]
        gyx, ghw, label = g[:, 0:2], g[:, 2:4], g[:, 4].long()
        g1, g2 = gyx - ghw / 2.0, gyx + ghw / 2.0
        pconf, pyx, phw = row[:, :21], row[:, 21:23], row[:, 23:25]
        with torch.no_grad():
            inter = torch.clamp(torch.minimum(a2[None], g2[:, None]) - torch.maximum(a1[None], g1[:, None]), min=0).prod(-1)
            iou = inter / (ahw.prod(-1)[None] + ghw.prod(-1)[:, None] - inter)
            best = torch.argmax(iou, dim=1)
            other = torch.ones(iou.shape[1], dtype=torch.bool, device=self.device)
            other[best] = False
            o_idx = torch.nonzero(other).squeeze(1)
            o_best, rg = iou[:, o_idx].max(dim=0)
            pos, neg = o_best > 0.5, o_best < 0.4
            pos_idx = torch.cat([best, o_idx[pos]])
            pos_g = torch.cat([torch.arange(cnt, device=self.device), rg[pos]])
            neg_idx = o_idx[neg]
        pp = torch.softmax(pconf[pos_idx], dim=-1).gather(1, label[pos_g].view(-1, 1)).squeeze(1).clamp(1e-8, 1.0)
        npb = torch.softmax(pconf[neg_idx], dim=-1)[:, 20].clamp(1e-8, 1.0)
        conf = (-(alpha * (1 - pp) ** gamma * torch.log(pp)).sum() - (alpha * (1 - npb) ** gamma * torch.log(npb)).sum()) \
            / pos_idx.numel()
        tyx = (gyx[pos_g] - ayx[pos_idx]) / ahw[pos_idx]
        thw = torch.log(ghw[pos_g] / ahw[pos_idx])
        sl1 = SSDTrainer._smooth_l1
        coord = (sl1(pyx[pos_idx] - tyx).sum(-1) + sl1(phw[pos_idx] - thw).sum(-1)).mean()
        return conf + coord

    def fcos_image_loss(self, row, gt):
        """FCOS.py:153-187,266-348 for one image: GT -> levels by sqrt(h*w) (inclusive, overlapping bounds), per level the
        inside-box targets with the minimal-area rule, -log IoU, centre-ness BCE over every cell, sigmoid focal loss,
        each level normalised by its number of positive class cells."""
        gt = torch.as_tensor(gt, device=self.device, dtype=self.dtype)
        cnt = int(torch.argmin(gt[:, 0]).item())
        g = gt[:cnt]
        size = torch.sqrt(g[:, 2] * g[:, 3])
        sel = [size <= 64, (size >= 64) & (size <= 128), (size >= 128) & (size <= 256), (size >= 256) & (size <= 512),
               size >= 512]
        nc = self.row - 5
        total, off = 0.0, 0
        for (h, w, _), m, s in zip(self.net.levels, sel, [8, 16, 32, 64, 128]):
            r = row[off:off + h * w].view(h, w, self.row)
            off += h * w
            if not bool(m.any()):
                continue
            gl = g[m]
            cls, ctr, reg = r[..., :nc], r[..., nc], r[..., nc + 1:nc + 5]
            with torch.no_grad():
                gy, gx, gh, gw = [gl[:, i] / s for i in range(4)]
                cid = gl[:, 4].long()
                y1, y2, x1, x2 = gy - gh / 2.0, gy + gh / 2.0, gx - gw / 2.0, gx + gw / 2.0
                yy = torch.arange(h, device=self.device, dtype=self.dtype).view(h, 1, 1)
                xx = torch.arange(w, device=self.device, dtype=self.dtype).view(1, w, 1)
                zero = torch.zeros((h, w, 1), device=self.device, dtype=self.dtype)
                dl, dr, dt, db = (xx - x1) + zero, (x2 - xx) + zero, (yy - y1) + zero, (y2 - yy) + zero
                heat = ((dt > 0) & (db > 0) & (dl > 0) & (dr > 0)).to(self.dtype)
                dl, dr, dt, db = dl * heat, dr * heat, dt * heat, db * heat
                loc = heat.max(dim=-1).values
                area = (dl + dr) * (dt + db)
                amin = (area + (1.0 - heat) * 1e8).min(dim=-1, keepdim=True).values
                dmask = (area == amin).to(self.dtype) * loc[..., None]
                dl, dr, dt, db = [(d * dmask).max(dim=-1).values for d in (dl, dr, dt, db)]
                lrmin, tbmin = torch.minimum(dl, dr), torch.minimum(dt, db)
                lrmax, tbmax = torch.maximum(dl, dr), torch.maximum(dt, db)
                cgt = torch.sqrt(lrmin * tbmin / (lrmax * tbmax + 1e-12))
                hgt = torch.zeros((h, w, nc), device=self.device, dtype=self.dtype)
                for c in torch.unique(cid).tolist():
                    hgt[..., c] = heat[..., cid == c].max(dim=-1).values
            p = torch.exp(reg)
            pl, pr, pt, pb = p[..., 0], p[..., 1], p[..., 2], p[..., 3]
            inter = (tf_minimum(dl, pl) + tf_minimum(dr, pr)) * (tf_minimum(dt, pt) + tf_minimum(db, pb))
            union = (dl + dr) * (dt + db) + (pl + pr) * (pt + pb) - inter
            iou_loss = (-torch.log(inter / (union + 1e-12) + 1e-12) * loc).sum()
            center = F.binary_cross_entropy_with_logits(ctr, cgt, reduction="sum")
            sg, ls = torch.sigmoid(cls), F.logsigmoid(cls)
            pos = (-0.25 * (1.0 - sg) ** 2 * ls * hgt).sum()
            neg = (-0.25 * sg ** 2 * (-cls + ls) * (1.0 - hgt)).sum()
            total = total + (iou_loss + pos + neg + center) / hgt.sum()
        return total

    def _yolo_level(self, r, pri, g, norm, clamp=False):
        """One YOLO level's matching of the image's GT g: the GT divided by `norm`, its cell (clamped to the grid for
        YOLOv2, as the kernels do), the first-maximum prior by unclamped IoU at that cell (YOLOv3.py:160-200)."""
        h, w = r.shape[0], r.shape[1]
        with torch.no_grad():
            gn = g / torch.tensor([norm] * 4 + [1.0], device=self.device, dtype=self.dtype)
            gyx, ghw, lab = gn[:, :2], gn[:, 2:4], gn[:, 4].long()
            fl = torch.floor(gyx).long()
            if clamp:
                fl = torch.stack([fl[:, 0].clamp(0, h - 1), fl[:, 1].clamp(0, w - 1)], dim=1)
            ayx = (fl.to(self.dtype) + 0.5)[:, None, :]
            a1, a2 = ayx - pri[None] / 2, ayx + pri[None] / 2
            g1, g2 = (gyx - ghw / 2.0)[:, None, :], (gyx + ghw / 2.0)[:, None, :]
            inter = (torch.minimum(g2, a2) - torch.maximum(g1, a1)).prod(-1)        # not clamped (:171-173)
            iou = inter / (pri.prod(-1)[None] + (g2 - g1).prod(-1) - inter)
            mx, idx = iou.max(dim=-1)
        return dict(r=r, pri=pri, gyx=gyx, ghw=ghw, lab=lab, fl=fl, g1=g1[:, 0], g2=g2[:, 0], idx=idx, mx=mx, h=h, w=w)

    def _yolo_terms(self, L_, m, nc, thr, acc):
        """acc = (coord, class, obj, noobj) sums plus one level's terms: the positive terms of the GTs that mask m
        selects, the no-object term of every (cell, prior) whose cell holds no GT and whose best IoU with the GTs is
        <= thr."""
        r, pri = L_["r"], L_["pri"]
        bce = F.binary_cross_entropy_with_logits
        coord, cls_l, obj_l, noobj = acc
        gi = torch.nonzero(m).squeeze(1)
        if gi.numel():
            rws = r[L_["fl"][gi, 0], L_["fl"][gi, 1], L_["idx"][gi]]                 # [n,row]
            tyx = L_["gyx"][gi] - torch.floor(L_["gyx"][gi])
            thw = torch.log(L_["ghw"][gi] / pri[L_["idx"][gi]])
            coord = coord + bce(rws[:, nc:nc + 2], tyx, reduction="sum") \
                + 0.5 * ((rws[:, nc + 2:nc + 4] - thw) ** 2).sum()
            cls_l = cls_l + bce(rws[:, :nc], F.one_hot(L_["lab"][gi], nc).to(self.dtype), reduction="sum")
            obj_l = obj_l + bce(rws[:, nc + 4], torch.ones_like(rws[:, nc + 4]), reduction="sum")
        h, w, a = L_["h"], L_["w"], pri.shape[0]
        with torch.no_grad():
            occ = torch.zeros((h, w), dtype=torch.bool, device=self.device)
            occ[L_["fl"][:, 0], L_["fl"][:, 1]] = True
            cy = (torch.arange(h, device=self.device, dtype=self.dtype) + 0.5).view(h, 1, 1, 1).expand(h, w, a, 1)
            cx = (torch.arange(w, device=self.device, dtype=self.dtype) + 0.5).view(1, w, 1, 1).expand(h, w, a, 1)
            ayx = torch.cat([cy, cx], dim=-1)
            yx_nb = ayx - pri.view(1, 1, a, 2) / 2.0        # really y1x1, re-used as a centre (:249-262)
            hw_nb = ayx + pri.view(1, 1, a, 2) / 2.0        # really y2x2, re-used as a size
            b1 = (yx_nb - hw_nb / 2.0)[..., None, :]
            b2 = (yx_nb + hw_nb / 2.0)[..., None, :]
            gg1, gg2 = L_["g1"].view(1, 1, 1, -1, 2), L_["g2"].view(1, 1, 1, -1, 2)
            inter = (torch.minimum(gg2, b2) - torch.maximum(gg1, b1)).prod(-1)
            iou = (inter / ((b2 - b1).prod(-1) + (gg2 - gg1).prod(-1) - inter)).max(dim=-1).values
            mask = ((iou <= thr) & (~occ)[..., None]).to(self.dtype)
        noobj = noobj + (bce(r[..., nc + 4], torch.zeros_like(r[..., nc + 4]), reduction="none") * mask).sum()
        return coord, cls_l, obj_l, noobj

    def _yolo_scales(self):
        return (float(self.cfg["coord_scale"]), float(self.cfg["noobj_scale"]), float(self.cfg["obj_scale"]),
                float(self.cfg["class_scale"]))

    def yolo_image_loss(self, row, gt):
        """YOLOv3.py:115-318 for one image, quirks kept (see oracle/loss.py::yolo_image_loss): returns pos_loss + neg_loss."""
        nc = self.row - 5
        cs, ns, os_, ks = self._yolo_scales()
        gt = torch.as_tensor(gt, device=self.device, dtype=self.dtype)
        cnt = int(torch.argmin(gt[:, 0]).item())
        g = gt[:cnt]
        norm, pstride = [32.0, 16.0, 8.0], [8.0, 16.0, 32.0]
        lv, off = [], 0
        for k, (h, w, a) in enumerate(self.net.levels):
            r = row[off:off + h * w * a].view(h, w, a, self.row)
            off += h * w * a
            pri = torch.tensor(self.cfg["priors"][k], device=self.device, dtype=self.dtype) / pstride[k]
            lv.append(self._yolo_level(r, pri, g, norm[k]))
        m1 = (lv[0]["mx"] > lv[1]["mx"]) & (lv[0]["mx"] > lv[2]["mx"])
        m2 = (lv[1]["mx"] > lv[0]["mx"]) & (lv[1]["mx"] > lv[2]["mx"])
        m3 = ~(m1 | m2)
        acc = (0.0, 0.0, 0.0, 0.0)
        for L_, m in zip(lv, (m1, m2, m3)):
            acc = self._yolo_terms(L_, m, nc, 0.5, acc)
        coord, cls_l, obj_l, noobj = acc
        ng = float(cnt)
        return (cs * coord + ks * cls_l + os_ * obj_l) / ng + ns * noobj / ng

    def yolo2_image_loss(self, row, gt):
        """YOLOv2.py:105-173 for one image: the YOLOv3 terms on its one level (GT / 32, priors in grid cells, the GT's
        cell clamped to the grid), the no-object term where the best IoU <= 0.6; cs * coord + ks * class + os * obj +
        ns * noobj, NOT divided by the GT count -- an image without boxes gets the no-object term of every row."""
        nc = self.row - 5
        cs, ns, os_, ks = self._yolo_scales()
        gt = torch.as_tensor(gt, device=self.device, dtype=self.dtype)
        cnt = int(torch.argmin(gt[:, 0]).item())
        if cnt == 0:  # no GT: no positive term, and every row is a no-object row (YOLOv2.py:155-171 over zero GTs)
            obj = row[:, nc + 4]
            return ns * F.binary_cross_entropy_with_logits(obj, torch.zeros_like(obj), reduction="sum")
        g = gt[:cnt]
        (h, w, a), = self.net.levels
        pri = torch.tensor(self.cfg["priors"], device=self.device, dtype=self.dtype)
        L_ = self._yolo_level(row.view(h, w, a, self.row), pri, g, 32.0, clamp=True)
        every = torch.ones(cnt, dtype=torch.bool, device=self.device)
        coord, cls_l, obj_l, noobj = self._yolo_terms(L_, every, nc, 0.6, (0.0, 0.0, 0.0, 0.0))
        return cs * coord + ks * cls_l + os_ * obj_l + ns * noobj

    def _pfpnet_anchors(self):
        """_get_abbox of PFPNetR.py:447-467 over the engine's levels: (y1x1, y2x2, yx, hw), each [N, 2]."""
        if self._anchor_cache is None:
            from . import nets as NN
            y1x1, y2x2 = [], []
            for (h, w, _), s in zip(self.net.levels, NN.PFPNET_STRIDES):
                pri = torch.tensor([[4 * s * (r ** 0.5), 4 * s / (r ** 0.5)] for r in NN.PFPNET_RATIOS],
                                   dtype=torch.float32).view(1, 1, -1, 2)
                cy = (torch.arange(h, dtype=torch.float32) + 0.5) * float(s)
                cx = (torch.arange(w, dtype=torch.float32) + 0.5) * float(s)
                yx = torch.stack(torch.meshgrid(cy, cx, indexing="ij"), dim=-1).view(h, w, 1, 2)
                y1x1.append((yx - pri / 2.0).reshape(-1, 2))
                y2x2.append((yx + pri / 2.0).reshape(-1, 2))
            a1 = torch.cat(y1x1).to(self.device, self.dtype)
            a2 = torch.cat(y2x2).to(self.device, self.dtype)
            self._anchor_cache = (a1, a2, a1 / 2.0 + a2 / 2.0, a2 - a1)
        return self._anchor_cache

    def pfpnet_image_loss(self, row, gt):
        """PFPNetR.py:469-610 for one image: row [N, 31] = [ODM logits(21), ODM t(4), ARM logits(2), ARM t(4)].  Per-GT
        arg-max anchors + IoU > 0.5 positive, < 0.4 negative; ARM: positives' cross-entropy to 0 and smooth-L1 to the
        anchor targets, hard negatives by NMS (IoU 0.7, min(#neg, 3 #pos)) scored by their cross-entropy to 1; ODM: the
        mined negatives whose raw ARM logit 1 is < 0.99, cross-entropy to 20; positives' cross-entropy to their class
        and smooth-L1 to targets from the decoded ARM box, differentiated through it.  A mean over no element is 0
        (csrc/loss.cu, DESIGN.md section 7)."""
        from torchvision.ops import nms
        a1, a2, ayx, ahw = self._pfpnet_anchors()
        gt = torch.as_tensor(gt, device=self.device, dtype=self.dtype)
        cnt = int(torch.argmin(gt[:, 0]).item())
        g = gt[:cnt]
        gyx, ghw, label = g[:, 0:2], g[:, 2:4], g[:, 4].long()
        g1, g2 = gyx - ghw / 2.0, gyx + ghw / 2.0
        oc, ot, ac, at = row[:, :21], row[:, 21:25], row[:, 25:27], row[:, 27:31]
        N = row.shape[0]
        dev = self.device
        with torch.no_grad():
            inter = torch.clamp(torch.minimum(a2[None], g2[:, None]) - torch.maximum(a1[None], g1[:, None]), min=0).prod(-1)
            iou = inter / (ahw.prod(-1)[None] + ghw.prod(-1)[:, None] - inter)
            best = torch.argmax(iou, dim=1) if cnt else torch.zeros(0, dtype=torch.long, device=dev)
            other = torch.ones(N, dtype=torch.bool, device=dev)
            other[best] = False
            o_idx = torch.nonzero(other).squeeze(1)
            if cnt:
                o_best, rg = iou[:, o_idx].max(dim=0)
            else:                                  # reduce_max over no GT: every anchor is a negative
                o_best = torch.full((o_idx.numel(),), -float("inf"), device=dev, dtype=self.dtype)
                rg = torch.zeros(o_idx.numel(), dtype=torch.long, device=dev)
            pos, neg = o_best > 0.5, o_best < 0.4
            pos_idx = torch.cat([best, o_idx[pos]])
            pos_g = torch.cat([torch.arange(cnt, device=dev), rg[pos]])
            neg_idx = o_idx[neg]

        def mean0(x):
            return x.sum() / x.numel() if x.numel() else x.sum()

        P, nneg = int(pos_idx.numel()), int(neg_idx.numel())
        chosen = 3 * P if nneg > 3 * P else nneg
        neg_arm = F.cross_entropy(ac[neg_idx], torch.ones(nneg, dtype=torch.long, device=dev), reduction="none")
        with torch.no_grad():
            nbox = torch.cat([ayx[neg_idx] - ahw[neg_idx] / 2.0, ayx[neg_idx] + ahw[neg_idx] / 2.0], dim=1)
            sel = nms(nbox.float(), neg_arm.detach().float(), 0.7)[:chosen]
            mined = neg_idx[sel]
            mined_odm = mined[ac[mined, 1] < 0.99]
        sl1 = SSDTrainer._smooth_l1
        arm = mean0(neg_arm[sel]) + mean0(F.cross_entropy(ac[pos_idx], torch.zeros(P, dtype=torch.long, device=dev),
                                                          reduction="none"))
        pa, pyx, phw = ahw[pos_idx], ayx[pos_idx], at[pos_idx]
        tyx, thw = (gyx[pos_g] - pyx) / pa, torch.log(ghw[pos_g] / pa)
        arm = arm + mean0(sl1(phw[:, :2] - tyx).sum(-1) + sl1(phw[:, 2:] - thw).sum(-1))
        arm_yx = phw[:, :2] * pa + pyx
        arm_hw = torch.exp(phw[:, 2:]) * pa
        oyx, ohw = (gyx[pos_g] - arm_yx) / arm_hw, torch.log(ghw[pos_g] / arm_hw)
        odm = mean0(F.cross_entropy(oc[mined_odm], torch.full((mined_odm.numel(),), 20, dtype=torch.long, device=dev),
                                    reduction="none"))
        odm = odm + mean0(F.cross_entropy(oc[pos_idx], label[pos_g], reduction="none"))
        odm = odm + mean0(sl1(ot[pos_idx, :2] - oyx).sum(-1) + sl1(ot[pos_idx, 2:] - ohw).sum(-1))
        return arm + odm

    def centernet_image_loss(self, row, gt):
        """CenterNet.py:187-270 for one image: row [H*W, C + 4] = [keypoint logits, dy, dx, h, w].  GT / 4, centres
        floored to their cells (clamped into the grid); one sigma, the least CornerNet radius over every GT; the per-class
        maximum of exp(-d^2 / 2 sigma^2) around the unfloored centres; focal terms summed / G; L1 means over G x 2 of the
        offsets and sizes at the centre cells; kp + 0.1 size + offset.  No GT: 0 (the reference's 0 / 0 is NaN)."""
        (h, w, _), = self.net.levels
        nc = self.row - 4
        gt = torch.as_tensor(gt, device=self.device, dtype=self.dtype)
        cnt = int(torch.argmin(gt[:, 0]).item())
        if cnt == 0:
            return row.sum() * 0.0
        g = gt[:cnt] / torch.tensor([4.0, 4.0, 4.0, 4.0, 1.0], device=self.device, dtype=self.dtype)
        with torch.no_grad():
            gy, gx, gh, gw, cid = g[:, 0], g[:, 1], g[:, 2], g[:, 3], g[:, 4].long()
            cell = (torch.floor(gy).long().clamp(0, h - 1) * w + torch.floor(gx).long().clamp(0, w - 1))
            sigma = torch.stack(centernet_radii(gh, gw)).min()
            yy = torch.arange(h, device=self.device, dtype=self.dtype).view(1, h, 1)
            xx = torch.arange(w, device=self.device, dtype=self.dtype).view(1, 1, w)
            heat = torch.exp(-((gy.view(-1, 1, 1) - yy) ** 2 + (gx.view(-1, 1, 1) - xx) ** 2)
                             / (2.0 * sigma * sigma)).view(cnt, h * w)
            red = torch.zeros((h * w, nc), device=self.device, dtype=self.dtype)
            pos = torch.zeros((h * w, nc), device=self.device, dtype=self.dtype)
            for c in torch.unique(cid).tolist():
                if 0 <= c < nc:
                    red[:, c] = heat[cid == c].max(dim=0).values
                    pos[cell[cid == c], c] = 1.0
            toff = torch.stack([gy - torch.floor(gy), gx - torch.floor(gx)], dim=1)
            tsize = torch.stack([gh, gw], dim=1)
        k = row[:, :nc]
        ls, p = F.logsigmoid(k), torch.sigmoid(k)
        kp = (-(1.0 - p) ** 2 * ls * pos).sum() / cnt \
            + (-(1.0 - red) ** 4 * p ** 2 * (-k + ls) * (1.0 - pos)).sum() / cnt
        at = row[cell]
        return kp + 0.1 * (tsize - at[:, nc + 2:nc + 4]).abs().mean() + (toff - at[:, nc:nc + 2]).abs().mean()

    def image_loss(self, row, gt):
        if self.kind == "ssd":
            return self._ssd.image_loss(row, gt)[0]
        return {"retina": self.retina_image_loss, "fcos": self.fcos_image_loss, "yolo": self.yolo_image_loss,
                "yolo2": self.yolo2_image_loss, "pfpnet": self.pfpnet_image_loss,
                "centernet": self.centernet_image_loss}[self.kind](row, gt)

    def total_loss(self, rows, ground_truth):
        if self._loss_kernels is not None:
            data = self._loss_kernels(rows, ground_truth).sum() / rows.shape[0]
        else:
            per = [self.image_loss(rows[b], ground_truth[b]) for b in range(rows.shape[0])]
            data = torch.stack([torch.as_tensor(p, device=self.device, dtype=self.dtype) for p in per]).sum() \
                / rows.shape[0]
        if self.kind == "yolo":
            data = 0.5 * data                                   # YOLOv3.py:313 (YOLOv2.py:174: no 0.5)
        l2 = sum((p * p).sum() for p in self.params.values()) * 0.5
        return data + self.weight_decay * l2, data

    def classify_loss(self, features, labels):
        """Pretraining mode (RetinaNet.py:123-133): mean-pooled logits, sparse softmax cross-entropy (MEAN over the
        batch) + weight_decay * sum(l2_loss) over the trainable variables -- all of them live in 'feature_extractor'
        here.  labels: int64 tensor [B].  Returns (loss, data term, logits)."""
        data, logits = pooled_xent(features, labels)
        l2 = sum((p * p).sum() for p in self.params.values()) * 0.5
        return data + self.weight_decay * l2, data, logits

    def step(self, images, ground_truth, lr):
        """One `sess.run([train_op, loss])`.  Pretraining mode: `ground_truth` is the label vector [B] and the step
        returns (loss, accuracy of the training-mode logits) like `sess.run([train_op, loss, accuracy])`."""
        stats = []
        accuracy = None
        if self.kind == "classify":
            lab = self.E.check_class_labels(ground_truth, len(images), self.features.C)
            lab = torch.from_numpy(lab).to(self.device)
            loss, _, logits = self.classify_loss(self.forward_features(images, True, stats), lab)
            accuracy = float((torch.argmax(logits, dim=1) == lab).to(torch.float32).mean())
        else:
            rows = self.forward_rows(images, True, stats)
            loss, _ = self.total_loss(rows, ground_truth)
        names = list(self.params)
        grads = torch.autograd.grad(loss, [self.params[k] for k in names], allow_unused=True)
        with torch.no_grad():
            if self.adam:
                self._adam(names, grads, lr)
            for name, gr in zip(names, grads):
                if gr is None or self.adam:
                    continue
                acc = self.slots[name]
                acc.mul_(0.9).add_(gr)
                self.params[name].sub_(acc, alpha=float(lr))
            for scope, mean, var in stats:
                self.buffers[scope + "/moving_mean"].mul_(BN_MOMENTUM).add_(mean, alpha=1 - BN_MOMENTUM)
                self.buffers[scope + "/moving_variance"].mul_(BN_MOMENTUM).add_(var, alpha=1 - BN_MOMENTUM)
        self.global_step += 1
        if accuracy is not None:
            return float(loss.detach()), accuracy
        return float(loss.detach())

    def _adam(self, names, grads, lr):
        """tf.train.AdamOptimizer(lr).minimize: lr_t = lr * sqrt(1 - beta2_power) / (1 - beta1_power); m = b1 m + (1 - b1) g;
        v = b2 v + (1 - b2) g^2; var -= lr_t m / (sqrt(v) + eps); then beta1_power *= b1, beta2_power *= b2."""
        lr_t = float(lr) * (1.0 - self.beta2_power) ** 0.5 / (1.0 - self.beta1_power)
        for name, gr in zip(names, grads):
            if gr is None:
                continue
            m, v = self.slots[name + "/Adam"], self.slots[name + "/Adam_1"]
            m.mul_(ADAM_BETA1).add_(gr, alpha=1.0 - ADAM_BETA1)
            v.mul_(ADAM_BETA2).addcmul_(gr, gr, value=1.0 - ADAM_BETA2)
            self.params[name].sub_(lr_t * m / (v.sqrt() + ADAM_EPS))
        self.beta1_power *= ADAM_BETA1
        self.beta2_power *= ADAM_BETA2

    export = SSDTrainer.export


def centernet_radii(h, w, min_overlap=0.7):
    """CornerNet's three radii as CenterNet.py:254-270 writes them: (b + sqrt(b^2 - 4ac)) / 2 for each quadratic."""
    b1, c1 = h + w, w * h * (1.0 - min_overlap) / (1.0 + min_overlap)
    r1 = (b1 + torch.sqrt(b1 ** 2 - 4.0 * c1)) / 2.0
    b2, c2 = 2.0 * (h + w), (1.0 - min_overlap) * w * h
    r2 = (b2 + torch.sqrt(b2 ** 2 - 16.0 * c2)) / 2.0
    a3, b3, c3 = 4.0 * min_overlap, -2.0 * min_overlap * (h + w), (min_overlap - 1.0) * w * h
    r3 = (b3 + torch.sqrt(b3 ** 2 - 4.0 * a3 * c3)) / 2.0
    return r1, r2, r3


class _RowsLoss(torch.autograd.Function):
    """Per-image losses [B] of the candidate rows [B, N, row] by one odt_<family>_loss_grad launch; the backward
    scales the gradient the same launch wrote by the incoming per-image weights."""

    @staticmethod
    def forward(ctx, rows, kernels, gt):
        loss, grad = kernels.launch(rows, gt)
        ctx.grad = grad         # the trainer's buffer: read by this step's backward, rewritten by the next launch
        return loss.clone()

    @staticmethod
    def backward(ctx, grad_output):
        return ctx.grad * grad_output.view(-1, 1, 1), None, None


class LossKernels:
    """The training step's data term on the GPU: the family's loss and its gradient with respect to the candidate
    rows, from the CUDA kernels (odt_<family>_loss_grad), on the tail parameters the inference engine builds for the
    same network.  Scratch, loss and gradient buffers are allocated once per batch size.  Ground truth goes through
    engine.loss_ground_truth (at most 128 GT rows per image)."""

    def __init__(self, trainer):
        from . import lib as L
        self.E, self.L, self.lib = trainer.E, L, L.load()
        self.kind, self.device, self.row = trainer.kind, trainer.device, trainer.row
        self.p = trainer.net.tail.params(trainer.net.levels)
        self.N = self.p.N
        cfg = trainer.cfg
        self.scalars = [float(cfg.get(k, d)) for k, d in trainer.E.Tail.LOSS_SCALARS[self.kind]]
        self.fn = getattr(self.lib, "odt_%s_loss_grad" % self.kind)
        self._bufs = {}

    def _buffers(self, B):
        if B not in self._bufs:
            import ctypes as C
            nbytes = getattr(self.lib, "odt_%s_loss_scratch_bytes" % self.kind)(C.byref(self.p), B)
            self._bufs[B] = (torch.zeros((nbytes + 7) // 8, dtype=torch.int64, device=self.device),
                             torch.zeros((B,), dtype=torch.float32, device=self.device),
                             torch.empty((B, self.N, self.row), dtype=torch.float32, device=self.device))
        return self._bufs[B]

    def launch(self, rows, gt):
        """rows fp32 [B, N, row] on the device, gt a float32 ndarray from loss_ground_truth -> (loss [B], gradient
        [B, N, row]); both are views of this object's buffers, valid until the next launch with the same B."""
        import ctypes as C
        B = rows.shape[0]
        assert rows.shape[1:] == (self.N, self.row) and rows.dtype == torch.float32
        rows = rows.contiguous()
        scratch, loss, grad = self._buffers(B)
        g = torch.from_numpy(gt).to(self.device)
        args = self.scalars + [scratch.data_ptr(), loss.data_ptr()]
        if self.kind == "ssd":
            args.append(None)
        self.L.check(self.fn(rows.data_ptr(), C.byref(self.p), B, g.data_ptr(), g.shape[1], *args, grad.data_ptr(),
                             torch.cuda.current_stream().cuda_stream), "%s_loss_grad" % self.kind)
        return loss, grad

    def __call__(self, rows, ground_truth):
        """Per-image losses [B] with the kernels' gradient attached to `rows`."""
        gt = self.E.loss_ground_truth(ground_truth)
        if gt.shape[0] != rows.shape[0]:
            raise ValueError("ground truth for %d images, rows for %d" % (gt.shape[0], rows.shape[0]))
        return _RowsLoss.apply(rows, self, gt)


def pooled_xent(features, labels):
    """reduce_mean(features, [H, W]) -> logits [B, C]; tf.losses.sparse_softmax_cross_entropy(labels, logits) with
    Reduction.MEAN (RetinaNet.py:125-126).  features NCHW, labels int64 [B].  Returns (mean loss, logits)."""
    logits = features.mean(dim=(2, 3))
    return F.cross_entropy(logits, labels, reduction="mean"), logits


def _resize_bilinear_legacy(x, oh, ow):
    """tf.image.resize_bilinear, TF1 default (align_corners=False, no half-pixel centres): src = dst * in/out,
    hi = min(lo + 1, in - 1) (RetinaNet.py:309, FCOS.py:372).  NCHW."""
    ih, iw = x.shape[2], x.shape[3]
    sy = torch.arange(oh, device=x.device, dtype=x.dtype) * (ih / oh)
    sx = torch.arange(ow, device=x.device, dtype=x.dtype) * (iw / ow)
    y0, x0 = torch.floor(sy).long(), torch.floor(sx).long()
    y1, x1 = torch.clamp(y0 + 1, max=ih - 1), torch.clamp(x0 + 1, max=iw - 1)
    ly, lx = (sy - y0.to(x.dtype)).view(1, 1, -1, 1), (sx - x0.to(x.dtype)).view(1, 1, 1, -1)
    top = x[:, :, y0][:, :, :, x0] + (x[:, :, y0][:, :, :, x1] - x[:, :, y0][:, :, :, x0]) * lx
    bot = x[:, :, y1][:, :, :, x0] + (x[:, :, y1][:, :, :, x1] - x[:, :, y1][:, :, :, x0]) * lx
    return top + (bot - top) * ly


def _resize_nearest_legacy(x, oh, ow):
    """tf.image.resize_nearest_neighbor, TF1 default: src = floor(dst * in/out) (YOLOv3.py:406)."""
    ih, iw = x.shape[2], x.shape[3]
    yi = torch.clamp(torch.floor(torch.arange(oh, device=x.device, dtype=torch.float32) * (ih / oh)).long(), max=ih - 1)
    xi = torch.clamp(torch.floor(torch.arange(ow, device=x.device, dtype=torch.float32) * (iw / ow)).long(), max=iw - 1)
    return x[:, :, yi][:, :, :, xi]
