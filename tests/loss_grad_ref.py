"""The training step's loss restatement (odt_b200/train.py, GraphTrainer.image_loss) on any level table, class count
and prior count, without a network: the reference the loss-gradient kernels are tested against.  `grad` runs it in
float64 with autograd on the rows of one image, `reference` chooses between the float64 and the float32 restatement,
and `bar` is the one comparison every gradient test applies."""
import types

import numpy as np
import torch

from helpers import BASE_CFG, model_cfg

F32 = np.float32
KIND_CFG = {"ssd": "ssd", "retina": "retinanet", "yolo": "yolov3", "fcos": "fcos"}
# YOLOv2's five VOC priors in grid cells (testYOLOv2.py:44), then four more for A up to 9
YOLO2_PRIORS = [[1.08, 1.19], [3.42, 4.41], [6.63, 11.38], [9.42, 5.11], [16.62, 10.52], [2.0, 2.5], [5.0, 3.0],
                [12.0, 14.0], [0.6, 0.7]]
BAR = 1e-5  # of the image's max |gradient|


def config(kind, size, nc=20, A=3, **over):
    """The family's config at image size `size` (SSD: 300 or 512), nc classes and A priors (YOLOv3, YOLOv2)."""
    if kind == "yolo2":
        c = dict(BASE_CFG)
        c.update(data_shape=[size, size, 3], coord_scale=1, noobj_scale=1, obj_scale=5., class_scale=1.,
                 rescore_confidence=False, priors=YOLO2_PRIORS[:A], num_classes=nc)
        c.update(over)
        return c
    if kind == "yolo":
        import prior_count_ref as PR
        over.setdefault("priors", PR.priors_for(A))
        over.setdefault("num_priors", A)
    if kind in ("yolo", "fcos"):
        over.setdefault("num_classes", nc)
    return model_cfg(KIND_CFG[kind], data_shape=[size, size, 3], **over)


def tail(kind, size, cfg):
    from odt_b200 import nets
    if kind == "ssd":
        return nets.ssd_tail(size, cfg)
    return {"retina": nets.retina_tail, "yolo": nets.yolo_tail, "yolo2": nets.yolo2_tail, "fcos": nets.fcos_tail}[kind](cfg)


def restatement(kind, levels, cfg, size, nc=20, dtype=torch.float64):
    """A GraphTrainer holding only what image_loss reads: kind, config, level table, row width, device, dtype."""
    from odt_b200.train import GraphTrainer, SSDTrainer
    tr = GraphTrainer.__new__(GraphTrainer)
    tr.kind, tr.cfg, tr.device, tr.dtype = kind, cfg, torch.device("cpu"), dtype
    tr.net = types.SimpleNamespace(levels=[tuple(lv) for lv in levels])
    tr.row = nc + 5
    tr._anchor_cache = None
    if kind == "ssd":
        tr._ssd = SSDTrainer.__new__(SSDTrainer)
        tr._ssd.device, tr._ssd.dtype, tr._ssd.size, tr._ssd._anchors = tr.device, dtype, size, None
        tr._ssd._shapes = [(h, w) for h, w, _ in levels]
    return tr


def grad(tr, row, gt):
    """(loss, d loss / d row) of one image in the restatement's dtype; a family whose loss does not depend on the
    rows (FCOS without GT on any level) gives a zero gradient."""
    r = torch.tensor(np.asarray(row), dtype=tr.dtype, requires_grad=True)
    loss = tr.image_loss(r, gt)
    if not torch.is_tensor(loss) or not loss.requires_grad:
        return float(loss), np.zeros(r.shape)
    return float(loss.detach()), torch.autograd.grad(loss, r)[0].numpy()


def reference(kind, levels, cfg, size, nc, row, gt):
    """(loss, gradient, dtype, float32 gradient) of the restatement.  The reference is the float64 restatement wherever
    float64 makes the matching decisions the float32 kernels make, i.e. where its loss equals the float32
    restatement's to 1e-6; elsewhere (a best IoU within float32 rounding of a threshold, float32 ties, SSD's mining
    order) it is the float32 restatement, whose decisions are the kernels'.  The float32 gradient also says where a
    float32 computation is not finite."""
    with np.errstate(all="ignore"):
        l32, g32 = grad(restatement(kind, levels, cfg, size, nc, dtype=torch.float32), row, gt)
        l64, g64 = grad(restatement(kind, levels, cfg, size, nc), row, gt)
    if abs(l64 - l32) <= 1e-6 * max(abs(l32), 1.0):
        return l64, g64, "float64", g32
    return l32, g32, "float32", g32


def bar(got, ref, ref32=None):
    """The gradient bar on one image: (ok, max |error|, max |reference|).  Every element within BAR of the image's max
    |reference|, and exact zeros where the reference is exactly zero.  With ref32 (the float32 restatement), elements
    it does not give finite must be the same non-finite value in `got` (NaN, +inf or -inf), and only the others are
    held to the bar."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    fin = np.ones(ref.shape, bool) if ref32 is None else np.isfinite(ref32)
    if ref32 is not None and not np.array_equal(got[~fin], np.asarray(ref32, np.float64)[~fin], equal_nan=True):
        return False, float("inf"), 0.0
    g, r = got[fin], ref[fin]
    if not (np.isfinite(g).all() and np.isfinite(r).all()):
        return False, float("inf"), 0.0
    scale = float(np.abs(r).max()) if r.size else 0.0
    err = float(np.abs(g - r).max()) if r.size else 0.0
    return bool(err <= BAR * scale and np.all(g[r == 0] == 0)), err, scale


def rows(kind, N, nc=20, B=1, seed=0):
    """Seeded rows [B, N, nc + 5] with the statistics of tests/test_gpu_loss.make_rows at any class count."""
    rng = np.random.default_rng(seed)
    r = np.empty((B, N, nc + 5), F32)
    if kind in ("ssd", "retina"):
        r[..., :21] = rng.standard_normal((B, N, 21)) * 2.0
        r[..., 21:] = rng.standard_normal((B, N, 4)) * 0.5
    elif kind in ("yolo", "yolo2"):
        r[..., :nc] = rng.standard_normal((B, N, nc)) * 2.0
        r[..., nc:nc + 4] = rng.standard_normal((B, N, 4)) * 0.5
        r[..., nc + 4] = rng.standard_normal((B, N)) * 2.0 + 1.0
    else:
        r[..., :nc] = rng.standard_normal((B, N, nc)) * 2.0
        r[..., nc] = rng.standard_normal((B, N)) * 2.0 + 1.0
        r[..., nc + 1:] = rng.standard_normal((B, N, 4)) * 0.5 + 1.0
    return r


def gt(rng, n, size, G, nc=20, lo=0.08, hi=0.6):
    """n boxes (y, x, h, w, class) inside a size x size image, padded with -1 to G rows."""
    g = np.full((G, 5), -1.0, F32)
    g[:n, 0:2] = rng.uniform(0.1 * size, 0.9 * size, (n, 2))
    g[:n, 2:4] = rng.uniform(lo * size, hi * size, (n, 2))
    g[:n, 4] = rng.integers(0, nc, n)
    return g
