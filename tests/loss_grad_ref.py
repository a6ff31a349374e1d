"""The training step's loss restatement (odt_b200/train.py, GraphTrainer.image_loss) on any level table, class count
and prior count, without a network: the reference the loss-gradient kernels are tested against.  `grad` runs it in
float64 with autograd on the rows of one image."""
import types

import numpy as np
import torch

from helpers import model_cfg

F32 = np.float32
KIND_CFG = {"ssd": "ssd", "retina": "retinanet", "yolo": "yolov3", "fcos": "fcos"}


def config(kind, size, nc=20, A=3, **over):
    """The family's config at image size `size` (SSD: 300 or 512), nc classes and A priors (YOLOv3)."""
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
    return {"retina": nets.retina_tail, "yolo": nets.yolo_tail, "fcos": nets.fcos_tail}[kind](cfg)


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


def rows(kind, N, nc=20, B=1, seed=0):
    """Seeded rows [B, N, nc + 5] with the statistics of tests/test_gpu_loss.make_rows at any class count."""
    rng = np.random.default_rng(seed)
    r = np.empty((B, N, nc + 5), F32)
    if kind in ("ssd", "retina"):
        r[..., :21] = rng.standard_normal((B, N, 21)) * 2.0
        r[..., 21:] = rng.standard_normal((B, N, 4)) * 0.5
    elif kind == "yolo":
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
