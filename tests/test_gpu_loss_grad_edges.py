"""The loss-gradient kernels (csrc/loss.cu, odt_<family>_loss_grad) at their edges, for RetinaNet, SSD, FCOS, YOLOv3
and YOLOv2: the non-smooth points (the FCOS min(d, exp(r)) tie, the smooth-L1 kinks, RetinaNet's clamp of the label
probability at 1e-8), saturated logits and sizes, the focal parameters, every element written, B = 65 and row counts
below one warp block and around the 1024-row grid-stride pass.  The cases and the band rule are built and checked on
the CPU in tests/test_loss_grad_edges.py; the bar is loss_grad_ref.bar.

Every launch here writes its gradient twice, once into a buffer filled with a NaN sentinel and once into a zeroed
one, and the two must be bit-identical: an element the kernel leaves unwritten shows as the sentinel."""
import numpy as np
import pytest
import torch

import loss_grad_ref as LR
import test_gpu_loss as GL
import test_loss_grad_edges as GE
from helpers import YOLO_PRIORS

pytestmark = pytest.mark.gpu
F32 = np.float32
SENTINEL = 0x7FC0DEAD  # a quiet NaN no arithmetic produces
YOLO_SCALES = GE.YOLO_SCALES


def _scalars(kind, cfg):
    from odt_b200.engine import Tail
    return {k: float(cfg[k]) for k, _ in Tail.LOSS_SCALARS[kind]}


def launch(kind, levels, size, cfg, rows, gt):
    """(loss [B], gradient [B,N,row]) of odt_<kind>_loss_grad, the gradient written over the sentinel and over zeros,
    bit-identical; the loss bit-identical to the forward's."""
    from odt_b200.engine import RowsHarness
    h = RowsHarness(LR.tail(kind, size, cfg), levels, rows)
    kw = _scalars(kind, cfg)
    filled = torch.full(rows.shape, SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    loss, grad = h.loss_grad(kind, gt, grad_out=filled, **kw)
    loss0, grad0 = h.loss_grad(kind, gt, grad_out=torch.zeros(rows.shape, device="cuda"), **kw)
    assert np.array_equal(grad.view(np.uint32), grad0.view(np.uint32)), "an element left unwritten"
    fwd = h.loss(kind, gt, **kw)
    assert np.array_equal(loss.view(np.uint32), fwd.view(np.uint32)) and np.array_equal(loss0.view(np.uint32),
                                                                                        fwd.view(np.uint32))
    return loss, grad


def check(c, got, resolve=None, tag=""):
    """One image against the restatement (loss_grad_ref.reference), non-finite elements against the float32
    restatement's; `resolve` puts rows whose decision float rounding may flip on the side the kernel took."""
    _, ref, dt, g32 = LR.reference(c["kind"], c["levels"], c["cfg"], c["size"], c["nc"], c["rows"], c["gt"])
    band = None
    if resolve is not None:
        ref, band = resolve(c, got, ref)
    ok, err, scale = LR.bar(got, ref, g32)
    bad = ~np.isfinite(g32)
    print("%s %s: %s reference, max|err| %.3g = %.3g of max|ref| %.3g; %d non-finite elements (%d NaN)%s"
          % (c["kind"], tag, dt, err, err / scale if scale else 0.0, scale, int(bad.sum()), int(np.isnan(g32).sum()),
             "" if band is None else "; clamp band %d ulps: %s" % (GE.CLAMP_BAND_ULPS, band)))
    assert ok
    return ref


def run(c, **kw):
    loss, grad = launch(c["kind"], c["levels"], c["size"], c["cfg"], c["rows"][None], c["gt"][None])
    return check(c, grad[0], **kw), grad[0]


# --------------------------------------------------------------------------------------------------- kinks --
@pytest.mark.parametrize("kind", ["retina", "ssd"])
def test_smooth_l1_kinks(built, kind):
    """Target exactly 0, deltas 0, +-1, +-1 +- 1 ulp: d = 0 gives exactly 0, |d| >= 1 gives exactly +-1 / #pos (TF's
    where(|d| < 1, ...) takes the linear branch at |d| = 1), 1 - 1 ulp gives (1 - 1 ulp) / #pos."""
    c = GE._kink(kind)
    _, g = run(c, tag="smooth-L1 kinks")
    n1, n2 = c["picks"]
    one = g[n1, 22]
    assert one > 0 and g[n1, 21] == 0 and g[n1, 23] == -one and g[n1, 24] == one
    assert g[n2, 24] == 0 and g[n2, 23] == -one and g[n2, 21] == -g[n2, 22] and 0 < one - g[n2, 21] <= one * 2 ** -23


def test_fcos_tie(built):
    """d = exp(r) = 1: the prediction gets no intersection gradient (TF's Minimum), only the union's."""
    c = GE._fcos_tie()
    ref, g = run(c, tag="min(d, exp(r)) ties")
    for n, col in c["ties"]:
        assert abs(g[n, col] - ref[n, col]) <= LR.BAR * np.abs(ref).max(), (n, col)


@pytest.mark.parametrize("gamma", [2.0, 0.0, 0.5])
def test_retina_clamp_band_and_q_one(built, gamma):
    """Straddle rows at 1e-8 (1 + k 2^-23): outside the band the reference's side, inside either side with the
    reference of that side.  Rows whose label probability rounds to 1: gamma 2 and 0 finite (the gamma == 0 branch),
    gamma 0.5 NaN on the 21 logits exactly where the float32 restatement has it (0 * inf in d (1 - q)^gamma)."""
    c = GE._retina_clamp()
    c["cfg"] = dict(c["cfg"], gamma=gamma)
    _, g = run(c, resolve=GE.resolve_clamp, tag="clamp, gamma %g" % gamma)
    ones = np.array(c["ones"])
    if gamma == 0.5:
        assert np.isnan(g[ones, :21]).all() and np.isfinite(g[ones, 21:]).all()
        assert np.isfinite(np.delete(g, ones, axis=0)).all()
    else:
        assert np.isfinite(g).all()


# ---------------------------------------------------------------------------------------------- saturation --
def _saturated(kind, L, seed):
    """Random rows with every logit at +-L; FCOS every fourth location's first distance logit at 100 (exp overflows);
    YOLO sizes of every seventh row at 1e20."""
    rng = np.random.default_rng(seed)
    if kind in ("retina", "ssd"):
        geo = GL.RET_SMALL if kind == "retina" else GL.SSD_FINE
        c = dict(kind=kind, levels=geo.levels, size=geo.size, cfg=LR.config(kind, geo.size), nc=20,
                 rows=LR.rows(kind, geo.N, seed=seed)[0], gt=LR.gt(rng, 4, geo.size, 6, lo=0.2, hi=0.6))
        c["rows"][:, :21] = rng.choice([-L, L], (geo.N, 21))
        return c
    if kind == "fcos":
        geo = GL.FCOS_SMALL
        gt = np.full((6, 5), -1.0, F32)
        gt[:4] = [[40, 50, 30, 40, 0], [60, 60, 64, 64, 19], [64, 64, 128, 128, 10], [50, 70, 90, 70, 3]]
        c = dict(kind=kind, levels=geo.levels, size=geo.size, cfg=LR.config(kind, geo.size), nc=20,
                 rows=LR.rows(kind, geo.N, seed=seed)[0], gt=gt)
        c["rows"][:, :21] = rng.choice([-L, L], (geo.N, 21))
        c["rows"][::4, 21] = 100.0
        return c
    if kind == "yolo":
        geo = GL.YOLO_SMALL
        c = dict(kind=kind, levels=geo.levels, size=geo.size, nc=20,
                 cfg=LR.config(kind, geo.size, priors=YOLO_PRIORS, **YOLO_SCALES),
                 rows=LR.rows(kind, geo.N, seed=seed)[0], gt=LR.gt(rng, 5, geo.size, 6))
    else:
        levels = [(13, 13, 5)]
        c = dict(kind=kind, levels=levels, size=416, nc=20, cfg=LR.config(kind, 416, A=5, **YOLO_SCALES),
                 rows=LR.rows(kind, 13 * 13 * 5, seed=seed)[0], gt=LR.gt(rng, 5, 416, 6))
    c["rows"][:, :20] = rng.choice([-L, L], (len(c["rows"]), 20))
    c["rows"][:, 24] = rng.choice([-L, L], len(c["rows"]))
    c["rows"][::7, 22:24] = 1e20
    return c


@pytest.mark.parametrize("L", [60.0, 100.0])
@pytest.mark.parametrize("kind", ["retina", "ssd", "fcos", "yolo", "yolo2"])
def test_saturation(built, kind, L):
    c = _saturated(kind, L, seed=int(L) + len(kind))
    _, g = run(c, tag="logits +-%g" % L)
    if kind != "fcos":
        assert np.isfinite(g).all()


# ------------------------------------------------------------------------------------------ focal parameters --
@pytest.mark.parametrize("alpha", [0.25, 0.75, 1.0])
@pytest.mark.parametrize("gamma", [0.0, 0.5, 1.0, 2.0, 3.5])
def test_focal_parameters(built, gamma, alpha):
    """The loss forward against oracle/loss.py and the gradient against the restatement at the config's alpha and
    gamma."""
    c = GE._retina_random()
    c["cfg"] = dict(c["cfg"], alpha=alpha, gamma=gamma)
    loss, grad = launch("retina", c["levels"], c["size"], c["cfg"], c["rows"][None], c["gt"][None])
    from oracle import loss as OL
    a = GL.RET_SMALL.anchors()
    r = c["rows"]
    want = OL.retina_image_loss(r[:, :21], r[:, 21:23], r[:, 23:], *a, c["gt"], alpha=alpha, gamma=gamma)[0]
    print("alpha %g gamma %g: loss %.7g oracle %.7g" % (alpha, gamma, loss[0], want))
    assert abs(loss[0] - want) <= 2e-5 * max(abs(want), 1.0)
    check(c, grad[0], tag="alpha %g gamma %g" % (alpha, gamma))


@pytest.mark.parametrize("kind", ["yolo", "yolo2"])
@pytest.mark.parametrize("zero", ["coord_class", "obj_noobj"])
def test_yolo_zero_scales(built, kind, zero):
    """A zero scale zeroes its columns exactly: coord and class, or objectness (obj and no-object)."""
    scales = dict(YOLO_SCALES, **({"coord_scale": 0.0, "class_scale": 0.0} if zero == "coord_class" else
                                  {"obj_scale": 0.0, "noobj_scale": 0.0}))
    c = _saturated(kind, 3.0, seed=80)
    c["rows"][:, 22:24] = np.random.default_rng(81).standard_normal((len(c["rows"]), 2)) * 0.5
    c["cfg"] = dict(c["cfg"], **scales)
    _, g = run(c, tag="scales %s" % zero)
    cols = np.r_[0:24] if zero == "coord_class" else np.r_[24:25]
    assert np.all(g[:, cols] == 0) and np.any(g != 0)


# ------------------------------------------------------------------------------------------ batch, geometry --
@pytest.mark.parametrize("kind", ["retina", "ssd", "fcos", "yolo", "yolo2"])
def test_batch_65(built, kind):
    """B = 65 (tests/test_gpu_loss.batch65_gt; YOLOv2 on YOLOv3's boxes, 13 x 13 x 5): each image bit-identical to
    the same image alone, the GT-free image 5 among them; images 0, 3, 4 and 64 against the restatement."""
    if kind == "yolo2":
        levels, size, cfg = [(13, 13, 5)], 416, LR.config("yolo2", 416, A=5, **YOLO_SCALES)
        gt = GL.batch65_gt("yolo", seed=52)
    else:
        geo = GL.TAIL_GEOS[kind]
        levels, size = geo.levels, geo.size
        cfg = LR.config(kind, size, priors=YOLO_PRIORS, **YOLO_SCALES) if kind == "yolo" else LR.config(kind, size)
        gt = GL.batch65_gt(kind, seed=52)
    N = sum(h * w * a for h, w, a in levels)
    rows = LR.rows(kind, N, B=65, seed=53)
    loss, grad = launch(kind, levels, size, cfg, rows, gt)
    for b in range(65):
        lb, gb = launch(kind, levels, size, cfg, rows[b:b + 1], gt[b:b + 1])
        assert lb[0].tobytes() == loss[b].tobytes() and np.array_equal(gb[0].view(np.uint32), grad[b].view(np.uint32)), b
    for b in (0, 3, 4, 64):
        check(dict(kind=kind, levels=levels, size=size, cfg=cfg, nc=20, rows=rows[b], gt=gt[b]), grad[b],
              tag="B = 65, image %d" % b)


GEOMETRIES = {  # (kind, level table, image size); N in the comment
    "ssd_1x1x4": ("ssd", [(1, 1, 4)], 300),                             # 4
    "fcos_5x1x1": ("fcos", [(1, 1, 1)] * 5, 128),                       # 5
    "yolo_3x1x1x2": ("yolo", [(1, 1, 2)] * 3, 32),                      # 6
    "yolo2_1x1x1": ("yolo2", [(1, 1, 1)], 32),                          # 1
    "yolo2_1x1x7": ("yolo2", [(1, 1, 7)], 32),                          # 7
    "yolo2_16x16x4": ("yolo2", [(16, 16, 4)], 512),                     # 1024: one full grid-stride pass
    "yolo2_5x41x5": ("yolo2", [(5, 41, 5)], 1312),                      # 1025: one row in the second pass
    "yolo2_1x683x3": ("yolo2", [(1, 683, 3)], 21856),                   # 2049: one row in the third pass
    "ssd_16x16x4": ("ssd", [(16, 16, 4)], 300),                         # 1024
    "ssd_1x257x4": ("ssd", [(1, 257, 4)], 300),                         # 1028
}


def _geometry_gt(kind, size):
    g = np.full((4, 5), -1.0, F32)
    if kind == "fcos":  # one box on P3 and one on P6, both around the single cell centre (0, 0)
        g[:2] = [[8, 8, 40, 40, 3], [100, 100, 300, 300, 11]]
    elif kind in ("yolo", "yolo2") and size == 32:
        g[:2] = [[4, 5, 10, 12, 2], [6, 3, 40, 30, 17]]
    else:
        g[:3] = LR.gt(np.random.default_rng(size), 3, size, 3, lo=0.1, hi=0.5)
    return g


@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_geometry(built, name):
    kind, levels, size = GEOMETRIES[name]
    A = levels[0][2]
    if kind == "yolo":
        cfg = LR.config(kind, size, A=A, **YOLO_SCALES)
    elif kind == "yolo2":
        cfg = LR.config(kind, size, A=A, **YOLO_SCALES)
    else:
        cfg = LR.config(kind, size)
    N = sum(h * w * a for h, w, a in levels)
    c = dict(kind=kind, levels=levels, size=size, cfg=cfg, nc=20, rows=LR.rows(kind, N, seed=N)[0],
             gt=_geometry_gt(kind, size))
    _, g = run(c, tag="%s N = %d" % (name, N))
    if N > 1024:
        assert kind == "ssd" or np.any(g[-1] != 0), "the last grid-stride pass carries a gradient"
