"""The four training-loss forward kernels (csrc/loss.cu) at their decision edges, at full GT capacity,
across the 64-image block of the final kernels and on full-size geometries, against the live CPU oracle
(oracle/loss.py).  Bar: |gpu - oracle| <= 2e-5 * max(|oracle|, 1) (float summation order); the SSD
(#pos, #neg, #mined) triple exact.

Each edge case is built so that the oracle sees the edge exactly (an IoU equal to a threshold in fp32,
a tie, a box edge on a grid line); CPU guards check that it does, and that moving the input the fewest
ulps across the edge (or, for a tie no input step can break, taking the other side of it) moves the
oracle loss by at least 100x the GPU tolerance, so a kernel that decides the other way cannot pass."""
import ctypes

import numpy as np
import pytest

from helpers import YOLO_PRIORS, model_cfg

F32 = np.float32
TOL = 2e-5


# ------------------------------------------------------------------ geometry --
class Geo:
    """kind, image size (SSD size / RetinaNet input width / unused) and the (H, W, A) level table."""

    def __init__(self, kind, size, levels):
        self.kind, self.size, self.levels = kind, size, [tuple(lv) for lv in levels]
        self.N = sum(h * w * a for h, w, a in self.levels)

    def index(self, level, y, x, a=0):
        off = sum(h * w * aa for h, w, aa in self.levels[:level])
        h, w, A = self.levels[level]
        return off + (y * w + x) * A + a

    def anchors(self):
        from oracle import tails as OT
        shapes = [(h, w) for h, w, _ in self.levels]
        if self.kind == "ssd":
            return OT.ssd_anchors(self.size, shapes)
        return OT.retina_anchors([self.size, self.size, 3], shapes)

    def tail(self):
        from odt_b200 import nets
        if self.kind == "ssd":
            return nets.ssd_tail(self.size, model_cfg("ssd"))
        if self.kind == "retina":
            return nets.retina_tail(model_cfg("retinanet", data_shape=[self.size, self.size, 3]))
        if self.kind == "yolo":
            return nets.yolo_tail(model_cfg("yolov3"))
        return nets.fcos_tail(model_cfg("fcos"))


RET_SMALL = Geo("retina", 64, [(8, 8, 9)])
SSD_TINY = Geo("ssd", 300, [(3, 3, 4)])          # N = 36 < 64 anchors: most anchor blocks are empty
SSD_FINE = Geo("ssd", 300, [(38, 38, 4)])        # adjacent anchors overlap with IoU 0.77 > 0.7
FCOS_SMALL = Geo("fcos", 128, [(16, 16, 1), (8, 8, 1), (4, 4, 1), (2, 2, 1), (1, 1, 1)])
YOLO_SMALL = Geo("yolo", 160, [(5, 5, 3), (10, 10, 3), (20, 20, 3)])
TAIL_GEOS = {  # the tail fixtures' tables (tests/golden/make_golden.py); N % 64 != 0 for all but FCOS
    "ssd": Geo("ssd", 300, [(38, 38, 4), (19, 19, 6), (10, 10, 6), (5, 5, 6), (5, 5, 4), (3, 3, 4)]),
    "retina": Geo("retina", 128, [(16, 16, 9), (8, 8, 9), (4, 4, 9), (2, 2, 9), (1, 1, 9)]),
    "yolo": YOLO_SMALL,
    "fcos": Geo("fcos", 256, [(32, 32, 1), (16, 16, 1), (8, 8, 1), (4, 4, 1), (2, 2, 1)]),
}
IMG = {"ssd": 300, "retina": 128, "yolo": 160, "fcos": 256}  # image size that places random GT boxes


def make_rows(kind, n, batch=1, seed=2):
    """Seeded head rows [B,N,25] with the statistics of tests/golden/make_golden.make_rows."""
    rng = np.random.default_rng(seed)
    rows = np.empty((batch, n, 25), F32)
    if kind in ("ssd", "retina"):
        rows[..., :21] = rng.standard_normal((batch, n, 21)) * 2.0
        rows[..., 21:] = rng.standard_normal((batch, n, 4)) * 0.5
    elif kind == "yolo":
        rows[..., :20] = rng.standard_normal((batch, n, 20)) * 2.0
        rows[..., 20:24] = rng.standard_normal((batch, n, 4)) * 0.5
        rows[..., 24] = rng.standard_normal((batch, n)) * 2.0 + 1.0
    else:
        rows[..., :20] = rng.standard_normal((batch, n, 20)) * 2.0
        rows[..., 20] = rng.standard_normal((batch, n)) * 2.0 + 1.0
        rows[..., 21:] = rng.standard_normal((batch, n, 4)) * 0.5 + 1.0
    return rows


def random_gt(rng, n, size, G, lo=0.08, hi=0.6):
    """n boxes (y, x, h, w, class) inside a size x size image, padded with -1 to G rows."""
    gt = np.full((G, 5), -1.0, F32)
    gt[:n, 0:2] = rng.uniform(0.1 * size, 0.9 * size, (n, 2))
    gt[:n, 2:4] = rng.uniform(lo * size, hi * size, (n, 2))
    gt[:n, 4] = rng.integers(0, 20, n)
    return gt


# -------------------------------------------------------------------- oracle --
def oracle(geo, rows, gt, **kw):
    """Oracle loss of one image: rows [N,25], gt [G,5] -> (loss, (#pos, #neg, #mined) for SSD else None)."""
    from oracle import loss as OL
    rows = np.asarray(rows, F32)
    gt = np.asarray(gt, F32)
    if geo.kind in ("ssd", "retina"):
        args = (rows[:, :21], rows[:, 21:23], rows[:, 23:], *geo.anchors(), gt)
        if geo.kind == "retina":
            return OL.retina_image_loss(*args)[0], None
        loss, info = OL.ssd_image_loss(*args)
        return loss, (info["num_pos"], info["num_neg"], info["selected"])
    off, lv = 0, []
    for h, w, a in geo.levels:
        blk = rows[None, off:off + h * w * a]
        if geo.kind == "yolo":
            lv.append(blk.reshape(1, h, w, a * 25))
        else:
            q = blk.reshape(1, h, w, 25)
            lv.append((q[..., :20], q[..., 20:21], q[..., 21:25]))
        off += h * w * a
    if geo.kind == "yolo":
        priors = kw.pop("priors", YOLO_PRIORS)
        with np.errstate(over="ignore"):
            return OL.yolo_image_loss(lv, priors, gt, **kw), None
    with np.errstate(divide="ignore", invalid="ignore"):
        return OL.fcos_image_loss(lv, gt), None


def match_iou(geo, gt):
    """IoU[G, N] of the valid GT rows with the anchors, in the oracle's operation order."""
    a1, a2, _, ahw = geo.anchors()
    g = np.asarray(gt, F32)
    g = g[:int(np.argmin(g, axis=0)[0])] if (g[:, 0] == -1).any() else g
    gyx, ghw = g[:, 0:2], g[:, 2:4]
    g1 = (gyx - ghw / F32(2.0)).astype(F32)
    g2 = (gyx + ghw / F32(2.0)).astype(F32)
    inter = np.prod(np.maximum(np.minimum(a2[None], g2[:, None]) - np.maximum(a1[None], g1[:, None]), F32(0)),
                    axis=-1).astype(F32)
    aarea = np.prod(ahw, axis=-1).astype(F32)[None]
    garea = np.prod(ghw, axis=-1).astype(F32)[:, None]
    return (inter / (aarea + garea - inter)).astype(F32)


def step_until(v, toward, pred, max_ulps=8):
    """The fp32 value a few ulps from v toward `toward` where pred first holds: the smallest input step
    that crosses an edge once the oracle's own roundings are applied."""
    v = F32(v)
    for _ in range(max_ulps):
        v = np.nextafter(v, F32(toward))
        if pred(v):
            return v
    raise AssertionError("no crossing within %d ulps" % max_ulps)


def bg_xent(row):
    """SSD background cross-entropy of one row, as oracle.loss.ssd_image_loss computes it."""
    z = (row[:21] - row[:21].max()).astype(F32)
    return F32(np.log(np.exp(z).astype(F32).sum(dtype=F32)) - z[20])


def close(got, ref):
    if np.isinf(ref):
        return got == ref
    return abs(float(got) - ref) <= TOL * max(abs(ref), 1.0)


# ---------------------------------------------------------------- edge cases --
# Each builder returns dict(geo, rows [N,25], gt [G,5], nudged=(rows, gt)); it asserts that the oracle sees
# the edge.  "nudged" is the same input moved by the smallest step that crosses the edge.
def _retina_pos_edge():
    """Retina positive rule bv > 0.5: a 32x32 anchor centred in a 64x32 GT has IoU exactly 0.5 (ignored)."""
    geo = RET_SMALL
    n = geo.index(0, 3, 4, 0)
    gt = np.array([[28, 36, 64, 32, 5], [-1] * 5], F32)
    iou = match_iou(geo, gt)
    assert iou[0, n] == F32(0.5) and iou[0].max() > F32(0.5), "anchor %d must sit on the 0.5 edge" % n
    gt2 = gt.copy()

    def crossed(h):
        gt2[0, 2] = h
        return match_iou(geo, gt2)[0, n] > F32(0.5)
    gt2[0, 2] = step_until(64, 0, crossed)
    rows = make_rows("retina", geo.N, seed=21)[0]
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))


def _retina_neg_edge():
    """Retina negative rule bv < 0.4: the anchor in an 80x32 GT has IoU exactly 0.4 (ignored, not negative).
    Its background logit is pushed down so that counting it as a negative costs a large focal term."""
    geo = RET_SMALL
    n = geo.index(0, 3, 4, 0)
    gt = np.array([[28, 36, 80, 32, 5], [-1] * 5], F32)
    iou = match_iou(geo, gt)
    assert iou[0, n] == F32(0.4) and np.argmax(iou[0]) != n
    gt2 = gt.copy()
    gt2[0, 2] = np.nextafter(F32(80), F32(1e9))
    assert match_iou(geo, gt2)[0, n] < F32(0.4)
    rows = make_rows("retina", geo.N, seed=22)[0]
    rows[n, 20] = -40.0
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))


def _retina_best_tie():
    """Best anchor per GT: a GT midway between two equal anchors (handled by different threads); the first
    maximum is the positive, the other is a negative.  Their box deltas differ so the choice shows."""
    geo = RET_SMALL
    gt = np.array([[28, 40, 8, 38, 5], [-1] * 5], F32)
    iou = match_iou(geo, gt)[0]
    ties = np.flatnonzero(iou == iou.max())
    assert len(ties) == 2 and ties[0] % 256 != ties[1] % 256 and iou.max() < F32(0.4), ties
    gt2 = gt.copy()
    gt2[0, 1] = np.nextafter(F32(40), F32(1e9))
    assert np.argmax(match_iou(geo, gt2)[0]) == ties[1]
    rows = make_rows("retina", geo.N, seed=23)[0]
    rows[ties[0], 21:25] = 0.0
    rows[ties[1], 21:25] = 4.0
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))


def _ssd_pos_edge():
    """SSD positive rule bv > 0.5 (no ignore band) on the 36-anchor geometry: IoU exactly 0.5 is negative."""
    geo = SSD_TINY
    n = geo.index(0, 1, 1, 0)
    gt = np.array([[150, 150, 120, 60, 3], [-1] * 5], F32)
    iou = match_iou(geo, gt)
    assert iou[0, n] == F32(0.5) and iou[0].max() > F32(0.5)
    gt2 = gt.copy()

    def crossed(h):
        gt2[0, 2] = h
        return match_iou(geo, gt2)[0, n] > F32(0.5)
    gt2[0, 2] = step_until(120, 0, crossed)
    rows = make_rows("ssd", geo.N, seed=24)[0]
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))


def _ssd_mining_tie():
    """Hard-negative mining with equal background losses: anchors P < Q (adjacent, IoU 0.77 > 0.7) tie for the
    top loss.  Taking P first suppresses Q and S (left of P) and keeps R (right of Q); taking Q first keeps
    S instead.  R and S have different losses, so the lower-index-first order shows in the mean."""
    geo = SSD_FINE
    S, P, Q, R = (geo.index(0, 20, x, 0) for x in (9, 10, 11, 12))
    rows = make_rows("ssd", geo.N, seed=25)[0]
    rows[P, 20] = -60.0
    rows[Q] = rows[P]
    rows[R], rows[S] = rows[P], rows[P]
    rows[R, 20], rows[S, 20] = -50.0, -30.0
    a = geo.anchors()[2:]
    gt = np.array([[a[0][geo.index(0, 3, 3)][0], a[0][geo.index(0, 3, 3)][1], 60, 60, 4], [-1] * 5], F32)
    assert bg_xent(rows[P]) == bg_xent(rows[Q])
    rows2 = rows.copy()
    while bg_xent(rows2[Q]) <= bg_xent(rows2[P]):  # a few ulps until Q's loss is strictly the larger
        rows2[Q, 20] = np.nextafter(rows2[Q, 20], F32(-1e9))
    assert rows2[Q, 20] >= np.float32(-60.0) - 8 * np.spacing(F32(60.0))
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows2, gt))


def _ssd_mining_dry():
    """Mining that runs dry: 20 GTs make #neg <= 3 #pos, the negatives suppress each other, so fewer than
    `chosen` are selected and the mean divides by the number selected."""
    geo = SSD_FINE
    rng = np.random.default_rng(5)
    gt = np.full((21, 5), -1.0, F32)
    gt[:20, :2] = rng.uniform(20, 280, (20, 2))
    gt[:20, 2:4] = 60
    gt[:20, 4] = rng.integers(0, 20, 20)
    rows = make_rows("ssd", geo.N, seed=26)[0]
    return dict(geo=geo, rows=rows, gt=gt, nudged=None)


def _fcos_grid_edge():
    """FCOS strict inside test: the GT's top and left edges lie on grid lines of P3 (l = t = 0 is outside)."""
    geo = FCOS_SMALL
    gt = np.array([[36, 36, 24, 24, 6], [-1] * 5], F32)
    y1 = F32(F32(36) / F32(8)) - F32(F32(24) / F32(8)) / F32(2)
    assert y1 == F32(3.0)
    gt2 = gt.copy()
    gt2[0, 0:2] = np.nextafter(F32(36), F32(0))   # the edges move just above the grid lines
    rows = make_rows("fcos", geo.N, seed=27)[0]
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))


def _fcos_level_bound(s):
    """FCOS level bounds are inclusive and overlap: sqrt(h*w) == s belongs to two levels."""
    def build():
        geo = FCOS_SMALL
        gt = np.array([[60, 60, s, s, 9], [-1] * 5], F32)
        assert np.sqrt(F32(s) * F32(s)).astype(F32) == F32(s)
        gt2 = gt.copy()
        gt2[0, 2:4] = np.nextafter(F32(s), F32(0))
        assert np.sqrt((gt2[0, 2] * gt2[0, 3]).astype(F32)).astype(F32) < F32(s)
        rows = make_rows("fcos", geo.N, seed=28 + s)[0]
        return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))
    return build


def _fcos_equal_area():
    """FCOS minimal-area target with ties: two 48x48 GTs (different classes) offset by one P3 cell; in the
    4x4 cells inside both the areas are equal and the target is the element-wise max of l, r, t, b."""
    geo = FCOS_SMALL
    gt = np.array([[64, 64, 48, 48, 3], [72, 72, 48, 48, 7], [-1] * 5], F32)
    gt2 = gt.copy()
    x2 = lambda w: F32(F32(72) / F32(8)) + F32(F32(w) / F32(8)) / F32(2)  # right edge in P3 cells
    gt2[1, 3] = step_until(48, 0, lambda w: x2(w) != x2(48))
    rows = make_rows("fcos", geo.N, seed=29)[0]
    for y in range(7, 11):      # the tied cells: a large centre-ness logit makes their target count
        for x in range(7, 11):
            rows[geo.index(0, y, x), 20] = 20.0
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))


def _yolo_noobj_quirk_box(geo, level, y, x, a):
    """The reference's no-object box of one (cell, prior): (yx - hw/2, yx + hw/2) re-used as (centre, size)."""
    pri = (np.array(YOLO_PRIORS[level][a], F32) / F32([8.0, 16.0, 32.0][level])).astype(F32)
    ayx = np.array([y + 0.5, x + 0.5], F32)
    c, s = (ayx - pri / F32(2.0)).astype(F32), (ayx + pri / F32(2.0)).astype(F32)
    return (c - s / F32(2.0)).astype(F32), (c + s / F32(2.0)).astype(F32)


def _yolo_noobj_edge():
    """YOLO no-object rule best <= 0.5: a GT twice as high as the no-object box of cell (1,1), prior 0 of the
    13x13-role level, has IoU exactly 0.5 with it (still no-object).  That anchor's objectness logit is
    large so the term it contributes shows."""
    geo = YOLO_SMALL
    b1, b2 = _yolo_noobj_quirk_box(geo, 0, 1, 1, 0)
    c, hw = (b1 + b2) / F32(2.0), (b2 - b1)
    gt = np.array([[c[0] * 32, c[1] * 32, hw[0] * 64, hw[1] * 32, 2], [-1] * 5], F32)
    g = (gt[0, :4] / F32(32)).astype(F32)
    g1, g2 = (g[:2] - g[2:] / F32(2.0)).astype(F32), (g[:2] + g[2:] / F32(2.0)).astype(F32)
    inter = F32(np.prod(np.minimum(g2, b2) - np.maximum(g1, b1)))
    area_b, area_g = F32(np.prod(b2 - b1)), F32(np.prod(g2 - g1))
    assert F32(inter / F32(area_b + area_g - inter)) == F32(0.5)
    assert tuple(np.floor(g[:2]).astype(int)) != (1, 1)   # the cell holds no GT centre
    n = geo.index(0, 1, 1, 0)
    gt2 = gt.copy()
    gt2[0, 2] = np.nextafter(gt[0, 2], F32(0))
    rows = make_rows("yolo", geo.N, seed=30)[0]
    rows[n, 24] = 20.0
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))


def _yolo_cell_boundary():
    """YOLO GT centres exactly on cell boundaries of every level (floor of an integer)."""
    geo = YOLO_SMALL
    gt = np.array([[64, 96, 50, 40, 1], [32, 128, 120, 90, 8], [-1] * 5], F32)
    gt2 = gt.copy()
    gt2[0, 0] = np.nextafter(F32(64), F32(0))
    rows = make_rows("yolo", geo.N, seed=31)[0]
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))


def yolo_level_iou(g):
    """IoU [3 levels, 3 priors] of one GT row (pixels) with the priors at its own cell, in the oracle's
    operation order (unclamped intersections, level k normalised by 32 / 16 / 8)."""
    out = []
    for k in range(3):
        pri = (np.array(YOLO_PRIORS[k], F32) / F32([8.0, 16.0, 32.0][k])).astype(F32)
        gn = (np.asarray(g[:4], F32) / F32([32.0, 16.0, 8.0][k])).astype(F32)
        ayx = (np.floor(gn[:2]) + F32(0.5)).astype(F32)
        a1, a2 = (ayx - pri / F32(2)).astype(F32), (ayx + pri / F32(2)).astype(F32)
        g1, g2 = (gn[:2] - gn[2:] / F32(2.0)).astype(F32), (gn[:2] + gn[2:] / F32(2.0)).astype(F32)
        inter = np.prod(np.minimum(g2, a2) - np.maximum(g1, a1), axis=-1).astype(F32)
        garea = np.prod(g2 - g1).astype(F32)
        aarea = np.prod(pri, axis=-1).astype(F32)
        out.append((inter / (aarea + garea - inter)).astype(F32))
    return np.stack(out)


def _yolo_level_tie():
    """YOLO level choice on ties: this GT's best prior IoU is the same fp32 value on the 32- and 16-normalised
    levels and lower on the 8-normalised one.  The strict comparisons send a tie to level 2."""
    geo = YOLO_SMALL
    gt = np.array([[68, 68, 82, 142.31303, 12], [-1] * 5], F32)
    mx = yolo_level_iou(gt[0]).max(axis=1)
    assert mx[0] == mx[1] and mx[0] > mx[2], mx
    gt2 = gt.copy()

    def broken(w):
        gt2[0, 3] = w
        m = yolo_level_iou(gt2[0]).max(axis=1)
        return m[0] != m[1]
    gt2[0, 3] = step_until(gt[0, 3], 1e9, broken)
    rows = make_rows("yolo", geo.N, seed=33)[0]
    return dict(geo=geo, rows=rows, gt=gt, nudged=(rows, gt2))


def _yolo_prior_tie():
    """YOLO first-max prior on ties: a 1e21-pixel GT has h*w = inf at every level, so every prior's IoU is
    inter / inf = 0 while log(h / prior) stays finite.  Level 2 and its prior 0 are chosen.  The three prior
    rows of that cell get different size deltas.  No input step breaks this tie, so the other side of the
    decision is stated to the oracle directly: the cell's three rows and the level's priors in reverse order
    make its first maximum the last prior."""
    geo = YOLO_SMALL
    gt = np.array([[80, 80, 1e21, 1e21, 4], [-1] * 5], F32)
    with np.errstate(over="ignore"):
        iou = yolo_level_iou(gt[0])
    assert np.all(iou == 0), iou
    cell = [geo.index(2, 10, 10, a) for a in range(3)]
    rows = make_rows("yolo", geo.N, seed=34)[0]
    rows[cell, 22:24] = np.array([[0.0, 0.0], [2.0, 2.0], [4.0, 4.0]], F32)
    rows_alt = rows.copy()
    rows_alt[cell] = rows[cell[::-1]]
    priors_alt = [YOLO_PRIORS[0], YOLO_PRIORS[1], YOLO_PRIORS[2][::-1]]
    return dict(geo=geo, rows=rows, gt=gt, nudged=None, other=(rows_alt, gt, dict(priors=priors_alt)))


EDGE_CASES = {
    "retina_pos_0.5": _retina_pos_edge,
    "retina_neg_0.4": _retina_neg_edge,
    "retina_best_anchor_tie": _retina_best_tie,
    "ssd_pos_0.5": _ssd_pos_edge,
    "ssd_mining_tie": _ssd_mining_tie,
    "ssd_mining_dry": _ssd_mining_dry,
    "fcos_edge_on_grid": _fcos_grid_edge,
    "fcos_level_64": _fcos_level_bound(64),
    "fcos_level_128": _fcos_level_bound(128),
    "fcos_level_256": _fcos_level_bound(256),
    "fcos_level_512": _fcos_level_bound(512),
    "fcos_equal_area": _fcos_equal_area,
    "yolo_noobj_0.5": _yolo_noobj_edge,
    "yolo_centre_on_cell_boundary": _yolo_cell_boundary,
    "yolo_level_tie": _yolo_level_tie,
    "yolo_prior_tie": _yolo_prior_tie,
}


# ------------------------------------------------------------ CPU guards ------
@pytest.mark.parametrize("name", sorted(EDGE_CASES))
def test_edge_case_is_on_the_edge(name):
    """The builder's own assertions pin the edge; here: one step across it moves the oracle loss by at least
    100x the GPU tolerance (so a kernel deciding the other way fails), and the loss is finite."""
    c = EDGE_CASES[name]()
    ref, info = oracle(c["geo"], c["rows"], c["gt"])
    assert np.isfinite(ref)
    if name == "ssd_mining_dry":
        num_pos, num_neg, sel = info
        chosen = min(num_neg, 3 * num_pos)
        assert sel < chosen, info
        return
    rows2, gt2, kw = c["other"] if c["nudged"] is None else (*c["nudged"], {})
    ref2, _ = oracle(c["geo"], rows2, gt2, **kw)
    assert np.isfinite(ref2) and abs(ref2 - ref) >= 100 * TOL * max(abs(ref), 1.0), (ref, ref2)


def test_fcos_subcell_gt_is_inf_in_the_oracle():
    """A GT smaller than one P3 stride with no grid point strictly inside: the reference's level loss divides
    by zero positive cells; the centre-ness sum is positive, so the loss is +inf."""
    geo = FCOS_SMALL
    gt = np.array([[12, 12, 6, 6, 2], [-1] * 5], F32)
    assert oracle(geo, make_rows("fcos", geo.N, seed=32)[0], gt)[0] == np.inf


# ---------------------------------------------------- argument rejection -----
def test_loss_entry_points_reject_bad_arguments_without_gpu(built):
    """Every check runs on the host before any launch: no device is touched."""
    from odt_b200 import lib
    L = lib.load()
    fake = ctypes.c_void_p(64)  # never dereferenced: every call below is rejected first

    def params(kind, levels, A=3):
        p = lib.TailParams()
        p.kind, p.num_levels, p.N, p.num_fg = kind, levels, 64, 20
        for i in range(levels):
            p.level[i].A = A
        return p

    def rejected(rc):
        return rc == -1 and b"invalid argument" in L.odt_last_error()

    ssd, fcos, yolo = params(lib.DECODE_SSD, 1), params(lib.DECODE_FCOS, 5), params(lib.DECODE_YOLO3, 3)
    retina = lambda p, B, G, scratch=fake: L.odt_retina_loss_fwd(fake, ctypes.byref(p), B, fake, G, 0.25, 2.0,
                                                                 scratch, fake, None)
    ssd_fwd = lambda p, B, G, scratch=fake: L.odt_ssd_loss_fwd(fake, ctypes.byref(p), B, fake, G, scratch, fake,
                                                               None, None)
    fcos_fwd = lambda p, B, G, scratch=fake: L.odt_fcos_loss_fwd(fake, ctypes.byref(p), B, fake, G, scratch, fake,
                                                                 None)
    yolo_fwd = lambda p, B, G, scratch=fake: L.odt_yolo_loss_fwd(fake, ctypes.byref(p), B, fake, G, 1.0, 1.0, 5.0,
                                                                 1.0, scratch, fake, None)
    for fwd, p in ((retina, ssd), (ssd_fwd, ssd), (fcos_fwd, fcos), (yolo_fwd, yolo)):
        for B, G in ((1, 0), (1, 129), (0, 4), (-1, 4)):
            assert rejected(fwd(p, B, G)), (fwd, B, G)
        wrong = yolo if p is not yolo else ssd
        assert rejected(fwd(wrong, 1, 4)), "wrong head kind"
        assert rejected(fwd(p, 1, 4, scratch=ctypes.c_void_p(68))), "unaligned scratch"
    assert rejected(fcos_fwd(params(lib.DECODE_FCOS, 3), 1, 4)), "FCOS level count"
    assert rejected(yolo_fwd(params(lib.DECODE_YOLO3, 2), 1, 4)), "YOLO level count"
    assert rejected(yolo_fwd(params(lib.DECODE_YOLO3, 3, A=2), 1, 4)), "YOLO priors per level"
    for family, p in (("retina", ssd), ("ssd", ssd), ("fcos", fcos), ("yolo", yolo)):
        size = getattr(L, "odt_%s_loss_scratch_bytes" % family)
        for B in (0, -3):
            assert size(ctypes.byref(p), B) == -1, (family, B)
        assert size(None, 2) == -1, family
        assert size(ctypes.byref(p), 2) > 0, family


# ------------------------------------------------------------------- GPU ------
def gpu_loss(geo, rows, gt, **kw):
    """Kernel losses [B] (+ SSD info [B,3]) on rows [B,N,25] and gt [B,G,5]."""
    from odt_b200.engine import RowsHarness
    h = RowsHarness(geo.tail(), geo.levels, rows)
    if geo.kind == "ssd":
        return h.loss("ssd", gt, return_info=True)
    return h.loss(geo.kind, gt, **kw), None


def check_images(geo, rows, gt, got, info, images, **kw):
    bad = []
    for b in images:
        ref, ri = oracle(geo, rows[b], gt[b], **kw)
        if not close(got[b], ref) or (ri is not None and tuple(info[b]) != ri):
            bad.append((b, float(got[b]), ref, None if info is None else tuple(info[b]), ri))
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(EDGE_CASES))
def test_edge_case_matches_oracle(built, name):
    """The kernel on the edge and one step across it (B=2: both sides in one launch)."""
    c = EDGE_CASES[name]()
    rows2, gt2 = c["nudged"] if c["nudged"] is not None else (c["rows"], c["gt"])
    rows = np.stack([c["rows"], rows2])
    gt = np.stack([c["gt"], gt2])
    got, info = gpu_loss(c["geo"], rows, gt)
    check_images(c["geo"], rows, gt, got, info, range(2))


@pytest.mark.gpu
def test_fcos_subcell_gt_is_inf_on_gpu(built):
    """Reference behaviour pinned, not fixed: a level with GT but no positive cell gives +inf."""
    geo = FCOS_SMALL
    gt = np.array([[[12, 12, 6, 6, 2], [-1] * 5]], F32)
    got, _ = gpu_loss(geo, make_rows("fcos", geo.N, seed=32), gt)
    assert got[0] == np.inf


def capacity_gt(kind, seed):
    """G = 128 in three forms, one per image: padded in the last row only; unpadded (the first minimum of
    column 0 -- at row 100 -- is the valid count); two tied minima of column 0 (rows 40 and 90)."""
    size = IMG[kind]
    rng = np.random.default_rng(seed)
    lo = 0.15 if kind == "fcos" else 0.08  # FCOS: no sub-stride boxes (their loss is +inf, tested above)
    gt = np.stack([random_gt(rng, 127, size, 128, lo=lo), random_gt(rng, 128, size, 128, lo=lo),
                   random_gt(rng, 128, size, 128, lo=lo)])
    gt[1, 100, 0] = 0.05 * size
    gt[2, 40, 0] = gt[2, 90, 0] = 0.04 * size
    assert int(np.argmin(gt[1], axis=0)[0]) == 100 and int(np.argmin(gt[2], axis=0)[0]) == 40
    return gt


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["retina", "ssd", "fcos", "yolo"])
def test_full_gt_capacity(built, kind):
    geo = TAIL_GEOS[kind]
    gt = capacity_gt(kind, seed=40)
    rows = make_rows(kind, geo.N, batch=3, seed=41)
    got, info = gpu_loss(geo, rows, gt)
    check_images(geo, rows, gt, got, info, range(3))


def batch65_gt(kind, seed):
    """B = 65 (one image past the 64-image block of the final kernels), G = 128: valid counts 1, 2, 127 and
    128, duplicated GT rows, one GT-free image (index 5), random counts elsewhere."""
    size = IMG[kind]
    rng = np.random.default_rng(seed)
    lo = 0.15 if kind == "fcos" else 0.08
    counts = [1, 2, 127, 128, 9, 0] + list(rng.integers(1, 40, 59))
    gt = np.stack([random_gt(rng, int(n), size, 128, lo=lo) for n in counts])
    gt[4, 3:6] = gt[4, 2]                # three duplicates of one box
    gt[64, :6] = random_gt(rng, 3, size, 6, lo=lo)[[0, 0, 1, 1, 2, 2]]
    gt[64, 6:] = -1.0
    return gt


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["retina", "ssd", "fcos", "yolo"])
def test_batch_of_65_and_isolation(built, kind):
    """Every image with GT matches the oracle; the GT-free image disturbs nobody (FCOS gives 0 there, the
    oracle's value; the other three divide 0 by 0, a case the reference leaves undefined); a second launch
    is bit-identical; every image's loss is bit-identical to the same image run alone at B=1."""
    geo = TAIL_GEOS[kind]
    gt = batch65_gt(kind, seed=50)
    rows = make_rows(kind, geo.N, batch=65, seed=51)
    got, info = gpu_loss(geo, rows, gt)
    images = [b for b in range(65) if b != 5]
    check_images(geo, rows, gt, got, info, images)
    if kind == "fcos":
        assert got[5] == 0.0
    again, info2 = gpu_loss(geo, rows, gt)
    np.testing.assert_array_equal(again, got)
    if info is not None:
        np.testing.assert_array_equal(info2, info)
    for b in range(65):
        alone, ia = gpu_loss(geo, rows[b:b + 1], gt[b:b + 1])
        assert alone[0].tobytes() == got[b].tobytes(), (b, alone[0], got[b])
        if info is not None:
            assert tuple(ia[0]) == tuple(info[b])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ssd", "yolo"])
def test_tiny_geometry_below_one_anchor_per_block(built, kind):
    """N < 64: one SSD level of 3x3x4 anchors, and a YOLO table of 1x1, 2x2, 4x4 cells (N = 63)."""
    geo = SSD_TINY if kind == "ssd" else Geo("yolo", 32, [(1, 1, 3), (2, 2, 3), (4, 4, 3)])
    assert geo.N < 64
    rng = np.random.default_rng(60)
    gt = np.stack([random_gt(rng, n, geo.size, 8, lo=0.2, hi=0.9) for n in (1, 3, 7)])
    rows = make_rows(kind, geo.N, batch=3, seed=61)
    got, info = gpu_loss(geo, rows, gt)
    check_images(geo, rows, gt, got, info, range(3))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["retina", "ssd", "fcos", "yolo"])
def test_saturated_rows(built, kind):
    """Logits at +-60; FCOS size deltas at 100 (exp overflows to inf, the IoU goes to 0) and YOLO size deltas
    at 1e20 (the squared error overflows): kernel and oracle agree, inf included."""
    geo = TAIL_GEOS[kind]
    rows = make_rows(kind, geo.N, batch=2, seed=70)
    ncls = 21 if kind in ("ssd", "retina") else 20
    rows[..., :ncls] = np.where(rows[..., :ncls] > 0, 60.0, -60.0)
    if kind == "fcos":
        rows[..., 20] = np.where(rows[..., 20] > 1, 60.0, -60.0)
        rows[1, :, 21:25] = 100.0
    if kind == "yolo":
        rows[..., 24] = np.where(rows[..., 24] > 1, 60.0, -60.0)
        rows[1, :, 22:24] = 1e20
    rng = np.random.default_rng(71)
    lo = 0.15 if kind == "fcos" else 0.08
    gt = np.stack([random_gt(rng, 6, IMG[kind], 8, lo=lo), random_gt(rng, 5, IMG[kind], 8, lo=lo)])
    got, info = gpu_loss(geo, rows, gt)
    check_images(geo, rows, gt, got, info, range(2))
    if kind == "yolo":
        assert got[1] == np.inf


def full_size(kind):
    """Level table of the full-size network (the engine's own, built without touching the GPU), its input
    size and the decode tail."""
    import importlib
    from odt_b200 import engine as E
    mod, cfg_kind, size = {"ssd300": ("SSD300", "ssd", 300), "ssd512": ("SSD512", "ssd", 512),
                           "retinanet800": ("RetinaNet", "retinanet", 800), "yolov3_416": ("YOLOv3", "yolov3", 416),
                           "fcos1024": ("FCOS", "fcos", 1024)}[kind]
    m = getattr(importlib.import_module(mod), mod)(model_cfg(cfg_kind, data_shape=[size, size, 3]), None)
    E.Net.spec_only = True
    try:
        net, _ = m._build(1, "fp32", False)
    finally:
        E.Net.spec_only = False
    gkind = {"ssd": "ssd", "retinanet": "retina", "yolov3": "yolo", "fcos": "fcos"}[cfg_kind]
    return Geo(gkind, size, net.levels)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,B", [("ssd300", 4), ("ssd512", 4), ("retinanet800", 4), ("yolov3_416", 4),
                                    ("fcos1024", 4)])
def test_full_size_geometry(built, kind, B):
    """Full-size anchor tables, B = 4, G = 128 realistic boxes (3% to 60% of the image side)."""
    geo = full_size(kind)
    # SSD: conv10_2 has stride 1 in the reference, so SSD300 has two 5x5 levels and SSD512 two 8x8 levels
    assert geo.N == {"ssd300": 8828, "ssd512": 24912, "retinanet800": 120087, "yolov3_416": 10647,
                     "fcos1024": 21824}[kind]
    rng = np.random.default_rng(80)
    lo = 0.03 if geo.kind != "fcos" else 0.04
    gt = np.stack([random_gt(rng, n, geo.size, 128, lo=lo) for n in (128, 127, 64, 128)[:B]])
    rows = make_rows(geo.kind, geo.N, batch=B, seed=81)
    got, info = gpu_loss(geo, rows, gt)
    check_images(geo, rows, gt, got, info, range(B))
