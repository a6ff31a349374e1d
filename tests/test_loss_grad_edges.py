"""The loss-gradient kernels' edges without a GPU: the constructed cases tests/test_gpu_loss_grad_edges.py runs (the
FCOS min(d, exp(r)) tie, the smooth-L1 kinks, RetinaNet's clamp of the label probability at 1e-8, label probabilities
that round to exactly 1), checks that each sits on its edge as the float32 kernels compute it, TF's tie rule in the
restatement, and the gradient bar (loss_grad_ref.bar) itself: it admits the float32 restatement against the float64
one on every case whose decisions agree, and rejects each planted gradient bug -- a mutation of the float64
restatement's gradient -- on a case where the bug matters."""
import numpy as np
import pytest
import torch

import loss_grad_ref as LR
import test_gpu_loss as GL
from helpers import YOLO_PRIORS

F32 = np.float32
ULP1 = 2.0 ** -23  # relative spacing of float32 in [1, 2)
STRADDLE_K = (-1024, -64, -4, -1, 0, 1, 4, 64, 1024)  # label probability 1e-8 * (1 + k * ULP1)
YOLO_SCALES = dict(coord_scale=2.0, noobj_scale=0.5, obj_scale=5.0, class_scale=1.5)


# ------------------------------------------------------------------------------------------------- cases --
def kernel_anchor(kind, size, cfg, levels, n):
    """(cy, cx, h, w) of anchor row n as csrc/tail_common.cuh anchor_ssd computes it in float32."""
    p = LR.tail(kind, size, cfg).params(levels)
    off = 0
    for i, (h, w, a) in enumerate(levels):
        if n < off + h * w * a:
            break
        off += h * w * a
    y, x, a = (n - off) // (w * a), (n - off) // a % w, (n - off) % a
    L = p.level[i]
    cy = F32(F32(F32(y + 0.5) * F32(L.cmul_y)) / F32(L.cdiv_y))
    cx = F32(F32(F32(x + 0.5) * F32(L.cmul_x)) / F32(L.cdiv_x))
    hh, hw = F32(F32(L.prior_h[a]) * F32(0.5)), F32(F32(L.prior_w[a]) * F32(0.5))
    y1, x1, y2, x2 = cy - hh, cx - hw, cy + hh, cx + hw
    return (F32(y1 * F32(0.5) + y2 * F32(0.5)), F32(x1 * F32(0.5) + x2 * F32(0.5)), F32(y2 - y1), F32(x2 - x1))


def kernel_box_target(anchor, g):
    """The smooth-L1 targets (y, x, h, w) of loss_anchor_grad_kernel for GT row g at an anchor, in float32."""
    cy, cx, h, w = anchor
    return (F32(F32(g[0] - cy) / h), F32(F32(g[1] - cx) / w), np.log(F32(g[2] / h)), np.log(F32(g[3] / w)))


ONE_M, ONE_P = np.nextafter(F32(1), F32(0)), np.nextafter(F32(1), F32(2))
KINK_DELTAS = (np.array([0, 1, -1, ONE_P], F32), np.array([ONE_M, -ONE_M, -ONE_P, 0], F32))


def _kink(kind):
    """Smooth-L1 at |d| = 1 and d = 0: two GTs equal to an anchor each (target exactly 0 in the kernel), that anchor's
    box deltas 0, +-1 and +-1 +- 1 ulp."""
    geo = GL.RET_SMALL if kind == "retina" else GL.SSD_FINE
    size = geo.size
    cfg = LR.config(kind, size)
    picks = (geo.index(0, 3, 3, 0), geo.index(0, 5, 6, 2)) if kind == "retina" else \
        (geo.index(0, 10, 12, 0), geo.index(0, 25, 20, 3))
    gt = np.full((6, 5), -1.0, F32)
    for j, n in enumerate(picks):
        gt[j, :4] = kernel_anchor(kind, size, cfg, geo.levels, n)
        gt[j, 4] = 3 + 5 * j
    gt[2] = [0.3 * size, 0.6 * size, 0.3 * size, 0.25 * size, 9]
    rows = LR.rows(kind, geo.N, seed=60)[0]
    for n, d in zip(picks, KINK_DELTAS):
        rows[n, 21:25] = d
    return dict(kind=kind, levels=geo.levels, size=size, cfg=cfg, nc=20, rows=rows, gt=gt, picks=picks, geo=geo)


def _fcos_tie():
    """FCOS min(d, exp(r)) ties: a 48 x 32 GT whose P3 edges lie on whole strides (x1 = 3, x2 = 9, y1 = 4, y2 = 8),
    every P3 distance logit 0 (exp = 1): the cells one stride inside an edge have d = 1 = exp(r).  A second GT on P4
    only, so two levels carry a loss with different counts."""
    geo = GL.FCOS_SMALL
    gt = np.full((4, 5), -1.0, F32)
    gt[0] = [48, 48, 32, 48, 3]
    gt[1] = [64, 64, 96, 80, 7]
    rows = LR.rows("fcos", geo.N, seed=61)[0]
    rows[:16 * 16, 21:25] = 0.0
    ties = [(geo.index(0, y, x), c) for y in range(5, 8) for x in range(4, 9)
            for c, hit in ((21, x == 4), (22, x == 8), (23, y == 5), (24, y == 7)) if hit]
    return dict(kind="fcos", levels=geo.levels, size=geo.size, cfg=LR.config("fcos", geo.size), nc=20, rows=rows,
                gt=gt, ties=ties, geo=geo)


def straddle_logits(q):
    """21 float32 logits whose float64 softmax gives class 20 the probability q: 19 zeros (the row maximum, so every
    x - max is exact in float32), class 20 at x and class 0 at y < 0, y the float32 value closest to the solution."""
    x = F32(np.log(q * 19.5))
    ey = np.exp(np.float64(x)) / q - np.exp(np.float64(x)) - 19.0
    y0 = F32(np.log(ey))
    cand = [y0]
    for _ in range(4):
        cand += [np.nextafter(cand[-2 if len(cand) > 1 else 0], F32(-1)), np.nextafter(cand[-1], F32(1))]
    row = np.zeros(21, F32)
    row[20] = x

    def p64(y):
        r = row.astype(np.float64)
        r[0] = y
        e = np.exp(r - r.max())
        return e[20] / e.sum()
    row[0] = min(cand, key=lambda y: abs(p64(y) - q))
    return row, p64(row[0])


def q_one_logits(label):
    """Logits whose float32 softmax puts exactly 1 on `label` (the 20 others at -25: their sum is under half an ulp
    of 1)."""
    r = np.full(21, -25.0, F32)
    r[label] = 0.0
    return r


def _retina_clamp():
    """RetinaNet's clamp at 1e-8: nine negatives with background probability 1e-8 * (1 + k 2^-23) for k in
    STRADDLE_K, and three negatives and one positive whose label probability rounds to exactly 1 in float32."""
    geo, size = GL.RET_SMALL, 64
    gt = np.full((4, 5), -1.0, F32)
    gt[0] = [20, 22, 24, 20, 4]
    gt[1] = [44, 40, 18, 30, 11]
    rows = LR.rows("retina", geo.N, seed=62)[0]
    iou = GL.match_iou(geo, gt)
    best = set(np.argmax(iou, axis=1).tolist())
    neg = [int(n) for n in np.flatnonzero(iou.max(0) < 0.4) if n not in best]
    straddle = neg[:len(STRADDLE_K)]
    p64 = []
    for n, k in zip(straddle, STRADDLE_K):
        rows[n, :21], p = straddle_logits(1e-8 * (1 + k * ULP1))
        p64.append(p)
    ones = neg[-3:]
    for n in ones:
        rows[n, :21] = q_one_logits(20)
    pos = int(np.argmax(iou[0]))
    rows[pos, :21] = q_one_logits(4)
    return dict(kind="retina", levels=geo.levels, size=size, cfg=LR.config("retina", size), nc=20, rows=rows, gt=gt,
                straddle=straddle, p64=np.array(p64), ones=ones + [pos], geo=geo)


# Rows whose float64 label probability lies within CLAMP_BAND_ULPS float32 ulps of 1e-8 may fall on either side of the
# clamp in a float32 softmax (expf within 2 ulps on 21 terms, their sum and a division: under 8 ulps).
CLAMP_BAND_ULPS = 16


def retina_npos(c):
    iou = GL.match_iou(c["geo"], c["gt"])
    best = np.argmax(iou, axis=1)
    return len(best) + int(np.sum(np.delete(iou.max(0), np.unique(best)) > 0.5))


def focal_row_grad(c, n, label):
    """float64 gradient of row n's focal term on `label` as if its probability were inside the clamp (the box columns
    get none: a negative)."""
    alpha, gam = c["cfg"]["alpha"], c["cfg"]["gamma"]
    p = _softmax64(np.asarray(c["rows"][n], np.float64))
    q = p[label]
    dq = -alpha * ((1 - q) ** gam / q - gam * (1 - q) ** (gam - 1) * np.log(q))
    hot = np.zeros(21)
    hot[label] = 1
    out = np.zeros(25)
    out[:21] = dq * q * (hot - p) / retina_npos(c)
    return out


def resolve_clamp(c, got, ref):
    """The reference of a retina_clamp image with each straddle row on the side `got` took (all zeros: clamped),
    after checking that rows outside the band took the reference's side.  Returns (reference, [(k, side)] of the
    rows in the band)."""
    ref = ref.copy()
    band = []
    for n, k in zip(c["straddle"], STRADDLE_K):
        clamped = not np.any(got[n] != 0)
        if abs(k) > CLAMP_BAND_ULPS:
            assert clamped == (k < 0), (k, got[n])
        else:
            band.append((k, "clamped" if clamped else "inside"))
        ref[n] = 0.0 if clamped else focal_row_grad(c, n, 20)
    return ref, band


CASES = {"retina_kink": lambda: _kink("retina"), "ssd_kink": lambda: _kink("ssd"), "fcos_tie": _fcos_tie,
         "retina_clamp": _retina_clamp}


def softmax32(r):
    """loss_anchor_grad_kernel's float32 softmax of one row's 21 logits (max subtracted, expf, sum, division)."""
    z = (r[:21] - r[:21].max()).astype(F32)
    e = np.exp(z).astype(F32)
    return (e / e.sum(dtype=F32)).astype(F32)


# ------------------------------------------------------------------------------------------- on the edge --
def test_fcos_tie_is_exact_in_float32():
    c = _fcos_tie()
    assert len(c["ties"]) == 16
    gy, gx, gh, gw = (c["gt"][0, :4] / F32(8)).astype(F32)
    x1, x2 = F32(gx - F32(gw / F32(2))), F32(gx + F32(gw / F32(2)))
    y1, y2 = F32(gy - F32(gh / F32(2))), F32(gy + F32(gh / F32(2)))
    assert (x1, x2, y1, y2) == (3, 9, 4, 8)
    assert F32(F32(4) - x1) == 1 and F32(x2 - F32(8)) == 1 and F32(F32(5) - y1) == 1 and F32(y2 - F32(7)) == 1
    assert np.exp(F32(0)) == F32(1)
    for n, col in c["ties"]:
        assert c["rows"][n, col] == 0


@pytest.mark.parametrize("kind", ["retina", "ssd"])
def test_gt_equal_to_an_anchor_has_target_zero(kind):
    c = _kink(kind)
    for j, n in enumerate(c["picks"]):
        anchor = kernel_anchor(kind, c["size"], c["cfg"], c["levels"], n)
        assert kernel_box_target(anchor, c["gt"][j]) == (0, 0, 0, 0)
        assert int(np.argmax(GL.match_iou(c["geo"], c["gt"])[j])) == n  # the anchor is the GT's best
    assert ONE_M == F32(1) - F32(2 ** -24) and ONE_P == F32(1) + F32(ULP1)


def test_retina_straddle_rows_sit_at_the_clamp():
    c = _retina_clamp()
    for k, p in zip(STRADDLE_K, c["p64"]):
        assert abs(p / 1e-8 - 1 - k * ULP1) <= 0.05 * ULP1, (k, p)
    for n in c["straddle"]:
        assert abs(softmax32(c["rows"][n])[20] / F32(1e-8) - 1) < 2e-4  # |k| <= 1024 ulps


def test_some_rows_round_q_to_exactly_one():
    c = _retina_clamp()
    labels = [20, 20, 20, 4]
    for n, lab in zip(c["ones"], labels):
        q = softmax32(c["rows"][n])
        assert q[lab] == F32(1) and 0 < q[(lab + 1) % 21] < 1e-10
        z = c["rows"][n].astype(np.float64)
        assert np.exp(z[lab]) / np.exp(z[:21]).sum() < 1.0  # float64 stays below 1


# ------------------------------------------------------------------------------------------ TF tie rule --
def test_tf_minimum_gives_the_tie_to_the_first_argument():
    from odt_b200.train import tf_minimum
    d = torch.tensor([1.0, 2.0, 1.0], dtype=torch.float64)
    p = torch.tensor([1.0, 1.5, 3.0], dtype=torch.float64, requires_grad=True)
    tf_minimum(d, p).sum().backward()
    assert p.grad.tolist() == [0.0, 1.0, 0.0]
    p2 = p.detach().clone().requires_grad_(True)
    torch.minimum(d, p2).sum().backward()
    assert p2.grad.tolist() == [0.5, 1.0, 0.0]  # what the restatement must not do


def _tie_split(monkeypatch, c):
    from odt_b200 import train
    with monkeypatch.context() as m:
        m.setattr(train, "tf_minimum", torch.minimum)
        return LR.grad(LR.restatement("fcos", c["levels"], c["cfg"], c["size"]), c["rows"], c["gt"])[1]


def test_fcos_restatement_follows_tf_at_the_tie(monkeypatch):
    """At a tie the prediction's gradient is the union term alone: -dl_diou * iou * psum / u * p * inv.  The 0.5 / 0.5
    split of torch.minimum adds half the intersection term."""
    c = _fcos_tie()
    g = LR.grad(LR.restatement("fcos", c["levels"], c["cfg"], c["size"]), c["rows"], c["gt"])[1]
    split = _tie_split(monkeypatch, c)
    for n, col in c["ties"]:
        assert g[n, col] != split[n, col]
        assert abs(g[n, col]) < abs(split[n, col]) or np.sign(g[n, col]) != np.sign(split[n, col])
    off_tie = np.ones(g.shape, bool)
    for n, col in c["ties"]:
        off_tie[n, col] = False
    np.testing.assert_array_equal(g[off_tie], split[off_tie])


# ------------------------------------------------------------------------------------------------- the bar --
def _ref(c):
    return LR.reference(c["kind"], c["levels"], c["cfg"], c["size"], c["nc"], c["rows"], c["gt"])


def _yolo_case(seed, n_gt=1, nc=20):
    geo = GL.YOLO_SMALL
    cfg = LR.config("yolo", geo.size, nc=nc, priors=YOLO_PRIORS, **YOLO_SCALES)
    gt = LR.gt(np.random.default_rng(seed), n_gt, geo.size, 4, nc=nc)
    return dict(kind="yolo", levels=geo.levels, size=geo.size, cfg=cfg, nc=nc,
                rows=LR.rows("yolo", geo.N, nc=nc, seed=seed)[0], gt=gt, geo=geo)


def _yolo2_case(levels, seed, A=5):
    cfg = LR.config("yolo2", 32 * levels[0][1], A=A)
    N = sum(h * w * a for h, w, a in levels)
    gt = np.full((4, 5), -1.0, F32)
    h, w, _ = levels[0]
    gt[:2] = [[16 * h, 8 * w, 20 * h, 12 * w, 2], [9 * h, 25 * w, 6 * h, 9 * w, 17]]
    return dict(kind="yolo2", levels=levels, size=32 * w, cfg=cfg, nc=20,
                rows=LR.rows("yolo2", N, seed=seed)[0], gt=gt)


def _ssd_dup():
    geo = GL.SSD_FINE
    gt = LR.gt(np.random.default_rng(63), 4, 300, 8, lo=0.15, hi=0.5)
    gt[4] = gt[1]
    gt[4, 4] = 13 if gt[1, 4] != 13 else 14
    return dict(kind="ssd", levels=geo.levels, size=300, cfg=LR.config("ssd", 300), nc=20,
                rows=LR.rows("ssd", geo.N, seed=64)[0], gt=gt, geo=geo)


def _retina_random():
    geo = GL.RET_SMALL
    gt = LR.gt(np.random.default_rng(65), 3, 64, 6, lo=0.3, hi=0.7)
    return dict(kind="retina", levels=geo.levels, size=64, cfg=LR.config("retina", 64), nc=20,
                rows=LR.rows("retina", geo.N, seed=66)[0], gt=gt, geo=geo)


HONEST = {**CASES, "ssd_dup": _ssd_dup, "retina_random": _retina_random, "yolo_one_gt": lambda: _yolo_case(67),
          "yolo2_1025": lambda: _yolo2_case([(5, 41, 5)], 68)}


@pytest.mark.parametrize("name", sorted(HONEST))
def test_bar_admits_the_float32_restatement(name):
    """An honest float32 computation passes: the float32 restatement against the float64 one, where they decide
    alike."""
    c = HONEST[name]()
    _, g64, dt, g32 = _ref(c)
    if name == "retina_clamp":  # the straddle rows decide by float rounding: compare each on the side it took
        g64, band = resolve_clamp(c, g32, g64)
        print("float32 restatement in the clamp band of %d ulps: %s" % (CLAMP_BAND_ULPS, band))
    else:
        assert dt == "float64", "the case's decisions differ in float32"
    ok, err, scale = LR.bar(g32, g64)
    print("%s: float32 restatement max|err| %.3g of max %.3g" % (name, err, scale))
    assert ok


def _retina_sets(c):
    """(best anchors with a multiplicity per GT, negatives) of a RetinaNet / SSD case, in the kernels' float32 IoU."""
    iou = GL.match_iou(c["geo"], c["gt"])
    best = np.argmax(iou, axis=1)
    other = np.ones(iou.shape[1], bool)
    other[best] = False
    thr = 0.4 if c["kind"] == "retina" else 0.5
    neg = np.flatnonzero(other & (iou.max(0) < thr) if c["kind"] == "retina" else other & (iou.max(0) <= thr))
    return best, neg


def _softmax64(r):
    e = np.exp(r[..., :21] - r[..., :21].max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def _bug_ssd_mined_by_pos(c, g):
    tr = LR.restatement("ssd", c["levels"], c["cfg"], c["size"])
    _, npos, _, nsel = tr._ssd.image_loss(torch.tensor(c["rows"], dtype=torch.float64), c["gt"])
    _, neg = _retina_sets(c)
    mined = [n for n in neg if np.any(g[n] != 0)]
    assert len(mined) == nsel and nsel != npos
    g[mined] *= nsel / npos


def _bug_retina_neg_without_alpha(c, g):
    _, neg = _retina_sets(c)
    g[neg] /= c["cfg"]["alpha"]


def _bug_focal_without_modulation(c, g):
    """d/dq of -alpha (1-q)^gamma log q with the first term's (1-q)^gamma dropped: -alpha (1/q - gamma (1-q)^(gamma-1)
    log q), on the negatives (q = background probability)."""
    _, neg = _retina_sets(c)
    gam = c["cfg"]["gamma"]
    q = _softmax64(np.asarray(c["rows"], np.float64)[neg])[:, 20]
    true = (1 - q) ** gam / q - gam * (1 - q) ** (gam - 1) * np.log(q)
    bug = 1 / q - gam * (1 - q) ** (gam - 1) * np.log(q)
    g[neg] *= (bug / true)[:, None]


def _bug_first_gt_of_shared_best_only(c, g):
    """The shared best anchor keeps only the first GT's contribution: minus the second GT's class term, half the box
    term (the duplicate's box is the same)."""
    best, _ = _retina_sets(c)
    cnt = int(np.argmin(c["gt"][:, 0]))
    i, j = [(a, b) for a in range(cnt) for b in range(a + 1, cnt) if best[a] == best[b]][0]
    n = best[i]
    npos = retina_npos(c)
    p = _softmax64(np.asarray(c["rows"][n], np.float64))
    hot = np.zeros(21)
    hot[int(c["gt"][j, 4])] = 1
    g[n, :21] -= (p - hot) / npos
    g[n, 21:] /= 2


def _bug_fcos_centre_other_level(c, g):
    """Level 0's centre-ness column divided by level 1's positive count: the counts come from a row outside every GT,
    where the centre-ness target is 0 and the gradient is sigmoid(x) / count."""
    geo = c["geo"]
    n0, n1 = geo.index(0, 0, 0), geo.index(1, 0, 0)
    sig = 1 / (1 + np.exp(-np.asarray(c["rows"], np.float64)[:, 20]))
    cnt0, cnt1 = round(sig[n0] / g[n0, 20]), round(sig[n1] / g[n1, 20])
    assert cnt0 != cnt1
    g[:16 * 16, 20] *= cnt0 / cnt1


def _bug_yolo_noobj_strict(c, g):
    n = c["geo"].index(0, 1, 1, 0)
    assert g[n, 24] != 0
    g[n, 24] = 0.0


def _bug_yolo_class_label_plus_one(c, g):
    """One GT (divisor 1): the class gradient class_scale * (sigmoid - onehot) taken against label + 1."""
    lab, ks = int(c["gt"][0, 4]), c["cfg"]["class_scale"]
    rows = np.flatnonzero(np.any(g[:, :c["nc"]] != 0, axis=1))
    assert len(rows) == 1
    g[rows[0], lab] += ks
    g[rows[0], (lab + 1) % c["nc"]] -= ks


def _bug_last_row_unwritten(c, g):
    assert np.any(g[-1] != 0) and len(g) > 1024
    g[-1] = 0.0


PLANTED = {
    "ssd_mined_negatives_by_npos": (_ssd_dup, _bug_ssd_mined_by_pos),
    "retina_negatives_without_alpha": (_retina_random, _bug_retina_neg_without_alpha),
    "focal_derivative_without_modulation": (_retina_random, _bug_focal_without_modulation),
    "shared_best_anchor_first_gt_only": (_ssd_dup, _bug_first_gt_of_shared_best_only),
    "fcos_tie_split": (_fcos_tie, None),
    "fcos_centre_other_level_count": (_fcos_tie, _bug_fcos_centre_other_level),
    "yolo_noobj_strict": (lambda: dict(GL.EDGE_CASES["yolo_noobj_0.5"](), kind="yolo", nc=20), _bug_yolo_noobj_strict),
    "yolo_class_on_label_plus_one": (lambda: _yolo_case(69), _bug_yolo_class_label_plus_one),
    "last_grid_stride_row_unwritten": (lambda: _yolo2_case([(5, 41, 5)], 70), _bug_last_row_unwritten),
}


@pytest.mark.parametrize("name", sorted(PLANTED))
def test_bar_rejects_planted_bug(name, monkeypatch):
    make, plant = PLANTED[name]
    c = make()
    if "levels" not in c:  # an edge case of tests/test_gpu_loss.py
        c.update(levels=c["geo"].levels, size=c["geo"].size,
                 cfg=LR.config("yolo", c["geo"].size, priors=YOLO_PRIORS))
    _, ref, dt, _ = _ref(c)
    if plant is None:
        bad = _tie_split(monkeypatch, c)
    else:
        bad = ref.copy()
        plant(c, bad)
    ok, err, scale = LR.bar(bad, ref)
    print("%s (%s reference): max|err| %.3g = %.3g of max|ref| (bar %.0e)" % (name, dt, err, err / scale, LR.BAR))
    assert not ok
