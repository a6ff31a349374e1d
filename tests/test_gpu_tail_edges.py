"""The inference tail (csrc/tail.cu: decode_candidates_kernel + nms_per_class_kernel) at its selection edges,
on every candidate-list path of the NMS kernel and at full-size geometries, against the live CPU oracle
(oracle/tails.py: numpy fp32 in the reference's op order + oracle/nms_ref.c).  Bar, as tests/test_gpu_tail.py:
class ids and keep indices identical, scores within 1e-6 relative, boxes within helpers.assert_boxes_close.

Three observables beyond the packed detection record:
- the decode stage's candidate lists (`Tail.cand_count` / `Tail.cand_keys`, read between the two launches):
  every row whose oracle score clears the threshold by more than the score bar (1e-6 relative) is present
  exactly once, every row below the band is absent, rows inside it may go either way;
- the box-pool bump counter (the int64 behind the per-image counters in `Tail.work`): zeroed per launch when a
  pool exists, it then holds the summed length of the lists that took the full-list (global memory) path;
- `select_threshold`, a CPU restatement of the kernel's radix-select prefilter, which predicts from the GPU's
  own keys whether each list runs in shared memory, on a prefilter subset, on the full list after the subset
  runs dry, or on the full list because the select never resolves (more than 1 024 tied top scores).

Each exact edge is built so that the oracle sees it exactly (an IoU equal to the threshold in fp32, a score
equal to the threshold, a background probability equal to the best foreground one, a tie); CPU guards check
that taking the other side of the comparison changes the oracle's keep list."""
import os

import numpy as np
import pytest

from helpers import YOLO_PRIORS, assert_boxes_close, model_cfg

F32 = np.float32
SMEM_KEYS = 1024   # kNmsSmemKeys = kNmsPrefilter (csrc/tail.cu): longer lists try the prefilter first
SELECT_MIN = 384   # kNmsSelectMin: the prefilter subset holds at least this many keys
NUM_SMS = 132      # kNumSMs (csrc/common.cuh)
DECODE_WARPS = 8   # kDecodeWarps: one warp decodes 32 consecutive rows per iteration
BAND = 1e-6        # the score bar: a row this close to a decision edge may be decided either way


# ------------------------------------------------------------------ geometry --
class Geo:
    """kind ('ssd' | 'retina' | 'yolo' | 'fcos'), image size (SSD size / RetinaNet input width) and the
    (H, W, A) level table in candidate order."""

    def __init__(self, kind, size, levels):
        self.kind, self.size, self.levels = kind, size, [tuple(lv) for lv in levels]
        self.N = sum(h * w * a for h, w, a in self.levels)
        self.nms_classes = 19 if kind == "fcos" else 20  # FCOS decodes 20 classes, NMS visits 19

    def index(self, level, y, x, a=0):
        off = sum(h * w * aa for h, w, aa in self.levels[:level])
        _, w, A = self.levels[level]
        return off + (y * w + x) * A + a

    def tail(self, thr, mb, iou):
        from odt_b200 import nets
        kw = dict(nms_score_threshold=float(thr), nms_max_boxes=int(mb), nms_iou_threshold=float(iou))
        if self.kind == "ssd":
            return nets.ssd_tail(self.size, model_cfg("ssd", **kw))
        if self.kind == "retina":
            return nets.retina_tail(model_cfg("retinanet", data_shape=[self.size, self.size, 3], **kw))
        if self.kind == "yolo":
            return nets.yolo_tail(model_cfg("yolov3", **kw))
        return nets.fcos_tail(model_cfg("fcos", **kw))

    def scores_boxes(self, rows):
        """Oracle per-row quantities of one image (rows [N,25]): confidences [N,20], boxes [N,4], the oracle's
        background filter [N] and, for SSD / RetinaNet, the background probability [N] (else None)."""
        from oracle import tails as OT
        rows = np.asarray(rows, F32)
        with np.errstate(over="ignore", under="ignore"):
            if self.kind in ("ssd", "retina"):
                shapes = [(h, w) for h, w, _ in self.levels]
                an = (OT.ssd_anchors(self.size, shapes) if self.kind == "ssd"
                      else OT.retina_anchors([self.size, self.size, 3], shapes))
                prob, boxes, valid = OT.softmax_scores_boxes(rows[:, :21], rows[:, 21:23], rows[:, 23:], an[2],
                                                             an[3], 20)
                return prob[:, :20], boxes, valid, prob[:, 20]
            lv = OT.rows_to_levels(rows[None], self.levels, self.kind)
            if self.kind == "yolo":
                conf, boxes = OT.yolo_scores_boxes(lv, YOLO_PRIORS, 0)
            else:
                conf, boxes = OT.fcos_scores_boxes(lv, 0)
        return conf, boxes, np.ones(self.N, bool), None


TAIL_GEOS = {  # the geometries of tests/golden/make_golden.py
    "ssd": Geo("ssd", 300, [(38, 38, 4), (19, 19, 6), (10, 10, 6), (5, 5, 6), (5, 5, 4), (3, 3, 4)]),
    "retina": Geo("retina", 128, [(16, 16, 9), (8, 8, 9), (4, 4, 9), (2, 2, 9), (1, 1, 9)]),
    "yolo": Geo("yolo", 0, [(5, 5, 3), (10, 10, 3), (20, 20, 3)]),
    "fcos": Geo("fcos", 0, [(32, 32, 1), (16, 16, 1), (8, 8, 1), (4, 4, 1), (2, 2, 1)]),
}
# thresholds of the golden cases: (score, max boxes, IoU)
THR = {"ssd": (0.30, 20, 0.5), "retina": (0.25, 10, 0.45), "yolo": (0.45, 10, 0.45), "fcos": (0.40, 10, 0.45)}
YOLO48 = Geo("yolo", 0, [(48, 48, 3)])   # N = 6 912: one level, lists longer than the shared-memory window
FCOS8 = Geo("fcos", 0, [(8, 8, 1)])      # one stride-8 level

# full-size networks: module, config kind, input size, N
FULL = {"ssd300": ("SSD300", "ssd", 300, 8828), "ssd512": ("SSD512", "ssd", 512, 24912),
        "retina800": ("RetinaNet", "retinanet", 800, 120087), "yolo416": ("YOLOv3", "yolov3", 416, 10647),
        "fcos800": ("FCOS", "fcos", 800, 13343), "fcos1024": ("FCOS", "fcos", 1024, 21824)}


def full_size(name):
    """Level table of a full-size network (the engine's own, built without touching the GPU)."""
    import importlib
    from odt_b200 import engine as E
    mod, cfg_kind, size, n = FULL[name]
    m = getattr(importlib.import_module(mod), mod)(model_cfg(cfg_kind, data_shape=[size, size, 3]), None)
    E.Net.spec_only = True
    try:
        net, _ = m._build(1, "fp32", False)
    finally:
        E.Net.spec_only = False
    kind = {"ssd": "ssd", "retinanet": "retina", "yolov3": "yolo", "fcos": "fcos"}[cfg_kind]
    geo = Geo(kind, size, net.levels)
    assert geo.N == n, (name, geo.N)
    return geo


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


def logit(p):
    """fp32 logit whose sigmoid is p (to a few ulps; the cases below keep scores far apart or exactly tied)."""
    p = np.asarray(p, np.float64)
    return np.log(p / (1.0 - p)).astype(F32)


# -------------------------------------------------------------------- oracle --
def oracle_tail(geo, rows, thr, mb, iou, flip=(), sb=None):
    """Oracle detections of one image -> (scores, boxes, class ids, keep indices).  `flip` takes the other
    side of a decision: 'score' (> instead of >= score_thr), 'iou' (>= instead of > iou_thr), 'bg' (background
    dropped when >= the best foreground instead of >), 'tie' (highest row first on equal scores)."""
    from oracle import tails as OT
    conf, boxes, valid, bg = sb if sb is not None else geo.scores_boxes(rows)
    if "bg" in flip:
        valid = bg < conf.max(axis=1)
    thr = F32(thr)
    iou_eff = np.nextafter(F32(iou), F32(-1)) if "iou" in flip else F32(iou)
    out = ([], [], [], [])
    for c in range(geo.nms_classes):
        s = conf[:, c]
        idx = np.nonzero(valid & ((s > thr) if "score" in flip else (s >= thr)))[0]
        if "tie" in flip:
            idx = idx[::-1]
        sel = OT.nms_c(boxes[idx], s[idx], mb, float(iou_eff))
        for o, v in zip(out, (s[idx][sel], boxes[idx][sel], np.full(len(sel), c, np.int32), idx[sel])):
            o.append(v)
    return (np.concatenate(out[0]).astype(F32), np.concatenate(out[1]).astype(F32).reshape(-1, 4),
            np.concatenate(out[2]).astype(np.int32), np.concatenate(out[3]).astype(np.int32))


def same_result(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def select_threshold(bits):
    """The kernel's radix-select prefilter restated: for a list of score bit patterns, None if it fits the
    shared-memory window (no prefilter), -1 if the select never resolves (more than SMEM_KEYS scores tied in
    the last bin: the full list runs at once), else the threshold T: the subset is every key with score bits
    >= T, of size SELECT_MIN..SMEM_KEYS.  Four passes over 8-bit digits, high to low; each keeps the highest
    bins until SELECT_MIN keys are reached, and stops if the bin that reaches it leaves the total <= SMEM_KEYS."""
    bits = np.asarray(bits, np.uint32)
    if bits.size <= SMEM_KEYS:
        return None
    prefix, mask, carry = 0, 0, 0
    for shift in (24, 16, 8, 0):
        live = bits[(bits & np.uint32(mask)) == np.uint32(prefix)]
        hist = np.bincount(((live >> np.uint32(shift)) & np.uint32(255)).astype(np.int64), minlength=256)
        cum = carry
        for b in range(255, -1, -1):
            h = int(hist[b])
            if cum + h >= SELECT_MIN:
                prefix |= b << shift
                if cum + h <= SMEM_KEYS:
                    return prefix
                carry = cum
                break
            cum += h
        mask |= 0xFF << shift
    return -1


def list_path(bits, rows, boxes, mb, iou):
    """Path of one candidate list (score bits and rows of its keys, the image's boxes): 'smem' (<= 1 024 keys),
    'subset' (the prefilter subset yields mb boxes), 'dry' (it yields fewer: the full list runs next) or
    'full' (the select does not resolve)."""
    from oracle import tails as OT
    t = select_threshold(bits)
    if t is None:
        return "smem"
    if t == -1:
        return "full"
    sub = np.asarray(bits, np.uint32) >= np.uint32(t)
    r, sc = rows[sub], np.asarray(bits, np.uint32)[sub].view(F32)
    o = np.argsort(r, kind="stable")  # nms_c breaks ties by position: lowest row first, as the kernel's key
    return "subset" if len(OT.nms_c(boxes[r[o]], sc[o], mb, iou)) >= mb else "dry"


def oracle_lists(geo, sb, thr):
    """The oracle's candidate list of every NMS class of one image: {c: (score bits, rows)}."""
    conf, _, valid, _ = sb
    out = {}
    for c in range(geo.nms_classes):
        idx = np.nonzero(valid & (conf[:, c] >= F32(thr)))[0]
        out[c] = (conf[idx, c].view(np.uint32), idx)
    return out


# ------------------------------------------------------------------ GPU runs --
def harness(geo, rows, thr, mb, iou, cap=None, pool_cap=None):
    from odt_b200.engine import RowsHarness
    tail = geo.tail(thr, mb, iou)
    if cap is not None:
        tail.cap = cap
    if pool_cap is not None:
        tail.pool_cap = pool_cap  # box-pool entries (read when the harness prepares the tail)
    return RowsHarness(tail, geo.levels, rows)


class Snap:
    """One decode + NMS launch: per-(image, class) candidate counts and sorted keys (read between the two
    kernels: the full-list path retires keys in place), the packed records, keep indices and pool counter."""

    def __init__(self, h):
        import torch
        t, B = h.tail, h.batch
        st = torch.cuda.current_stream().cuda_stream
        t.launch_decode(h, st)
        self.cnt = t.cand_count.cpu().numpy().copy()
        keys = t.cand_keys.cpu().numpy().view(np.uint64)
        self.cap, self.D, self.B = t.p.cap, t.D, B
        self.keys = {(b, c): np.sort(keys[b, c, :min(int(self.cnt[b, c]), self.cap)])
                     for b in range(B) for c in range(t.num_fg)}
        del keys
        t.launch_nms(h, st)
        self.rec = t.rec.cpu().numpy().copy()
        self.anchor = t.det_anchor.cpu().numpy().copy()
        w = t.work.cpu().numpy()
        off = (B + 1) & ~1
        self.counter = int(w[off:off + 2].copy().view(np.int64)[0])
        self.pool_entries = t.pool_entries
        self.count = self.rec[:, self.D * 6].astype(np.int64)
        self.flags = self.rec[:, self.D * 6 + 1].copy()

    def list(self, b, c):
        """(score bits, rows, scores) of one candidate list."""
        k = self.keys[(b, c)]
        bits = (k >> np.uint64(32)).astype(np.uint32)
        rows = (np.uint64(0xFFFFFFFF) - (k & np.uint64(0xFFFFFFFF))).astype(np.int64)
        return bits, rows, bits.view(F32)

    def image(self, b):
        """(scores, boxes, class ids, keep) of image b, read from the record itself."""
        n = int(self.count[b])
        r = self.rec[b, :self.D * 6].reshape(self.D, 6)[:n]
        return r[:, 0], r[:, 1:5], r[:, 5].astype(np.int32), self.anchor[b, :n]

    def assert_same(self, other, what):
        assert self.keys.keys() == other.keys.keys()
        np.testing.assert_array_equal(self.cnt, other.cnt, err_msg=what + ": candidate counts")
        for k in self.keys:
            assert np.array_equal(self.keys[k], other.keys[k]), (what, "candidate keys", k)
        np.testing.assert_array_equal(self.count, other.count, err_msg=what + ": detection counts")
        np.testing.assert_array_equal(self.flags, other.flags, err_msg=what + ": overflow flags")
        for b in range(self.B):
            for x, y, name in zip(self.image(b), other.image(b), ("scores", "boxes", "class ids", "keep")):
                assert x.tobytes() == y.tobytes(), (what, name, b)


def check_decode(geo, snap, rows, thr, sbs):
    """Every (image, class) candidate list of the decode kernel, all 20 classes (FCOS class 19 included),
    against the oracle's thresholded set (see the module docstring)."""
    thr64 = float(F32(thr))
    lo, hi = thr64 - BAND * abs(thr64), thr64 + BAND * abs(thr64)
    bad = []
    for b in range(snap.B):
        conf, _, _, bg = sbs[b]
        if bg is None:
            sure_in, sure_out = np.ones(geo.N, bool), np.zeros(geo.N, bool)
        else:  # the background filter: dropped only if strictly greater than the best foreground probability
            best, bg64 = conf.max(axis=1).astype(np.float64), bg.astype(np.float64)
            sure_in, sure_out = bg64 < best * (1 - BAND), bg64 > best * (1 + BAND)
        for c in range(20):
            assert snap.cnt[b, c] <= snap.cap, (b, c, "list overflowed")
            _, r, sc = snap.list(b, c)
            assert len(r) == snap.cnt[b, c]
            assert r.min(initial=0) >= 0 and r.max(initial=0) < geo.N, (b, c, "row out of range")
            if len(np.unique(r)) != len(r):
                bad.append((b, c, "duplicate rows", len(r) - len(np.unique(r))))
            s = conf[:, c].astype(np.float64)
            got = np.zeros(geo.N, bool)
            got[r] = True
            missing = np.nonzero(sure_in & (s >= hi) & ~got)[0]
            extra = np.nonzero(got & (sure_out | (s < lo)))[0]
            if missing.size or extra.size:
                bad.append((b, c, "missing", missing[:5].tolist(), "extra", extra[:5].tolist()))
            np.testing.assert_allclose(sc, conf[r, c], rtol=1e-6, atol=0, err_msg="scores (%d, %d)" % (b, c))
    assert not bad, bad[:10]


def check_records(geo, snap, rows, thr, mb, iou, sbs, images=None):
    for b in range(snap.B) if images is None else images:
        assert snap.flags[b] == 0.0, (b, "overflow flag")
        s, bx, cid, kp = oracle_tail(geo, rows[b], thr, mb, iou, sb=sbs[b])
        gs, gb, gc, gk = snap.image(b)
        np.testing.assert_array_equal(gc, cid, err_msg="class ids, image %d" % b)
        np.testing.assert_array_equal(gk, kp, err_msg="NMS keep indices, image %d" % b)
        np.testing.assert_allclose(gs, s, rtol=1e-6, atol=0, err_msg="scores, image %d" % b)
        assert_boxes_close(gb, bx, what="boxes, image %d" % b)


def predict_paths(geo, snap, mb, iou, sbs):
    """{(b, c): path} from the GPU's own keys, and the pool counter it implies."""
    paths, counter = {}, 0
    for b in range(snap.B):
        for c in range(geo.nms_classes):
            bits, r, _ = snap.list(b, c)
            p = list_path(bits, r, sbs[b][1], mb, iou)
            paths[(b, c)] = p
            if p in ("dry", "full"):
                counter += len(r)
    return paths, counter


def check_all(geo, rows, thr, mb, iou, snap, expect=None):
    """Decode lists, records and the pool counter of one launch against the oracle; `expect`: {(b, c): path}
    the case was built to take."""
    sbs = [geo.scores_boxes(rows[b]) for b in range(snap.B)]
    check_decode(geo, snap, rows, thr, sbs)
    check_records(geo, snap, rows, thr, mb, iou, sbs)
    paths, counter = predict_paths(geo, snap, mb, iou, sbs)
    for k, v in (expect or {}).items():
        assert paths[k] == v, (k, paths[k], v)
    if snap.pool_entries:
        assert snap.counter == counter, ("pool counter", snap.counter, counter)
    return paths, counter


# ------------------------------------------------------- A. decode candidates --
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ssd", "retina", "yolo", "fcos"])
def test_decode_lists_match_oracle(built, kind):
    """The decode stage alone: each candidate exactly once, none missing or extra, scores to 1e-6 (B=5)."""
    geo = TAIL_GEOS[kind]
    thr, mb, iou = THR[kind]
    rows = make_rows(kind, geo.N, batch=5, seed=31)
    snap = Snap(harness(geo, rows, thr, mb, iou))
    check_all(geo, rows, thr, mb, iou, snap)


# --------------------------------------------------- B. decode iterations -----
GRID_CASES = {  # name -> (full-size network, B); B*N % 32 != 0 and N % 32 != 0 for all of them
    "retina800_b4": ("retina800", 4), "yolo416_b7": ("yolo416", 7), "fcos800_b6": ("fcos800", 6),
    "retina800_b1": ("retina800", 1)}


def decode_grid(B, N, per_sm=6):
    """odt_decode_candidates' grid restated: (groups of 32 rows, groups between two iterations of a warp)."""
    rows = B * N
    groups = (rows + 31) // 32
    blocks = min((groups + DECODE_WARPS - 1) // DECODE_WARPS, NUM_SMS * per_sm)
    return groups, blocks * DECODE_WARPS


def grid_facts(B, N, per_sm):
    """(iterations of warp 0, an image boundary inside a group on an iteration > 0, ragged last group)."""
    groups, step = decode_grid(B, N, per_sm)
    iters = (groups + step - 1) // step
    straddle = any((k * N) % 32 and (k * N) // 32 >= step for k in range(1, B))
    return iters, straddle, (B * N) % 32 != 0


@pytest.mark.parametrize("name", sorted(GRID_CASES))
def test_decode_grid_runs_several_iterations(name):
    """With ODT_DECODE_BLOCKS_PER_SM=1 every case gives a warp >= 3 iterations, a group that straddles two images
    on a later iteration (B > 1) and a ragged last group; RetinaNet-800 B=4 does so on the default grid too."""
    net, B = GRID_CASES[name]
    N = FULL[net][3]
    assert N % 32 and (B * N) % 32
    iters, straddle, ragged = grid_facts(B, N, 1)
    assert iters >= 3 and ragged and (straddle or B == 1), (iters, straddle, ragged)
    if name == "retina800_b4":
        assert grid_facts(B, N, 6) == (3, True, True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GRID_CASES))
def test_decode_configs_are_bit_identical_and_exact(built, monkeypatch, name):
    """ODT_DECODE_CFG in {3x2, 2x4} x ODT_DECODE_BLOCKS_PER_SM in {default, 1}: the sorted candidate keys and the
    records are bit-identical across the four, and equal to the oracle."""
    net, B = GRID_CASES[name]
    geo = full_size(net)
    thr, mb, iou = THR[geo.kind]
    rows = make_rows(geo.kind, geo.N, batch=B, seed=33)
    h = harness(geo, rows, thr, mb, iou)
    snaps = {}
    for cfg in ("3x2", "2x4"):
        for per_sm in (None, "1"):
            monkeypatch.setenv("ODT_DECODE_CFG", cfg)
            if per_sm is None:
                monkeypatch.delenv("ODT_DECODE_BLOCKS_PER_SM", raising=False)
            else:
                monkeypatch.setenv("ODT_DECODE_BLOCKS_PER_SM", per_sm)
            snaps[(cfg, per_sm)] = Snap(h)
    base = snaps[("3x2", None)]
    for k, s in snaps.items():
        base.assert_same(s, str(k))
    check_all(geo, rows, thr, mb, iou, base)


# --------------------------------------------------------- C. NMS list paths --
def _yolo48(rng, batch=1, cls=-30.0):
    """YOLO48 rows: every class logit `cls`, objectness 30 (sigmoid exactly 1.0, so a score is the class
    sigmoid), box deltas N(0, 0.5): boxes of 1-5 cells on the 48 x 48 grid."""
    rows = np.full((batch, YOLO48.N, 25), cls, F32)
    rows[..., 20:24] = rng.standard_normal((batch, YOLO48.N, 4)) * 0.5
    rows[..., 24] = 30.0
    return rows


def _huge(rows, idx):
    rows[..., idx, 22:24] = 7.0  # exp(7) = 1 097 cells high and wide: IoU > 0.9 among any two of them


def _list_lengths():
    """Lists of exactly 1 024 (shared memory, no prefilter) and 1 025 keys (prefilter subset)."""
    rng = np.random.default_rng(40)
    rows = _yolo48(rng, 2)
    for b, n in ((0, 1024), (1, 1025)):
        idx = rng.choice(YOLO48.N, n, replace=False)
        rows[b, idx, 0] = logit(rng.permutation(np.linspace(0.3, 0.95, n)))
    return dict(rows=rows, thr=0.2, mb=20, iou=0.45, expect={(0, 0): "smem", (1, 0): "subset"})


def _tied_bin():
    """Class 0: 300 huge boxes at distinct scores in [0.9, 0.99] (one survives), 200 moderate boxes tied at
    0.76 and 600 lower scores in [0.5, 0.7]: the select refines the [0.5, 1] bin and stops on the tied one,
    so the subset is the 500 best with every tie in it, and the kept boxes come from the ties, lowest row
    first.  Class 1: 380 distinct scores above 10 tied ones and 700 lower: a subset of 390, just above 384."""
    rng = np.random.default_rng(41)
    rows = _yolo48(rng)
    perm = rng.permutation(YOLO48.N)
    hi, tie, low = perm[:300], perm[300:500], perm[500:1100]
    _huge(rows, hi)
    rows[0, hi, 0] = logit(rng.permutation(np.linspace(0.9, 0.99, 300)))
    rows[0, tie, 0] = logit(0.76)
    rows[0, low, 0] = logit(rng.permutation(np.linspace(0.5, 0.7, 600)))
    perm = rng.permutation(YOLO48.N)
    rows[0, perm[:380], 1] = logit(rng.permutation(np.linspace(0.9, 0.99, 380)))
    rows[0, perm[380:390], 1] = logit(0.76)
    rows[0, perm[390:1090], 1] = logit(rng.permutation(np.linspace(0.5, 0.7, 700)))
    return dict(rows=rows, thr=0.2, mb=20, iou=0.45, expect={(0, 0): "subset", (0, 1): "subset"}, flip="tie",
                subset={(0, 0): 500, (0, 1): 390})


def _top_ties():
    """Class 0: 1 100 scores of exactly 1.0 (sigmoid(30)) and 300 lower: the select never resolves and the full
    list runs, ties kept lowest row first.  Class 1: exactly 1 024 keys at 1.0 and 300 below 0.5: the top bin
    alone fills the window (cum + h == 1 024), a subset of all 1 024 ties."""
    rng = np.random.default_rng(42)
    rows = _yolo48(rng)
    perm = rng.permutation(YOLO48.N)
    rows[0, perm[:1100], 0] = 30.0
    rows[0, perm[1100:1400], 0] = logit(rng.permutation(np.linspace(0.3, 0.45, 300)))
    perm = rng.permutation(YOLO48.N)
    rows[0, perm[:1024], 1] = 30.0
    rows[0, perm[1024:1324], 1] = logit(rng.permutation(np.linspace(0.3, 0.45, 300)))
    return dict(rows=rows, thr=0.2, mb=20, iou=0.45, expect={(0, 0): "full", (0, 1): "subset"}, flip="tie",
                subset={(0, 1): 1024})


def _dry_subsets():
    """score_thr = 0: every class lists all 6 912 rows.  Classes 0-2: 700 huge, mutually suppressing boxes
    hold the best scores, so their subsets yield one box and the full list runs; the other classes keep
    mb boxes inside their subsets."""
    rng = np.random.default_rng(43)
    rows = _yolo48(rng, 2)
    rows[..., :20] = rng.standard_normal((2, YOLO48.N, 20)) * 2.0
    rows[..., :3] = rng.standard_normal((2, YOLO48.N, 3)) * 0.5 - 4.0  # [0.5, 1]: huge boxes only
    for b in range(2):
        idx = rng.choice(YOLO48.N, 700, replace=False)
        _huge(rows[b], idx)
        for c in range(3):
            rows[b, idx, c] = rng.permutation(np.linspace(4.0, 8.0, 700)).astype(F32)
    expect = {(b, c): ("dry" if c < 3 else "subset") for b in range(2) for c in range(20)}
    return dict(rows=rows, thr=0.0, mb=25, iou=0.6, expect=expect)


PATH_CASES = {"list_1024_1025": _list_lengths, "tied_threshold_bin": _tied_bin, "top_ties": _top_ties,
              "dry_subsets": _dry_subsets}


@pytest.mark.parametrize("name", sorted(PATH_CASES))
def test_path_case_takes_its_path(name):
    """On the oracle's own lists the select restatement predicts the path each case was built for, and the
    subset sizes it claims; for the tie cases, the highest-row-first tie rule changes the keep list."""
    c = PATH_CASES[name]()
    geo, rows = YOLO48, c["rows"]
    for b in range(rows.shape[0]):
        sb = geo.scores_boxes(rows[b])
        lists = oracle_lists(geo, sb, c["thr"])
        for (bb, cc), want in c["expect"].items():
            if bb != b:
                continue
            bits, r = lists[cc]
            assert list_path(bits, r, sb[1], c["mb"], c["iou"]) == want, (bb, cc, want)
            if (bb, cc) in c.get("subset", {}):
                t = select_threshold(bits)
                assert (bits >= t).sum() == c["subset"][(bb, cc)], (bb, cc, int((bits >= t).sum()))
        if "flip" in c:
            ref = oracle_tail(geo, rows[b], c["thr"], c["mb"], c["iou"], sb=sb)
            assert not same_result(ref, oracle_tail(geo, rows[b], c["thr"], c["mb"], c["iou"], (c["flip"],), sb))


def test_select_restatement_edges():
    """The select restatement itself on hand-made lists."""
    one = np.float32(1.0).view(np.uint32)
    lowbits = np.linspace(0.1, 0.4, 300).astype(F32).view(np.uint32)
    assert select_threshold(np.full(1024, one)) is None
    assert select_threshold(np.concatenate([np.full(1025, one), lowbits])) == -1
    assert select_threshold(np.concatenate([np.full(1024, one), lowbits])) == 0x3F000000
    spread = np.linspace(0.01, 1.0, 5000).astype(F32).view(np.uint32)
    t = select_threshold(spread)
    assert SELECT_MIN <= (spread >= t).sum() <= SMEM_KEYS


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PATH_CASES))
def test_nms_path_matches_oracle(built, monkeypatch, name):
    """Each case on the GPU: the path predicted from the GPU's keys is the intended one, the pool counter is
    the summed length of the full-list lists, the records equal the oracle's; ODT_NMS_ADAPT=0 is bit-identical."""
    c = PATH_CASES[name]()
    geo, rows = YOLO48, c["rows"]
    h = harness(geo, rows, c["thr"], c["mb"], c["iou"])
    snap = Snap(h)
    check_all(geo, rows, c["thr"], c["mb"], c["iou"], snap, c["expect"])
    monkeypatch.setenv("ODT_NMS_ADAPT", "0")
    Snap(h).assert_same(snap, "ODT_NMS_ADAPT=0")


@pytest.mark.gpu
def test_dry_subsets_with_pool_present_partial_exhausted_and_absent(built, monkeypatch):
    """Six dry lists of 6 912 keys per launch: with the default pool every list caches its boxes; with room for
    2.5 lists some do and some re-decode; with room for less than one list all re-decode; without a pool the
    counter is untouched.  All records bit-identical (ODT_NMS_ADAPT=0 too) and equal to the oracle."""
    c = _dry_subsets()
    geo, rows = YOLO48, c["rows"]
    L = geo.N
    snaps = {}
    for pool in (None, 5 * L // 2, L - 1, 0):
        for adapt in (None, "0"):
            if adapt is None:
                monkeypatch.delenv("ODT_NMS_ADAPT", raising=False)
            else:
                monkeypatch.setenv("ODT_NMS_ADAPT", adapt)
            snaps[(pool, adapt)] = Snap(harness(geo, rows, c["thr"], c["mb"], c["iou"], pool_cap=pool))
    base = snaps[(None, None)]
    _, counter = check_all(geo, rows, c["thr"], c["mb"], c["iou"], base, c["expect"])
    assert counter == 6 * L and base.counter == counter and base.pool_entries >= counter
    for (pool, adapt), s in snaps.items():
        base.assert_same(s, "pool_cap=%s ODT_NMS_ADAPT=%s" % (pool, adapt))
        if pool == 0:
            assert s.pool_entries == 0 and s.counter == 0
        elif pool is not None:
            assert s.counter == counter and s.pool_entries == pool
    assert L <= 5 * L // 2 < counter  # the partial pool holds the first list to claim it, not all six


# ------------------------------------------------------------ D. exact edges --
def _iou_equal():
    """FCOS rows with l = r = t = b = 0 decode through exp(0) = 1 to 2 x 2-cell boxes; side-by-side
    neighbours have IoU exactly fl(1/3) = iou_thr, which does not suppress (strict >)."""
    rows = np.full((1, FCOS8.N, 25), -30.0, F32)
    rows[0, :, 20] = 30.0
    rows[0, :, 21:25] = 0.0
    for i, x in enumerate(range(1, 7)):
        rows[0, FCOS8.index(0, 3, x), 0] = 6.0 - i     # a row of cells, scores falling left to right
        rows[0, FCOS8.index(0, x, 5), 2] = 6.0 - i     # a column of cells
    return dict(geo=FCOS8, rows=rows, thr=0.5, mb=10, iou=float(F32(1 / 3)), flip="iou")


def _zero_area():
    """Regression logits of -100 give exp = 0 to fp32 precision: point boxes (all four) and a line box
    (left / right only), on cells off the zero grid lines.  Their IoU with anything is 0: all are kept, also
    inside a kept box, whereas the same rows with unit regressions suppress each other."""
    rows = np.full((1, FCOS8.N, 25), -30.0, F32)
    rows[0, :, 20] = 30.0
    rows[0, :, 21:25] = 0.0
    for i, (y, x) in enumerate([(5, 6), (5, 5), (5, 7), (4, 6), (2, 2), (2, 3)]):
        rows[0, FCOS8.index(0, y, x), 1] = 6.0 - i
    for y, x in [(5, 5), (5, 7), (2, 2), (2, 3)]:
        rows[0, FCOS8.index(0, y, x), 21:25] = -100.0
    rows[0, FCOS8.index(0, 4, 6), 21:23] = -100.0
    return dict(geo=FCOS8, rows=rows, thr=0.5, mb=10, iou=0.2, zero=[(5, 5), (5, 7), (2, 2), (2, 3), (4, 6)])


def _score_equal():
    """Saturated scores of exactly 1.0 (sigmoid(30) * sigmoid(30)) with score_thr = 1.0 pass (>=); scores one
    ulp below (sigmoid(16)) do not.  The same rows in classes 2 and 7 and in both images: ties everywhere."""
    geo = TAIL_GEOS["yolo"]
    rng = np.random.default_rng(50)
    rows = np.full((1, geo.N, 25), -30.0, F32)
    rows[0, :, 20:24] = rng.standard_normal((geo.N, 4)) * 0.5
    rows[0, :, 24] = 30.0
    perm = rng.permutation(geo.N)
    for c in (2, 7):
        rows[0, perm[:40], c] = 30.0
        rows[0, perm[40:80], c] = 16.0
    return dict(geo=geo, rows=np.concatenate([rows, rows]), thr=1.0, mb=10, iou=0.45, flip="score")


def _ssd_score_equal():
    """A softmax with one dominant logit (the others 100 below: exp = 0 to fp32 precision) is exactly 1.0 and
    passes score_thr = 1.0; a second logit 15 below the dominant one leaves it a few ulps under 1.0.  Rows of
    both kinds in classes 5 and 9: ties across classes.  Every other row is background."""
    geo = Geo("ssd", 300, [(19, 19, 4)])
    rng = np.random.default_rng(54)
    rows = np.full((1, geo.N, 25), -100.0, F32)
    rows[0, :, 21:] = rng.standard_normal((geo.N, 4)) * 0.5
    rows[0, :, 20] = 0.0
    perm = rng.permutation(geo.N)
    for c, r in ((5, perm[:80]), (9, perm[80:160])):
        rows[0, r, c] = 0.0
        rows[0, r, 20] = -100.0
        rows[0, r[40:], 12] = -15.0
    return dict(geo=geo, rows=rows, thr=1.0, mb=20, iou=0.5, flip="score")


def _bg_tie():
    """SSD rows whose background logit equals the best foreground logit have equal probabilities (exp(0) = 1
    for both): the row is kept (dropped only if background is strictly greater).  Rows with background one ulp
    above are dropped, rows with background below are kept."""
    geo = Geo("ssd", 300, [(19, 19, 4)])
    rng = np.random.default_rng(51)
    rows = np.full((1, geo.N, 25), -10.0, F32)
    rows[0, :, 21:] = rng.standard_normal((geo.N, 4)) * 0.5
    rows[0, :, 20] = 5.0
    perm = rng.permutation(geo.N)
    rows[0, perm[:90], 3] = 5.0
    rows[0, perm[30:60], 20] = np.nextafter(F32(5.0), F32(6.0))
    rows[0, perm[60:90], 20] = 4.5
    return dict(geo=geo, rows=rows, thr=0.3, mb=100, iou=0.5, flip="bg")  # mb: room for all 60 candidates


def _boundary_rows():
    """YOLO48, class 0 (class 1 and image 1 identical: ties across classes and images): 500 scores in
    [0.55, 0.99] form the prefilter subset (the [0.5, 1] bin), 530 in [0.25, 0.45] sit below it.  Subset ranks
    0 and 9-498 are huge boxes (one survives), ranks 1-8 and 499 small isolated ones, as is every box below
    the subset: greedy NMS keeps its 10th box on the subset's last key, so max_boxes is reached exactly at the
    boundary and the full list must not run."""
    rng = np.random.default_rng(52)
    rows = _yolo48(rng)
    # small: anchor 0 of every other cell, centred on the cell corner, exp(-30) = 0 -> the prior alone,
    # 1.25 x 1.625 cells, two cells apart (no overlap); huge: anchor 1 of any cell
    small = [int(i) for i in rng.permutation([YOLO48.index(0, y, x, 0) for y in range(0, 48, 2)
                                               for x in range(0, 48, 2)])]
    huge = [int(i) for i in rng.permutation([YOLO48.index(0, y, x, 1) for y in range(48) for x in range(48)])]
    sub_rows = [huge[0]] + small[:8] + huge[1:491] + [small[8]]
    low_rows = small[9:539]
    rows[0, small[:539], 20:22] = 0.0
    rows[0, small[:539], 22:24] = -30.0
    _huge(rows[0], huge[:491])
    for c in (0, 1):
        rows[0, sub_rows, c] = logit(np.linspace(0.99, 0.55, 500))
        rows[0, low_rows, c] = logit(np.linspace(0.45, 0.25, 530))
    return dict(geo=YOLO48, rows=np.concatenate([rows, rows]), thr=0.2, mb=10, iou=0.45, sub_rows=sub_rows,
                expect={(b, c): "subset" for b in range(2) for c in range(2)})


EDGE_CASES = {"iou_equals_threshold": _iou_equal, "zero_area_boxes": _zero_area,
              "score_equals_threshold": _score_equal, "ssd_score_equals_threshold": _ssd_score_equal,
              "ssd_background_tie": _bg_tie,
              "max_boxes_at_subset_boundary": _boundary_rows}


@pytest.mark.parametrize("name", sorted(EDGE_CASES))
def test_edge_case_is_on_the_edge(name):
    """The oracle sees each case exactly on its edge: taking the other side of the comparison changes its
    keep list (or, for zero-area boxes and the subset boundary, the property the case is built on holds)."""
    from oracle import tails as OT
    c = EDGE_CASES[name]()
    geo, rows = c["geo"], c["rows"]
    sb = geo.scores_boxes(rows[0])
    ref = oracle_tail(geo, rows[0], c["thr"], c["mb"], c["iou"], sb=sb)
    assert len(ref[3]) > 0
    if "flip" in c:
        other = oracle_tail(geo, rows[0], c["thr"], c["mb"], c["iou"], (c["flip"],), sb)
        assert not same_result(ref, other), name
    conf, boxes, valid, bg = sb
    if name == "iou_equals_threshold":
        k = [FCOS8.index(0, 3, x) for x in (1, 2)]
        assert OT._iou_py(boxes[k[0]], boxes[k[1]]) == F32(c["iou"])
        assert len(ref[3]) == 12
    if name == "zero_area_boxes":
        z = [FCOS8.index(0, y, x) for y, x in c["zero"]]
        area = (boxes[z, 2] - boxes[z, 0]) * (boxes[z, 3] - boxes[z, 1])
        assert np.all(area == 0) and set(z) <= set(ref[3].tolist())
        unit = rows[0].copy()
        unit[z, 21:25] = 0.0
        assert len(oracle_tail(geo, unit, c["thr"], c["mb"], c["iou"])[3]) < len(ref[3])
    if name == "score_equals_threshold":
        assert np.all((conf == 1.0).sum(axis=0)[[2, 7]] == 40) and np.all((conf >= 0.5).sum(axis=0)[[2, 7]] == 80)
        assert conf[conf < 1.0].max() < 1.0 and set(ref[2].tolist()) == {2, 7}
    if name == "ssd_score_equals_threshold":
        assert np.all((conf == 1.0).sum(axis=0)[[5, 9]] == 40) and np.all((conf >= 0.5).sum(axis=0)[[5, 9]] == 80)
        assert set(ref[2].tolist()) == {5, 9}
    if name == "ssd_background_tie":
        tie = valid & (bg == conf.max(axis=1))
        assert tie.sum() == 30 and np.isin(np.nonzero(tie)[0], ref[3]).any()
    if name == "max_boxes_at_subset_boundary":
        bits, r = oracle_lists(geo, sb, c["thr"])[0]
        t = select_threshold(bits)
        assert (bits >= t).sum() == 500 and list_path(bits, r, boxes, c["mb"], c["iou"]) == "subset"
        keep0 = ref[3][ref[2] == 0]
        assert len(keep0) == c["mb"] and keep0[-1] == c["sub_rows"][-1]
        # one key fewer in the subset and it runs dry
        sub = np.sort(r[bits >= t])
        sub = sub[sub != c["sub_rows"][-1]]
        assert len(OT.nms_c(boxes[sub], conf[sub, 0], c["mb"], c["iou"])) == c["mb"] - 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(EDGE_CASES))
def test_edge_case_matches_oracle(built, name):
    c = EDGE_CASES[name]()
    geo, rows = c["geo"], c["rows"]
    snap = Snap(harness(geo, rows, c["thr"], c["mb"], c["iou"]))
    check_all(geo, rows, c["thr"], c["mb"], c["iou"], snap, c.get("expect"))


def _overflow_rows():
    """SSD300, cap 64: image 0 has 20 candidates in each of classes 0-9; image 1 the same plus 100 in class 4."""
    geo = TAIL_GEOS["ssd"]
    rng = np.random.default_rng(53)
    rows = np.full((2, geo.N, 25), -10.0, F32)
    rows[..., 21:] = rng.standard_normal((2, geo.N, 4)) * 0.5
    rows[..., 20] = 5.0
    for b in range(2):
        for c in range(10):
            rows[b, rng.choice(geo.N, 20, replace=False), c] = rng.uniform(7.0, 9.0, 20)
    rows[1, rng.choice(geo.N, 100, replace=False), 4] = rng.uniform(7.0, 9.0, 100)
    return geo, rows


def test_overflow_case_overflows_one_image():
    geo, rows = _overflow_rows()
    for b, over in ((0, set()), (1, {4})):
        conf, _, valid, _ = geo.scores_boxes(rows[b])
        n = (valid[:, None] & (conf >= F32(0.5))).sum(axis=0)
        assert set(np.nonzero(n > 64)[0].tolist()) == over, (b, n)


@pytest.mark.gpu
def test_overflow_flags_only_the_overflowing_image(built):
    """The per-image flag of the packed record is [0, 1], run() raises, and image 0's record is exact."""
    import torch
    from odt_b200 import lib
    geo, rows = _overflow_rows()
    h = harness(geo, rows, 0.5, 20, 0.5, cap=64)
    h.tail.launch(h, torch.cuda.current_stream().cuda_stream)
    rec = h.tail.rec.cpu().numpy()
    D = h.tail.D
    np.testing.assert_array_equal(rec[:, D * 6 + 1], [0.0, 1.0])
    assert int(h.tail.status.cpu().numpy()[0]) != 0
    n = int(rec[0, D * 6])
    got = rec[0, :D * 6].reshape(D, 6)[:n]
    s, bx, cid, kp = oracle_tail(geo, rows[0], 0.5, 20, 0.5)
    np.testing.assert_array_equal(got[:, 5].astype(np.int32), cid)
    np.testing.assert_array_equal(h.tail.det_anchor.cpu().numpy()[0, :n], kp)
    np.testing.assert_allclose(got[:, 0], s, rtol=1e-6, atol=0)
    assert_boxes_close(got[:, 1:5], bx)
    with pytest.raises(lib.OdtError, match="overflow"):
        h.run()


# ------------------------------------------------------- E. full-size tails ---
FULL_CASES = {  # name -> (network, B, score threshold or ('q', fraction of N per class passing))
    "ssd300_b64": ("ssd300", 64, 0.30), "ssd512_b2": ("ssd512", 2, 0.30),
    "retina800_2pct": ("retina800", 2, ("q", 0.02)), "retina800_10pct": ("retina800", 2, ("q", 0.10)),
    "yolo416_b2": ("yolo416", 2, 0.45), "fcos1024_b2": ("fcos1024", 2, 0.40)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FULL_CASES))
def test_full_size_tail_matches_oracle_on_every_image(built, name):
    net, B, thr = FULL_CASES[name]
    geo = full_size(net)
    _, mb, iou = THR[geo.kind]
    rows = make_rows(geo.kind, geo.N, batch=B, seed=60)
    if isinstance(thr, tuple):  # the oracle quantile that passes this fraction of N per class on image 0
        conf, _, valid, _ = geo.scores_boxes(rows[0])
        thr = float(np.quantile(np.where(valid[:, None], conf, 0.0), 1.0 - thr[1]))
    snap = Snap(harness(geo, rows, thr, mb, iou))
    paths, _ = check_all(geo, rows, thr, mb, iou, snap)
    if name == "retina800_10pct":
        assert min(len(snap.keys[(b, c)]) for b in range(B) for c in range(20)) > SMEM_KEYS
        assert set(paths.values()) <= {"subset", "dry"}
