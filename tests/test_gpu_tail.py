"""GPU parity, stage (i): the decode + per-class NMS kernels fed known candidate
rows, against the committed golden fixtures and the live CPU oracle.  Bar:
class ids and NMS keep indices bit-exact; scores within 1 ulp-scale (1e-6 rel);
box coordinates within 1e-4 absolute (+1e-6 relative head-room for the 1-2 ulp
expf difference on out-of-image random-weight boxes)."""
import os

import numpy as np
import pytest

from helpers import assert_boxes_close, model_cfg

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _tail_for(name, case):
    from odt_b200 import nets
    kw = dict(nms_score_threshold=case["score_thr"], nms_max_boxes=case["max_boxes"],
              nms_iou_threshold=case["iou_thr"])
    if case["kind"] == "ssd":
        return nets.ssd_tail(case["size"], model_cfg("ssd", **kw))
    if case["kind"] == "retina":
        return nets.retina_tail(model_cfg("retinanet", data_shape=case["data_shape"], **kw))
    if case["kind"] == "yolo":
        return nets.yolo_tail(model_cfg("yolov3", **kw))
    return nets.fcos_tail(model_cfg("fcos", **kw))


def _check(res, keep, exp, near_ok=False):
    s, bx, cid, kp = exp
    np.testing.assert_array_equal(res[2], cid, err_msg="class ids")
    np.testing.assert_array_equal(keep, kp, err_msg="NMS keep indices")
    np.testing.assert_allclose(res[0], s, rtol=1e-6, atol=0)
    assert_boxes_close(res[1], bx)


@pytest.mark.parametrize("name", ["tail_ssd", "tail_retina", "tail_yolo", "tail_fcos"])
def test_tail_matches_committed_golden(built, name):
    from golden import make_golden as mg
    from odt_b200.engine import RowsHarness
    d = np.load(os.path.join(GOLD, name + ".npz"))
    case = mg.CASES[name]
    h = RowsHarness(_tail_for(name, case), case["levels"], d["rows"][None])
    res = h.run()[0]
    _check(res, h.keep_indices()[0], (d["scores"], d["bbox"], d["class_id"], d["keep"]))


@pytest.mark.parametrize("name", ["tail_ssd", "tail_retina", "tail_yolo", "tail_fcos"])
def test_tail_batch_matches_live_oracle(built, name):
    """B=5 (rows of one warp straddle images for the small cases), fresh seed."""
    from golden import make_golden as mg
    from odt_b200.engine import RowsHarness
    case = mg.CASES[name]
    rows = mg.make_rows(name, batch=5, seed=11)
    h = RowsHarness(_tail_for(name, case), case["levels"], rows)
    res, keep = h.run(), h.keep_indices()
    for b in range(5):
        _check(res[b], keep[b], mg.run_case(name, rows, image=b))
    # replays are bit-identical (atomics only reorder candidates before the sort)
    res2 = h.run()
    for b in range(5):
        for a, c in zip(res[b], res2[b]):
            np.testing.assert_array_equal(a, c)


def test_tail_empty_and_single(built):
    from golden import make_golden as mg
    from odt_b200.engine import RowsHarness
    case = dict(mg.CASES["tail_yolo"], score_thr=2.0)  # nothing can pass
    rows = mg.make_rows("tail_yolo", batch=2)
    res = RowsHarness(_tail_for("tail_yolo", case), case["levels"], rows).run()
    for r in res:
        assert r[0].shape == (0,) and r[1].shape == (0, 4) and r[2].shape == (0,)
        assert r[2].dtype == np.int32 and r[0].dtype == np.float32
    # exactly one candidate
    rows = np.full((1, 1575, 25), -20.0, np.float32)
    rows[0, 700, 3] = 9.0
    rows[0, 700, 24] = 9.0
    rows[0, :, 20:24] = 0.0
    case = dict(mg.CASES["tail_yolo"], score_thr=0.5)
    h = RowsHarness(_tail_for("tail_yolo", case), case["levels"], rows)
    res = h.run()[0]
    assert list(res[2]) == [3] and list(h.keep_indices()[0]) == [700]


def test_tail_prefilter_subset_on_lists_longer_than_smem(built):
    """6 912 random-score candidates per class (longer than the 1 024-entry shared-memory window): every list
    runs on its radix-select prefilter subset in shared memory, which yields max_boxes boxes, so no list takes
    the full-list path: the box-pool bump counter (int64 behind the per-image counters in `work`) stays 0."""
    from golden import make_golden as mg
    from odt_b200.engine import RowsHarness
    name = "tail_yolo"
    case = dict(mg.CASES[name], levels=[(48, 48, 3)], score_thr=0.0, max_boxes=25, iou_thr=0.6)
    mg.CASES["_spill"] = case
    try:
        rows = mg.make_rows("_spill", batch=2, seed=3)
        assert rows.shape[1] == 6912
        h = RowsHarness(_tail_for(name, case), case["levels"], rows)
        res, keep = h.run(), h.keep_indices()
        assert np.all(h.tail.cand_count.cpu().numpy() == 6912) and h.tail.box_pool is not None
        assert int(h.tail.work.cpu().numpy()[2:4].view(np.int64)[0]) == 0, "a list took the full-list path"
        for b in range(2):
            _check(res[b], keep[b], mg.run_case("_spill", rows, image=b))
    finally:
        del mg.CASES["_spill"]


def test_tail_prefilter_falls_back_when_subset_runs_dry(built):
    """Long lists run NMS on the top-scoring subset first (exact when nms_max_boxes boxes are kept inside
    it).  Here the ~700 best candidates of class 0 are huge, mutually suppressing boxes, so the subset
    yields one box and the kernel must redo the class on the full list."""
    from golden import make_golden as mg
    from odt_b200.engine import RowsHarness
    name = "tail_yolo"
    case = dict(mg.CASES[name], levels=[(48, 48, 3)], score_thr=0.0, max_boxes=25, iou_thr=0.6)
    mg.CASES["_dry"] = case
    try:
        rows = mg.make_rows("_dry", batch=2, seed=9)
        rng = np.random.default_rng(4)
        idx = rng.choice(rows.shape[1], 700, replace=False)
        for b in range(2):
            rows[b, idx, 0] = np.linspace(4.0, 8.0, 700, dtype=np.float32)[rng.permutation(700)]
            rows[b, idx, 24] = 8.0            # objectness
            rows[b, idx, 22:24] = 7.0         # exp(7) grid units high and wide: IoU among them > 0.8
        h = RowsHarness(_tail_for(name, case), case["levels"], rows)
        res, keep = h.run(), h.keep_indices()
        for b in range(2):
            exp = mg.run_case("_dry", rows, image=b)
            assert (exp[2] == 0).sum() == 25   # the oracle does reach max_boxes for class 0
            _check(res[b], keep[b], exp)
    finally:
        del mg.CASES["_dry"]


def test_tail_overflow_is_reported(built):
    from golden import make_golden as mg
    from odt_b200 import lib
    from odt_b200.engine import RowsHarness
    case = mg.CASES["tail_ssd"]
    tail = _tail_for("tail_ssd", case)
    tail.cap = 8
    h = RowsHarness(tail, case["levels"], mg.make_rows("tail_ssd"))
    with pytest.raises(lib.OdtError, match="overflow"):
        h.run()


def test_tail_full_size_properties(built):
    """BASELINE size (SSD300, B=64, N=8828): size-independent properties."""
    from golden import make_golden as mg
    from odt_b200.engine import RowsHarness
    from oracle.tails import _iou_py
    case = mg.CASES["tail_ssd"]
    rows = mg.make_rows("tail_ssd", batch=64, seed=5)
    h = RowsHarness(_tail_for("tail_ssd", case), case["levels"], rows)
    res = h.run()
    for b in range(64):
        s, bx, cid = res[b]
        assert np.all(np.diff(cid) >= 0), "class-major order"
        assert np.all(s >= np.float32(case["score_thr"]))
        for c in np.unique(cid):
            m = cid == c
            assert m.sum() <= case["max_boxes"]
            assert np.all(np.diff(s[m]) <= 0), "descending score inside a class"
        if b < 4:  # pairwise IoU of kept boxes never exceeds the threshold
            for c in np.unique(cid):
                bb = bx[cid == c]
                for i in range(len(bb)):
                    for j in range(i):
                        assert _iou_py(bb[i], bb[j]) <= np.float32(case["iou_thr"])
    exp = mg.run_case("tail_ssd", rows, image=63)
    _check(res[63], h.keep_indices()[63], exp)


@pytest.mark.parametrize("name,kind", [("loss_ssd", "ssd"), ("loss_retina", "retina"), ("loss_yolo", "yolo"),
                                       ("loss_fcos", "fcos")])
def test_loss_kernels_match_committed_golden(built, name, kind):
    """The four training-loss forward kernels on the committed seeded rows vs the frozen oracle values
    (2e-5 relative: float summation order)."""
    from golden import make_golden as mg
    from odt_b200.engine import RowsHarness
    d = np.load(os.path.join(GOLD, name + ".npz"))
    tail_name = mg.LOSS_CASES[name][0]
    case = mg.CASES[tail_name]
    h = RowsHarness(_tail_for(tail_name, case), case["levels"], d["rows"])
    got = h.loss(kind, d["gt"])
    for b in range(len(got)):
        assert abs(got[b] - d["loss"][b]) <= 2e-5 * max(abs(d["loss"][b]), 1.0), (name, b, got[b], d["loss"][b])
