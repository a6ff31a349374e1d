"""CPU suite, part 2: host logic and the C-ABI surface (no GPU compute)."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from helpers import model_cfg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(built):
    from odt_b200 import lib
    hdr = open(os.path.join(ROOT, "include", "odt_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(odt_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    so = ctypes.CDLL(lib.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(so, name), "symbol %s declared in include/odt_b200.h is not exported" % name
    assert declared == set(lib.SYMBOLS), declared ^ set(lib.SYMBOLS)
    L = lib.load()
    assert L.odt_abi_version() == 5


def test_same_pad_abi_matches_host_and_oracle(built):
    from odt_b200 import lib
    from odt_b200.engine import same_pad
    from oracle import tfops
    for size, k, s, d in [(19, 3, 2, 1), (10, 3, 2, 1), (800, 7, 2, 1), (75, 2, 2, 1), (19, 3, 1, 2),
                          (416, 3, 2, 1), (300, 3, 1, 1), (5, 1, 1, 1)]:
        assert lib.same_pad(size, k, s, d) == same_pad(size, k, s, d) == tfops.same_pad(size, k, s, d)


def test_abi_rejects_bad_arguments_without_gpu(built):
    from odt_b200 import lib
    L = lib.load()
    p = lib.ConvParams()
    assert L.odt_conv2d_f16_tc(None, None, ctypes.byref(p), None) == -1
    assert b"invalid argument" in L.odt_last_error()
    t = lib.TailParams()
    assert L.odt_decode_candidates(None, ctypes.byref(t), 1, None, None, None) == -1


def test_missing_extension_fails_loudly(tmp_path, monkeypatch):
    from odt_b200 import lib
    monkeypatch.setattr(lib, "LIB_PATH", str(tmp_path / "nope.so"))
    monkeypatch.setattr(lib, "_lib", None)
    with pytest.raises(lib.OdtError, match="no CPU fallback"):
        lib.load()


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "object-detection-tensorflow_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), f
    for f in ("SSD300.py", "SSD512.py", "RetinaNet.py", "YOLOv3.py", "FCOS.py"):
        assert "oracle" not in open(os.path.join(ROOT, f)).read()


@pytest.mark.parametrize("mod,cls,kind,nvars", [
    ("SSD300", "SSD300", "ssd", 123), ("SSD512", "SSD512", "ssd", 141),
    ("RetinaNet", "RetinaNet", "retinanet", 732), ("YOLOv3", "YOLOv3", "yolov3", 450),
    ("FCOS", "FCOS", "fcos", 344)])
def test_model_surface_and_variable_names(mod, cls, kind, nvars):
    """Reference module/class/ctor/method names (SURVEY 8b) and TF1 variable naming (App. D)."""
    m = getattr(__import__(mod), cls)(model_cfg(kind), None)
    for meth in ("test_one_image", "train_one_epoch", "save_weight", "load_weight"):
        assert callable(getattr(m, meth))
    v = m.variables()
    assert len(v) == nvars
    names = list(v)
    if kind == "ssd":
        assert "feature_extractor/kenrel_conv2_1" in v and "feature_extractor/bias_conv_3_1" in v
        assert v["feature_extractor/conv6/kernel"][0] == (3, 3, 512, 1024)
        assert v["regressor/pred1/kernel"][0] == (3, 3, 512, 100)
        assert "feature_extractor/l2_norm_factor" in v
    if kind == "retinanet":
        assert v["feature_extractor/conv2d/kernel"][0] == (7, 7, 3, 16)
        # widths 7*2^i quirk and 3x3 shortcut
        assert v["feature_extractor/block1_unit1/conv_branch/conv2d/kernel"][0] == (1, 1, 16, 7)
        assert v["feature_extractor/block1_unit1/identity_branch/conv2d/kernel"][0] == (3, 3, 16, 28)
        assert v["regressor/conv2d_4/kernel"][0] == (3, 3, 256, 189)
        assert v["regressor/conv2d_9/kernel"][0] == (3, 3, 256, 36)
        assert "regressor/conv2d_49/kernel" in v and "regressor/conv2d_50/kernel" not in v
    if kind == "yolov3":
        assert v["backone/conv2d/kernel"][0] == (3, 3, 3, 32)
        assert v["head/pyd2/conv2d/kernel"][0] == (1, 1, 512, 256)      # lateral on the top-down
        assert v["head/pyd2/conv2d_1/kernel"][0] == (1, 1, 768, 128)    # after concat
        assert v["head/pyd1/conv2d_6/kernel"][0] == (1, 1, 1024, 75)
    if kind == "fcos":
        assert v["head/classifier_head/conv2d_4/kernel"][0] == (3, 3, 256, 20)
        assert v["head/classifier_head/conv2d_5/kernel"][0] == (3, 3, 256, 1)
        assert v["head/regress_head/conv2d_4/kernel"][0] == (3, 3, 256, 4)
        assert "backone/GroupNorm/gamma" in v
    assert len(set(names)) == len(names)


def test_config_validation_matches_reference():
    import SSD300
    with pytest.raises(AssertionError):
        SSD300.SSD300(model_cfg("ssd", mode="infer"), None)
    with pytest.raises(AssertionError):
        SSD300.SSD300(model_cfg("ssd", data_format="NHWC"), None)
    c = model_cfg("ssd")
    del c["nms_max_boxes"]
    with pytest.raises(KeyError):
        SSD300.SSD300(c, None)


def test_reference_driver_preamble_runs_unchanged(tmp_path):
    """The import block + get_generator + ctor sequence of testSSD300.py:1-60
    (rewritten, not copied) must work against the drop-in modules."""
    (tmp_path / "data").mkdir()
    code = """
from __future__ import absolute_import, division, print_function
from utils import tfrecord_voc_utils as voc_utils
import tensorflow as tf
import numpy as np
import SSD300 as net
import os
from utils.voc_classname_encoder import classname_to_ids
config = {'mode': 'train', 'data_format': 'channels_last', 'num_classes': 20, 'weight_decay': 1e-4,
          'keep_prob': 0.5, 'batch_size': 32, 'nms_score_threshold': 0.5, 'nms_max_boxes': 20,
          'nms_iou_threshold': 0.5, 'pretraining_weight': os.path.join('.', 'vgg_16.ckpt')}
data = [os.path.join('./data/', n) for n in os.listdir('./data/')]
gen = voc_utils.get_generator(data, 32, 1024, {'output_shape': [300, 300]})
provider = {'data_shape': [300, 300, 3], 'num_train': 5000, 'num_val': 0, 'train_generator': gen,
            'val_generator': None}
m = net.SSD300(config, provider)
assert m.batch_size == 32 and m.num_classes == 21 and classname_to_ids['tvmonitor'] == 19
print('ok')
"""
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr
    # like NewCheckpointReader (SSD300.py:31), a missing ./vgg_16.ckpt is an error when the weights are needed,
    # unless the random-init opt-in of BASELINE config 0 is given
    code2 = code.replace("print('ok')", "m.get_weights(); print('ok')")
    r = subprocess.run([sys.executable, "-c", code2], cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=120)
    assert r.returncode != 0 and "FileNotFoundError" in r.stderr
    r = subprocess.run([sys.executable, "-c", code2], cwd=str(tmp_path), env=dict(env, ODT_ALLOW_RANDOM_INIT="1"),
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr


def test_other_class_counts_are_rejected():
    """25-float candidate rows: only 20 foreground classes (ADVICE r1)."""
    import RetinaNet
    import SSD300
    with pytest.raises(ValueError):
        SSD300.SSD300(model_cfg("ssd", num_classes=80), None)
    with pytest.raises(ValueError):
        RetinaNet.RetinaNet(model_cfg("retinanet", num_classes=10), None)


def test_init_weights_deterministic_and_layouts():
    import YOLOv3
    from odt_b200.engine import init_weights
    v = YOLOv3.YOLOv3(model_cfg("yolov3"), None).variables()
    a, b = init_weights(v, 1, "trained"), init_weights(v, 1, "trained")
    assert all(np.array_equal(a[k], b[k]) for k in a)
    assert a["backone/conv2d/kernel"].shape == (3, 3, 3, 32)  # HWIO
    c = init_weights(v, 2, "trained")
    assert not np.array_equal(a["backone/block1/conv2d/kernel"], c["backone/block1/conv2d/kernel"])


def test_fusion_plan_retinanet():
    """BN+ReLU pre-activations fold into producer epilogues; tower raw outputs vanish."""
    import RetinaNet
    from odt_b200 import engine as E
    m = RetinaNet.RetinaNet(model_cfg("retinanet"), None)
    E.Net.spec_only = True
    try:
        net, _ = m._build(1, "fp16", True)
    finally:
        E.Net.spec_only = False
    n_aff = sum(isinstance(o, E.AffineActOp) for o in net.ops)
    net.fuse()
    n_aff2 = sum(isinstance(o, E.AffineActOp) for o in net.ops)
    fused = sum((o.pre is not None) + (getattr(o, "pre2", None) is not None)
                for o in net.ops if isinstance(o, (E.ConvOp, E.UpsampleAddOp, E.PoolOp)))
    assert n_aff == 122 - 1  # every conv but the stem is pre-activated
    assert fused + n_aff2 == n_aff and n_aff2 <= 6  # only third consumers of one tensor stay stand-alone
    pool = [o for o in net.ops if isinstance(o, E.PoolOp)][0]
    assert pool.pre is not None and pool.pre2 is not None and not pool.y.needed  # pooled stem: both BNs fused, raw dropped
    dropped = sum(1 for t in net.acts if not t.needed)
    assert dropped >= 40  # the 4x2x5 tower intermediates at least


@pytest.mark.parametrize("model,min_lanes", [("ssd300", 2), ("retinanet", 4), ("yolov3", 2), ("fcos", 4)])
def test_lane_plan_respects_dataflow(model, min_lanes):
    """Multi-stream capture plan: every producer is either earlier on the same lane or
    waited on through an event; independent heads / pyramid levels get their own lanes."""
    import importlib
    from odt_b200 import engine as E
    mod = {"ssd300": "SSD300", "retinanet": "RetinaNet", "yolov3": "YOLOv3", "fcos": "FCOS"}[model]
    m = getattr(importlib.import_module(mod), mod)(model_cfg(model), None)
    E.Net.spec_only = True
    try:
        net, _ = m._build(1, "fp16", True)
    finally:
        E.Net.spec_only = False
    net.fuse()
    lane_of, waits, tails = net.plan_lanes(8)
    assert len(lane_of) == len(net.ops) and max(lane_of) < 8 and lane_of[0] == 0
    assert len(tails) >= min_lanes
    producer = {}
    for i, op in enumerate(net.ops):
        for t in op.reads:
            p = producer.get(id(t))
            if p is None:
                continue
            assert p < i
            assert lane_of[p] == lane_of[i] or p in waits[i]
        for w in waits[i]:
            assert w < i and lane_of[w] != lane_of[i]
        outs = list(op.writes) + [pr[2] for pr in (getattr(op, "pre", None), getattr(op, "pre2", None)) if pr]
        for t in outs:
            producer[id(t)] = i
    one, w1, t1 = net.plan_lanes(1)
    assert set(one) == {0} and not any(w1)


def _gloo_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from odt_b200 import dist as od
    lo, hi = od.shard_range(8, rank, world)
    D = 5
    dets = torch.zeros((hi - lo, D, 6))
    cnt = torch.zeros((hi - lo,), dtype=torch.int32)
    for i, g in enumerate(range(lo, hi)):
        k = g % (D + 1)
        cnt[i] = k
        dets[i, :k, 0] = g + 0.5
        dets[i, :k, 5] = g
    # the packed record the NMS kernel writes: [B, D*6 + 2] = D rows, then (count, overflow flag)
    local = torch.zeros((hi - lo, D * 6 + 2))
    local[:, :D * 6] = dets.reshape(hi - lo, -1)
    local[:, D * 6] = cnt.to(torch.float32)
    rec = od.gather_records(local)
    from odt_b200.engine import unpack_records
    out = unpack_records(rec.numpy())
    assert len(out) == 8 and len(out[-1]) == 3 and len(out[0:2]) == 2
    pre = torch.empty((world * (hi - lo), D * 6 + 2))
    assert od.gather_records(local, out=pre) is pre and torch.equal(pre, rec)
    flagged = rec.clone()
    flagged[3, -1] = 1.0             # an image whose candidate list overflowed must not pass silently
    try:
        unpack_records(flagged.numpy())
        raise AssertionError("overflow flag ignored")
    except RuntimeError:
        pass
    w = od.broadcast_weights({"a": np.full((3,), rank + 1.0, np.float32)})
    q.put((rank, [(len(s), float(s[0]) if len(s) else -1.0, int(c[0]) if len(c) else -1)
                  for s, _, c in out], float(w["a"][0])))
    dist.destroy_process_group()


def test_sharded_gather_world2_gloo():
    """N>1 path on CPU: contiguous image shards + ONE all-gather of packed records."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + os.getpid() % 300
    ps = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = [q.get(timeout=120) for _ in ps]
    for p in ps:
        p.join(60)
    for rank, out, w0 in res:
        assert w0 == 1.0  # rank 0's weights everywhere
        assert len(out) == 8
        for g, (k, s0, c0) in enumerate(out):
            assert k == g % 6
            if k:
                assert s0 == g + 0.5 and c0 == g


def test_lane_plan_on_random_dags():
    """plan_lanes on synthetic op graphs: dependencies are honoured for any lane budget."""
    hyp = pytest.importorskip("hypothesis")
    from hypothesis import given, settings, strategies as st
    from odt_b200 import engine as E

    class _T:
        pass

    class _Op:
        def __init__(self, reads, writes):
            self.reads, self.writes = tuple(reads), tuple(writes)

    @settings(max_examples=80, deadline=None)
    @given(st.lists(st.lists(st.integers(0, 10 ** 6), max_size=3), min_size=1, max_size=40), st.integers(1, 6))
    def run(spec, lanes):
        tensors, ops = [], []
        for picks in spec:
            reads = [tensors[p % len(tensors)] for p in picks] if tensors else []
            out = _T()
            tensors.append(out)
            ops.append(_Op(reads, [out]))
        net = E.Net.__new__(E.Net)
        net.ops = ops
        lane_of, waits, tails = E.Net.plan_lanes(net, lanes)
        assert len(lane_of) == len(ops) and max(lane_of) < lanes and len(tails) <= lanes
        producer = {}
        for i, op in enumerate(ops):
            for t in op.reads:
                p = producer[id(t)]
                assert p < i and (lane_of[p] == lane_of[i] or p in waits[i])
            producer[id(op.writes[0])] = i
    run()
