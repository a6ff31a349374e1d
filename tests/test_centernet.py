"""CenterNet without a GPU: the constructor's checks, TF's variable names (the untaken shortcut branches included), the
oracle's tail and loss on known answers, the training executor against the oracle, the loss restatement against the
oracle and finite differences, one Adam step, the checkpoint rules and the C argument checks."""
import numpy as np
import pytest
import torch

F32 = np.float32


def cfg(**over):
    c = dict(mode="test", data_format="channels_last", num_classes=20, weight_decay=1e-4, keep_prob=0.5, batch_size=1,
             input_size=96, score_threshold=0.1, top_k_results_output=100, bn_init="trained", device="cpu")
    c.update(over)
    return c


def model(**over):
    import CenterNet
    return CenterNet.CenterNet(cfg(**over), None)


@pytest.mark.parametrize("key,bad", [("input_size", 100), ("input_size", 0), ("input_size", 96.0),
                                     ("num_classes", 0), ("num_classes", 129), ("num_classes", True),
                                     ("top_k_results_output", 0), ("top_k_results_output", 1025)])
def test_config_is_validated(key, bad):
    with pytest.raises(ValueError):
        model(**{key: bad})


def test_config_without_nms_keys():
    m = model(num_classes=1, top_k_results_output=1024, input_size=32)
    assert m.score_threshold == 0.1 and m.top_k_results_output == 1024 and m.data_shape == [32, 32, 3]
    assert not hasattr(m, "nms_score_threshold")


def _expected_names(nc):
    """A hand enumeration of CenterNet.py's variables in creation order."""
    names, n = [], {"backone": [0, 0], "upsampling": [0, 0, 0], "center_detector": [0, 0]}

    def un(scope, i, base):
        k = n[scope][i]
        n[scope][i] += 1
        return "%s/%s%s" % (scope, base, "" if k == 0 else "_%d" % k)

    def conv(scope, shape):
        vs, bs = un(scope, 0, "conv2d"), un(scope, 1, "batch_normalization")
        names.append((vs + "/kernel", shape))
        names.append((vs + "/bias", (shape[3],)))
        names.extend((bs + "/" + v, (shape[3],)) for v in ("gamma", "beta", "moving_mean", "moving_variance"))

    def dconv(cin, cout):
        vs, bs = un("upsampling", 2, "conv2d_transpose"), un("upsampling", 1, "batch_normalization")
        names.extend([(vs + "/kernel", (4, 4, cout, cin)), (vs + "/bias", (cout,))])
        names.extend((bs + "/" + v, (cout,)) for v in ("gamma", "beta", "moving_mean", "moving_variance"))

    def block(cin, f):  # conv, conv, then the 1x1 shortcut whether or not it is taken
        conv("backone", (3, 3, cin, f))
        conv("backone", (3, 3, f, f))
        conv("backone", (1, 1, cin, f))

    def dla(cin, f, levels):
        if levels == 1:
            block(cin, f)
            block(f, f)
        else:
            dla(cin, f, levels - 1)
            dla(f, f, levels - 1)
        conv("backone", (3, 3, f, f))

    conv("backone", (7, 7, 3, 16))
    conv("backone", (3, 3, 16, 16))
    conv("backone", (3, 3, 16, 32))
    dla(32, 64, 1)
    for cin, f, lv in ((64, 128, 2), (128, 256, 2), (256, 512, 1)):
        dla(cin, f, lv)
        conv("backone", (1, 1, cin, f))
    conv("upsampling", (1, 1, 512, 256))
    for _ in range(3):
        dconv(256, 256)
    conv("upsampling", (1, 1, 256, 256))
    conv("upsampling", (3, 3, 256, 256))
    dconv(256, 256)
    dconv(256, 256)
    conv("upsampling", (1, 1, 128, 256))
    conv("upsampling", (3, 3, 256, 256))
    dconv(256, 256)
    conv("upsampling", (3, 3, 256, 256))
    conv("upsampling", (1, 1, 256, 256))
    for c in (nc, 2, 2):
        conv("center_detector", (3, 3, 256, c))
    return names


@pytest.mark.parametrize("nc", [20, 3])
def test_variable_names_and_shapes(nc):
    v = model(num_classes=nc).variables()
    assert [(k, s) for k, (s, _) in v.items()] == _expected_names(nc)


def test_untaken_shortcuts_own_variables_but_run_nothing():
    """block2 of every generator takes the identity: its 1x1 shortcut is declared but no op reads its kernel, and the
    executor leaves its BN moving statistics alone."""
    from odt_b200 import engine as E
    m = model()
    net = m._build_spec()
    used = {op.kernel for op in net.ops if isinstance(op, E.ConvOp)}
    kernels = [k for k in net.vars if k.endswith("/kernel")]
    unused = [k for k in kernels if k not in used]
    # of the 2 + 4 + 4 + 2 blocks, only the first of each stage changes the channel count
    assert len(unused) == 1 + 3 + 3 + 1, unused
    assert all(k.startswith("backone/") and m.get_weights()[k].shape[:2] == (1, 1) for k in unused)
    tr = m.trainer()
    before = {k: v.clone() for k, v in tr.buffers.items()}
    stats = []
    tr.forward_rows(np.zeros((2, 96, 96, 3), F32), True, stats)
    touched = {s for s, _, _ in stats}
    for k in unused:
        bn = k.replace("conv2d", "batch_normalization").replace("/kernel", "")
        assert bn not in touched
        assert torch.equal(before[bn + "/moving_mean"], tr.buffers[bn + "/moving_mean"])


# --------------------------------------------------------------------------------------------------- oracle ----
def test_oracle_sigma_is_one_scalar():
    """tf.reduce_min over every GT and all three radii: the small box sets the heatmap width of the large one."""
    from oracle.centernet import centernet_image_loss, gaussian_radius
    big = [40.0, 40.0, 64.0, 64.0, 1]
    small = [200.0, 200.0, 8.0, 6.0, 2]
    rows = np.zeros((48 * 48, 24), F32)
    gt = np.array([big, small, [-1] * 5], F32)
    _, sigma = centernet_image_loss(rows, 48, 48, gt)
    want = min(min(r) for r in zip(*gaussian_radius(np.array([16.0, 2.0]), np.array([16.0, 1.5]))))
    assert sigma == pytest.approx(want)
    _, alone = centernet_image_loss(rows, 48, 48, np.array([big, [-1] * 5], F32))
    assert alone > 2 * sigma


def test_oracle_tail_plateaus_ties_and_threshold():
    from oracle.centernet import centernet_tail
    h, w = 6, 7
    rows = np.full((h * w, 6), -30.0, F32)
    rows[[8, 9, 15], 0] = 40.0         # a plateau of saturated sigmoids: every cell of it is a peak
    rows[30, 1] = 0.0                  # 0.5, tied with cell 33
    rows[33, 1] = 0.0
    rows[40, 1] = np.log(0.2 / 0.8)    # sigmoid 0.2: exactly at a 0.2 threshold -> dropped (strict)
    rows[:, 2:] = 0.25
    s, b, c, k = centernet_tail(rows, h, w, 0.2, 10)
    assert k.tolist() == [8, 9, 15, 30, 33] and c.tolist() == [0, 0, 0, 1, 1]
    assert s.tolist() == [1.0, 1.0, 1.0, 0.5, 0.5]
    assert b[0].tolist() == [(1 + 0.25 - 0.125) * 4, (1 + 0.25 - 0.125) * 4, (1 + 0.25 + 0.125) * 4,
                             (1 + 0.25 + 0.125) * 4]
    assert centernet_tail(rows, h, w, 0.2, 4)[3].tolist() == [8, 9, 15, 30]


# -------------------------------------------------------------------------------------------------- executor ----
@pytest.mark.parametrize("size", [96, 128])
def test_executor_matches_oracle(size):
    from oracle.centernet import centernet_heads, centernet_rows
    m = model(input_size=size)
    img = np.random.default_rng(size).integers(0, 256, (2, size, size, 3)).astype(F32)
    rows = m.trainer().forward_rows(img, False).detach().numpy()
    ref = centernet_rows(centernet_heads(m.get_weights(), img))
    assert rows.shape == ref.shape == (2, (size // 4) ** 2, 24)
    assert np.abs(rows - ref).max() <= 1e-5 * np.abs(ref).max()


# ------------------------------------------------------------------------------------------------------ loss ----
def loss_rows(n, nc, seed):
    r = np.random.default_rng(seed)
    rows = np.zeros((n, nc + 4), F32)
    rows[:, :nc] = r.standard_normal((n, nc)) * 2.0 - 2.0
    rows[:, nc:nc + 2] = r.uniform(0, 1, (n, 2))
    rows[:, nc + 2:] = r.uniform(0, 20, (n, 2))
    return rows


def loss_gt(rng, size, n, G, nc=20):
    gt = np.full((G, 5), -1.0, F32)
    for i in range(n):
        hh, ww = rng.uniform(2, size / 2, 2)
        gt[i] = [rng.uniform(0, size - 1), rng.uniform(0, size - 1), hh, ww, rng.integers(0, nc)]
    return gt


def loss_cases(nc=20, h=24, w=24):
    """(name, rows, gt): the edge cases the kernels and the restatement share."""
    rng = np.random.default_rng(5)
    rows = loss_rows(h * w, nc, 11)
    S = 4 * h
    two = np.array([[41.0, 41.0, 20.0, 16.0, 3], [42.5, 43.0, 10.0, 30.0, 3], [-1] * 5], F32)  # one cell, one class
    tiny = np.array([[50.3, 22.7, 1.5, 2.5, 0], [-1] * 5], F32)                              # smaller than a cell
    return [("regular", rows, loss_gt(rng, S, 6, 8, nc)), ("no boxes", rows, np.full((3, 5), -1.0, F32)),
            ("two GTs on one cell", rows, two), ("box smaller than a cell", rows, tiny),
            ("one class only", rows, np.array([[30.0, 60.0, 24.0, 12.0, 7], [-1] * 5], F32))]


def _trainer(h=24, nc=20):
    return model(input_size=4 * h, num_classes=nc).trainer()


@pytest.mark.parametrize("case", range(5))
def test_loss_restatement_matches_oracle(case):
    from oracle.centernet import centernet_image_loss
    name, rows, gt = loss_cases()[case]
    got = float(_trainer().image_loss(torch.from_numpy(rows), gt))
    want, _ = centernet_image_loss(rows, 24, 24, gt)
    assert abs(got - want) <= 2e-5 * max(abs(want), 1.0), (name, got, want)
    if name == "no boxes":
        assert got == 0.0


@pytest.mark.parametrize("case", [0, 2, 3])
def test_loss_restatement_gradient_by_finite_differences(case):
    name, rows, gt = loss_cases(nc=3, h=8, w=8)[case]
    gt = gt.copy()
    gt[:, :4] = np.where(gt[:, :4] >= 0, gt[:, :4] % 32, gt[:, :4])
    gt[:, 4] = np.where(gt[:, 4] >= 0, gt[:, 4] % 3, -1)
    tr = _trainer(h=8, nc=3)
    tr.dtype = torch.float64
    r = torch.from_numpy(rows.astype(np.float64)).requires_grad_(True)
    tr.image_loss(r, gt).backward()
    ana = r.grad.numpy()
    rng = np.random.default_rng(case)
    for _ in range(40):
        i, j = int(rng.integers(0, rows.shape[0])), int(rng.integers(0, 3))
        e = 1e-6
        rp, rm = rows.astype(np.float64), rows.astype(np.float64)
        rp[i, j] += e
        rm[i, j] -= e
        num = (float(tr.image_loss(torch.from_numpy(rp), gt)) - float(tr.image_loss(torch.from_numpy(rm), gt))) / (2 * e)
        assert abs(num - ana[i, j]) <= 1e-6 + 1e-5 * abs(num), (name, i, j, num, ana[i, j])


def test_adam_step_matches_the_formula():
    """Two steps of the trainer against TF's Adam written out, for one kernel, one BN beta and one untaken shortcut
    kernel (moved by the decay term alone)."""
    m = model(input_size=32, mode="test")
    tr = m.trainer()
    names = ["backone/conv2d_1/kernel", "backone/batch_normalization_3/beta", "backone/conv2d_8/kernel"]
    w0 = {k: tr.params[k].detach().clone().double() for k in names}
    mm = {k: torch.zeros_like(w0[k]) for k in names}
    vv = {k: torch.zeros_like(w0[k]) for k in names}
    img = np.random.default_rng(1).integers(0, 256, (2, 32, 32, 3)).astype(F32)
    gt = np.array([[[10.0, 12.0, 8.0, 9.0, 2], [-1] * 5]] * 2, F32)
    b1p, b2p = 0.9, 0.999
    for step, lr in ((1, 1e-3), (2, 5e-4)):
        rows = tr.forward_rows(img, True, [])
        loss, _ = tr.total_loss(rows, gt)
        g = torch.autograd.grad(loss, [tr.params[k] for k in names])
        tr.step(img, gt, lr)
        lr_t = lr * (1 - b2p) ** 0.5 / (1 - b1p)
        for k, gk in zip(names, g):
            mm[k] = 0.9 * mm[k] + 0.1 * gk.double()
            vv[k] = 0.999 * vv[k] + 0.001 * gk.double() ** 2
            w0[k] = w0[k] - lr_t * mm[k] / (vv[k].sqrt() + 1e-8)
            assert torch.allclose(tr.params[k].double(), w0[k], rtol=1e-5, atol=1e-7), (step, k)
        b1p, b2p = b1p * 0.9, b2p * 0.999
    assert tr.global_step == 2 and tr.beta1_power == pytest.approx(0.9 ** 3)
    unused = tr.params["backone/conv2d_8/kernel"]
    assert "backone/conv2d_8/kernel/Adam_1" in tr.slots and unused.shape[:2] == (1, 1)


# ------------------------------------------------------------------------------------------------ checkpoints ----
def test_checkpoint_rules(tmp_path):
    from odt_b200 import tf_checkpoint
    m = model()
    path = m.save_weight("latest", str(tmp_path / "ck" / "test"))
    m2 = model()
    m2.set_weights({k: v * 0 for k, v in m.get_weights().items()})
    m2.load_weight(path)
    assert all(np.array_equal(m2.get_weights()[k], v) for k, v in m.get_weights().items())
    with pytest.raises(tf_checkpoint.CheckpointError):
        model(num_classes=3).load_weight(path)  # another class count: the keypoint conv has another shape
    w = dict(m.get_weights())
    w.pop("backone/conv2d_8/kernel")  # an untaken shortcut's kernel is part of the checkpoint too
    partial = str(tmp_path / "partial-0")
    tf_checkpoint.write_checkpoint(partial, w)
    m3 = model()
    before = dict(m3.get_weights())
    with pytest.raises(tf_checkpoint.CheckpointError):
        m3.load_weight(partial)
    assert all(np.array_equal(m3.get_weights()[k], v) for k, v in before.items())


def test_pretrained_weight_restores_backone_trainables_only(tmp_path):
    from odt_b200 import tf_checkpoint
    src = model()
    w = src.get_weights()
    back = {k: v + 1 for k, v in w.items() if k.startswith("backone/") and "moving" not in k}
    path = str(tmp_path / "pre-0")
    tf_checkpoint.write_checkpoint(path, back)
    m = model()
    m.set_weights({k: v.copy() for k, v in w.items()})
    m.load_pretrained_weight(path)
    got = m.get_weights()
    for k, v in w.items():
        assert np.array_equal(got[k], back[k] if k in back else v), k
    back.pop(next(iter(back)))
    tf_checkpoint.write_checkpoint(path, back)
    with pytest.raises(tf_checkpoint.CheckpointError):
        model().load_pretrained_weight(path)


# --------------------------------------------------------------------------------------------- C argument checks ----
def test_c_argument_checks(built):
    """The entry points refuse bad parameters before any launch (no device needed to reach the checks)."""
    import ctypes as C
    from odt_b200 import lib as L
    from odt_b200.nets import centernet_tail
    lib = L.load()
    tail = centernet_tail(cfg())
    p = tail.params([(24, 24, 1)])
    assert lib.odt_peak_topk_scratch_bytes(C.byref(p), 2) == 2 * 576 * 16
    per_image = lib.odt_centernet_loss_scratch_bytes(C.byref(p), 1)  # 3 partial pairs + the GT summary
    assert per_image > 3 * 16 and per_image % 8 == 0
    assert lib.odt_centernet_loss_scratch_bytes(C.byref(p), 2) == 2 * per_image
    dummy = C.c_void_p(256)
    assert lib.odt_peak_topk(dummy, C.byref(p), 0, dummy, dummy, 602, None, None) == -1        # B
    assert lib.odt_peak_topk(dummy, C.byref(p), 1, dummy, dummy, 601, None, None) == -1        # rec_ld < 6K + 2
    for field, val in (("kind", 0), ("num_fg", 129), ("N", 575), ("max_boxes", 1025), ("max_boxes", 0)):
        q = tail.params([(24, 24, 1)])
        setattr(q, field, val)
        assert lib.odt_peak_topk(dummy, C.byref(q), 1, dummy, dummy, 6 * 1025 + 2, None, None) == -1, field
    assert lib.odt_centernet_loss_fwd(dummy, C.byref(p), 1, dummy, 129, dummy, dummy, None) == -1    # G > 128
    assert lib.odt_centernet_loss_fwd(dummy, C.byref(p), 1, dummy, 0, dummy, dummy, None) == -1      # G = 0
    assert lib.odt_centernet_loss_grad(dummy, C.byref(p), 1, dummy, 4, dummy, dummy, None, None) == -1
    assert lib.odt_dla_join(dummy, dummy, dummy, 1, 1, 4, 4, 8, 8, 8, 4, 1, None) == -1         # out_ld < C
    assert lib.odt_dla_join(dummy, dummy, dummy, 1, 1, 4, 4, 8, 8, 8, 8, 2, None) == -1         # pooled
