"""The loss-gradient entry points (csrc/loss.cu, odt_<family>_loss_grad) without a GPU: the gradient they restate --
the training step's autograd loss -- against central finite differences, their host-side argument checks, and the
ground-truth trimming of the training step's GPU path."""
import ctypes

import numpy as np
import pytest
import torch

import loss_grad_ref as LR

F32 = np.float32


# ----------------------------------------------------------------- finite differences --
def _fd_check(tr, row, g, n_pick=24, seed=0, eps=1e-6):
    """Central differences on the float64 rows at entries with a gradient and at a few without one."""
    loss, gr = LR.grad(tr, row, g)
    assert np.isfinite(loss) and np.isfinite(gr).all()
    r64 = np.asarray(row, np.float64)
    nz = np.argwhere(np.abs(gr) > 1e-9)
    z = np.argwhere(gr == 0)
    assert len(nz) > 20
    rng = np.random.default_rng(seed)
    pick = [tuple(i) for i in nz[rng.choice(len(nz), min(n_pick, len(nz)), replace=False)]]
    pick += [tuple(i) for i in z[rng.choice(len(z), min(6, len(z)), replace=False)]] if len(z) else []
    scale = np.abs(gr).max()
    for i, j in pick:
        rp, rm = r64.copy(), r64.copy()
        rp[i, j] += eps
        rm[i, j] -= eps
        fd = (float(tr.image_loss(torch.from_numpy(rp), g)) - float(tr.image_loss(torch.from_numpy(rm), g))) / (2 * eps)
        assert abs(fd - gr[i, j]) <= 1e-6 * scale + 1e-4 * abs(fd), (i, j, fd, gr[i, j])


def test_retina_gradient_matches_finite_differences():
    levels, size = [(8, 8, 9)], 64
    cfg = LR.config("retina", size)
    tr = LR.restatement("retina", levels, cfg, size)
    row = LR.rows("retina", 8 * 8 * 9, seed=3)[0]
    g = LR.gt(np.random.default_rng(4), 3, size, 6, lo=0.3, hi=0.7)
    _fd_check(tr, row, g)


@pytest.mark.parametrize("A", [1, 3, 9])
@pytest.mark.parametrize("nc", [1, 80])
def test_yolo_gradient_matches_finite_differences(A, nc):
    levels, size = [(5, 5, A), (10, 10, A), (20, 20, A)], 160
    cfg = LR.config("yolo", size, nc=nc, A=A, coord_scale=2, noobj_scale=0.5, obj_scale=5, class_scale=1.5)
    tr = LR.restatement("yolo", levels, cfg, size, nc=nc)
    row = LR.rows("yolo", sum(h * w * a for h, w, a in levels), nc=nc, seed=A + nc)[0]
    g = LR.gt(np.random.default_rng(A * nc), 4, size, 6, nc=nc)
    _fd_check(tr, row, g, seed=A)


@pytest.mark.parametrize("nc", [1, 80])
def test_fcos_gradient_matches_finite_differences(nc):
    levels, size = [(16, 16, 1), (8, 8, 1), (4, 4, 1), (2, 2, 1), (1, 1, 1)], 128
    cfg = LR.config("fcos", size, nc=nc)
    tr = LR.restatement("fcos", levels, cfg, size, nc=nc)
    row = LR.rows("fcos", sum(h * w for h, w, _ in levels), nc=nc, seed=nc)[0]
    g = np.array([[40, 50, 30, 40, 0], [70, 60, 90, 70, nc - 1], [64, 64, 200, 180, nc // 2], [-1] * 5], F32)
    _fd_check(tr, row, g)


# -------------------------------------------------------------------- C ABI checks --
GRAD_SYMBOLS = ("odt_retina_loss_grad", "odt_ssd_loss_grad", "odt_fcos_loss_grad", "odt_yolo_loss_grad")


def test_grad_symbols_are_exported(built):
    from odt_b200 import lib
    so = ctypes.CDLL(lib.LIB_PATH)
    for name in GRAD_SYMBOLS:
        assert hasattr(so, name) and name in lib.SYMBOLS


def _params(kind, nc=20, A=3):
    size = {"ssd": 300, "retina": 64, "yolo": 160, "fcos": 128}[kind]
    levels = {"ssd": [(3, 3, 4)], "retina": [(8, 8, 9)], "yolo": [(5, 5, A), (10, 10, A), (20, 20, A)],
              "fcos": [(16, 16, 1), (8, 8, 1), (4, 4, 1), (2, 2, 1), (1, 1, 1)]}[kind]
    return LR.tail(kind, size, LR.config(kind, size, nc=nc, A=A)).params(levels)


def _call(L, kind, p, G=4, null=None):
    """One gradient call with fake (never dereferenced) device pointers; `null` names the pointer to pass as NULL."""
    fake = ctypes.c_void_p(64)
    ptr = {k: (None if k == null else fake) for k in ("head", "gt", "scratch", "loss", "grad")}
    pre = (ptr["head"], ctypes.byref(p), 2, ptr["gt"], G)
    if kind == "retina":
        return L.odt_retina_loss_grad(*pre, 0.25, 2.0, ptr["scratch"], ptr["loss"], ptr["grad"], None)
    if kind == "ssd":
        return L.odt_ssd_loss_grad(*pre, ptr["scratch"], ptr["loss"], None, ptr["grad"], None)
    if kind == "fcos":
        return L.odt_fcos_loss_grad(*pre, ptr["scratch"], ptr["loss"], ptr["grad"], None)
    return L.odt_yolo_loss_grad(*pre, 1.0, 1.0, 5.0, 1.0, ptr["scratch"], ptr["loss"], ptr["grad"], None)


@pytest.mark.parametrize("kind", ["retina", "ssd", "fcos", "yolo"])
def test_grad_entry_points_reject_bad_arguments_without_gpu(built, kind):
    """Null pointers (the gradient among them), a head of another kind, G = 129 and class counts out of range are
    the argument error, decided on the host before any CUDA call."""
    from odt_b200 import lib
    L = lib.load()

    def rejected(rc):
        return rc == -1 and b"invalid argument" in L.odt_last_error()

    for null in ("head", "gt", "scratch", "loss", "grad"):
        assert rejected(_call(L, kind, _params(kind), null=null)), null
    p = _params(kind)
    p.kind = lib.DECODE_FCOS if kind != "fcos" else lib.DECODE_YOLO3
    assert rejected(_call(L, kind, p))
    assert rejected(_call(L, kind, _params(kind), G=129)) and b"G <= 128" in L.odt_last_error()
    assert rejected(_call(L, kind, _params(kind), G=0))
    for nc in ((19, 21) if kind in ("ssd", "retina") else (0, 129)):
        p = _params(kind)
        p.num_fg = nc
        assert rejected(_call(L, kind, p)), nc
    if kind == "yolo":
        for A in (0, 10):
            p = _params(kind)
            for i in range(3):
                p.level[i].A = A
            assert rejected(_call(L, kind, p)), A


# ------------------------------------------------------------------ ground truth --
def _padded(counts, G):
    g = np.full((len(counts), G, 5), -1.0, F32)
    for b, n in enumerate(counts):
        g[b, :n] = [100.0, 100.0, 20.0, 20.0, 1.0]
    return g


def test_ground_truth_up_to_128_rows_passes_unchanged():
    from odt_b200.engine import loss_ground_truth
    for G in (1, 60, 128):
        g = _padded([0, min(5, G - 1)], G)
        out = loss_ground_truth(g)
        assert out.dtype == np.float32 and np.array_equal(out, g)
    g = np.full((1, 128, 5), 50.0, F32)  # no padding row at all: the count is the argmin, as in the reference
    assert np.array_equal(loss_ground_truth(g), g)


def test_ground_truth_beyond_128_rows_is_trimmed_to_the_counts():
    from odt_b200.engine import loss_ground_truth
    g = _padded([3, 40, 0], 300)
    out = loss_ground_truth(g)
    assert out.shape == (3, 41, 5) and np.array_equal(out, g[:, :41])
    assert list(np.argmin(out[:, :, 0], axis=1)) == [3, 40, 0]
    out = loss_ground_truth(_padded([127, 2], 200))
    assert out.shape == (2, 128, 5) and list(np.argmin(out[:, :, 0], axis=1)) == [127, 2]


def test_ground_truth_with_too_many_boxes_is_rejected():
    from odt_b200.engine import loss_ground_truth
    for counts in ([128, 1], [2, 150]):
        with pytest.raises(ValueError, match="128"):
            loss_ground_truth(_padded(counts, 200))
    with pytest.raises(ValueError, match="shape"):
        loss_ground_truth(np.zeros((2, 5), F32))


def test_training_data_term_rejects_too_many_boxes_before_any_launch(built):
    """The GPU data term checks the ground truth first: the ValueError comes before any buffer or launch (here on a
    CPU trainer, where a launch could not run at all)."""
    import YOLOv3
    from helpers import model_cfg
    from odt_b200.train import GraphTrainer, LossKernels
    tr = GraphTrainer(YOLOv3.YOLOv3(model_cfg("yolov3"), None), "cpu")
    assert tr._loss_kernels is None  # the CPU keeps the restatement
    k = LossKernels(tr)
    rows = torch.zeros((2, k.N, tr.row))
    with pytest.raises(ValueError, match="128"):
        k(rows, _padded([3, 129], 140))
    assert not k._bufs
