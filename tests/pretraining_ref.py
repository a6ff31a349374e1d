"""Test references for RetinaNet's ImageNet-pretraining mode, composed from the CPU oracle's RetinaNet pieces
(oracle/nets.py) and numpy: the last feature tensor of the ResNet, the pooled logits and TF's sparse softmax
cross-entropy (ref RetinaNet.py:120-127)."""
import numpy as np

F32 = np.float32


def retinanet_features(weights, images, block_list=(3, 4, 6, 3)):
    """`_feature_extractor(images - mean)[-1]` (RetinaNet.py:121-122): the last bottleneck's conv + shortcut sum,
    NHWC float32 -- the same ResNet, with the same variable names, as oracle.nets.retinanet_heads."""
    from oracle import nets as ON
    from oracle import tfops as T
    c = ON.Ctx(weights)
    x = (images.astype(F32) - T.RGB_MEAN.reshape(1, 1, 1, 3)).astype(F32)
    filters = [7 * (2 ** i) for i in range(len(block_list))]
    with c.n.scope("feature_extractor"):
        _, _, features = ON._resnet(c, x, filters, list(block_list), "bn")
    return features


def pooled_logits(features):
    """reduce_mean over [1, 2] of NHWC features, float64."""
    return np.asarray(features, np.float64).mean(axis=(1, 2))


def sparse_softmax_xent(logits, labels):
    """Per-example sparse softmax cross-entropy as TF computes it, in float32:
    log(sum exp(x - max)) - (x_label - max)."""
    x = np.asarray(logits, F32)
    m = x.max(axis=1, keepdims=True)
    s = np.exp(x - m).sum(axis=1, dtype=F32)
    lab = np.asarray(labels, np.int64)
    return (np.log(s) - (x[np.arange(len(lab)), lab] - m[:, 0])).astype(F32)


def sparse_softmax_xent64(logits, labels):
    """The same in float64 (the kernel's reference)."""
    x = np.asarray(logits, np.float64)
    m = x.max(axis=1, keepdims=True)
    lab = np.asarray(labels, np.int64)
    return np.log(np.exp(x - m).sum(axis=1)) - (x[np.arange(len(lab)), lab] - m[:, 0])
