"""The training-mode ops of the reference's spectrogram U-Net (Models/UnetSpectrogramSeparator.py with training=True),
layered onto tf_shim.py + tf_shim_spectrogram.py without changing them:

    tf.contrib.layers.batch_norm(is_training=True)  TF 1.8 defaults center=True, scale=False, epsilon=1e-3, decay=0.999,
        fused: normalise with the batch mean and the biased batch variance over N*H*W; the UPDATE_OPS values
        moving -= (moving - batch value) * (1 - decay), with the Bessel-corrected variance var * n / max(n - 1, 1) (what
        FusedBatchNorm returns for the moving average, as recalled - no TensorFlow source is available here), are recorded
        in TRAIN.moving
    tf.layers.dropout(training=True)                 rate 0.5: x / 0.5 * keep, the keep masks popped from TRAIN.masks in
        call order (TF's stateful RNG cannot be reproduced; the masks are inputs of the fixture instead)

Inference-mode calls go to tf_shim_spectrogram's ops unchanged.  Used ONLY by make_spectrogram_train_golden.py.
"""
import sys

import torch

import tf_shim_spectrogram
from tf_shim import T, _make_var, _unique


class _Train:
    def __init__(self):
        self.reset()

    def reset(self):
        self.moving = {}        # moving-statistic name -> value after this step's UPDATE_OPS
        self.masks = []         # keep masks (bool, NHWC) for the dropout calls, in call order


TRAIN = _Train()
DECAY = 0.999


def _batch_norm(inputs, activation_fn=None, is_training=True, **kw):
    if not is_training:
        return _inference_batch_norm(inputs, activation_fn=activation_fn, is_training=False, **kw)
    x = inputs.t
    c = x.shape[-1]
    scope = _unique("BatchNorm")
    beta = _make_var(scope + "/beta", (c,), zeros=True)
    moving_mean = _make_var(scope + "/moving_mean", (c,), zeros=True)
    moving_var = tf_shim_spectrogram._make_ones_var(scope + "/moving_variance", (c,))
    n = x.shape[0] * x.shape[1] * x.shape[2]
    mean = x.mean(dim=(0, 1, 2))
    var = ((x - mean) ** 2).mean(dim=(0, 1, 2))
    with torch.no_grad():
        TRAIN.moving[scope + "/moving_mean"] = (moving_mean - (moving_mean - mean) * (1.0 - DECAY)).numpy().copy()
        unbiased = var * n / max(n - 1, 1)
        TRAIN.moving[scope + "/moving_variance"] = (moving_var - (moving_var - unbiased) * (1.0 - DECAY)).numpy().copy()
    out = T((x - mean) / torch.sqrt(var + 1e-3) + beta)
    return activation_fn(out) if activation_fn is not None else out


def _dropout(x, rate=0.5, training=False, **kw):
    if not training:
        return x
    keep = torch.as_tensor(TRAIN.masks.pop(0), dtype=x.t.dtype)
    assert tuple(keep.shape) == tuple(x.t.shape)
    return T(x.t / (1.0 - rate) * keep)


_inference_batch_norm = None


def install():
    """tf_shim_spectrogram.install(), then the training-mode batch norm and dropout."""
    global _inference_batch_norm
    tf = tf_shim_spectrogram.install()
    _inference_batch_norm = tf.contrib.layers.batch_norm
    tf.contrib.layers.batch_norm = _batch_norm
    tf.layers.dropout = _dropout
    sys.modules["tensorflow.contrib.layers"].batch_norm = _batch_norm
    return tf

