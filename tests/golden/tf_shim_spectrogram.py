"""The ops the reference's spectrogram U-Net (Models/UnetSpectrogramSeparator.py) touches, added to the eager `tensorflow`
stand-in of tf_shim.py, inference graph only:

    tf.contrib.signal.stft / inverse_stft / inverse_stft_window_fn, the tensorflow.contrib.signal.python.ops.window_ops
    module path (hann_window), tf.layers.conv2d / conv2d_transpose / dropout, tf.contrib.layers.batch_norm,
    tf.log1p / abs / angle / complex / exp / multiply / pad, tf.nn.relu (squeeze, expand_dims, sigmoid come from tf_shim)

Leaf ops follow the TF-1.8 op definitions on float64 / complex128 torch-CPU tensors.  Variables go through tf_shim's
registry, so their names and creation order are the ones the reference's graph code produces.  Used ONLY by
make_spectrogram_golden.py.
"""
import math
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

import tf_shim
from tf_shim import STATE, T, _make_var, _unique


def _make_ones_var(name, shape):
    """A variable initialised to ones (batch norm's moving_variance)."""
    if name not in STATE.vars:
        STATE.vars[name] = torch.ones(shape, dtype=STATE.dtype, requires_grad=True)
    return STATE.vars[name]


def _glorot_kernel(name, shape):
    receptive = shape[0] * shape[1]
    return _make_var(name, shape, glorot_fans=(receptive * shape[2], receptive * shape[3]))


def _conv2d_layer(inputs, filters, kernel_size, strides=(1, 1), activation=None, padding="valid", **kw):
    """tf.layers.conv2d, NHWC; kernel [kh, kw, C_in, filters].  'same' pads (total - total // 2) after, as TF does."""
    x = inputs.t
    kh, kw = kernel_size
    lname = _unique("conv2d")
    kern = _glorot_kernel(lname + "/kernel", (kh, kw, x.shape[3], filters))
    bias = _make_var(lname + "/bias", (filters,), zeros=True)
    xt = x.permute(0, 3, 1, 2)
    if padding.lower() == "same":
        pads = []
        for size, k, st in ((x.shape[2], kw, strides[1]), (x.shape[1], kh, strides[0])):
            out = -(-size // st)
            total = max((out - 1) * st + k - size, 0)
            pads += [total // 2, total - total // 2]
        xt = F.pad(xt, pads)
    y = F.conv2d(xt, kern.permute(3, 2, 0, 1), bias, stride=tuple(strides)).permute(0, 2, 3, 1)
    return activation(T(y)) if activation is not None else T(y)


def _conv2d_transpose_layer(inputs, filters, kernel_size, strides=(1, 1), activation=None, padding="valid", **kw):
    """tf.layers.conv2d_transpose, NHWC; kernel [kh, kw, filters, C_in].  'same': the adjoint of a 'same' conv whose input
    is size * stride long, i.e. the full transposed conv cropped by that conv's front padding (total // 2)."""
    x = inputs.t
    kh, kw = kernel_size
    assert padding.lower() == "same"
    lname = _unique("conv2d_transpose")
    kern = _make_var(lname + "/kernel", (kh, kw, filters, x.shape[3]),
                     glorot_fans=(kh * kw * x.shape[3], kh * kw * filters))
    bias = _make_var(lname + "/bias", (filters,), zeros=True)
    y = F.conv_transpose2d(x.permute(0, 3, 1, 2), kern.permute(3, 2, 0, 1), stride=tuple(strides))
    crops = []
    for size, k, st in ((x.shape[1], kh, strides[0]), (x.shape[2], kw, strides[1])):
        total = max((size - 1) * st + k - size * st, 0)
        crops.append((total // 2, total // 2 + size * st))
    y = y[:, :, crops[0][0]:crops[0][1], crops[1][0]:crops[1][1]] + bias.view(1, -1, 1, 1)
    out = T(y.permute(0, 2, 3, 1))
    return activation(out) if activation is not None else out


def _batch_norm(inputs, activation_fn=None, is_training=True, **kw):
    """tf.contrib.layers.batch_norm defaults (center=True, scale=False, epsilon=1e-3), inference form only."""
    if is_training:
        raise NotImplementedError("tf_shim: batch_norm is implemented in inference mode only")
    x = inputs.t
    c = x.shape[-1]
    scope = _unique("BatchNorm")
    beta = _make_var(scope + "/beta", (c,), zeros=True)
    mean = _make_var(scope + "/moving_mean", (c,), zeros=True)
    var = _make_ones_var(scope + "/moving_variance", (c,))
    out = T((x - mean) / torch.sqrt(var + 1e-3) + beta)
    return activation_fn(out) if activation_fn is not None else out


def _hann_window(window_length, periodic=True, dtype=None):
    n = int(window_length)
    denom = n if periodic else n - 1
    j = torch.arange(n, dtype=torch.float64)
    return T(0.5 - 0.5 * torch.cos(2 * math.pi * j / denom))


def _stft(signals, frame_length, frame_step, fft_length=None, window_fn=_hann_window, pad_end=False):
    assert not pad_end
    frames = signals.t.unfold(-1, frame_length, frame_step)
    if window_fn is not None:
        frames = frames * window_fn(frame_length, dtype=None).t
    return T(torch.fft.rfft(frames, n=fft_length or frame_length))


def _inverse_stft_window_fn(frame_step, forward_window_fn=_hann_window):
    def fn(frame_length, dtype=None):
        w = forward_window_fn(frame_length, dtype=dtype).t
        overlaps = -(-frame_length // frame_step)
        d = F.pad(w * w, (0, overlaps * frame_step - frame_length)).view(overlaps, frame_step).sum(0, keepdim=True)
        d = d.repeat(overlaps, 1).reshape(-1)[:frame_length]
        return T(w / d)
    return fn


def _inverse_stft(stfts, frame_length, frame_step, fft_length=None, window_fn=_hann_window):
    frames = torch.fft.irfft(stfts.t, n=fft_length or frame_length)[..., :frame_length]
    if window_fn is not None:
        frames = frames * window_fn(frame_length, dtype=None).t
    n = frames.shape[-2]
    out = torch.zeros(frames.shape[:-2] + ((n - 1) * frame_step + frame_length,), dtype=frames.dtype)
    for f in range(n):
        out[..., f * frame_step:f * frame_step + frame_length] += frames[..., f, :]
    return T(out)


def _pad(tensor, paddings, mode="CONSTANT", constant_values=0):
    assert mode.upper() == "CONSTANT"
    flat = []
    for before, after in reversed([tuple(p) for p in paddings]):
        flat += [before, after]
    return T(F.pad(tensor.t, flat, value=constant_values))


def _complex(real, imag):
    r = real.t if isinstance(real, T) else torch.as_tensor(real, dtype=torch.float64)
    i = imag.t if isinstance(imag, T) else torch.as_tensor(imag, dtype=torch.float64)
    r, i = torch.broadcast_tensors(r, i)
    return T(torch.complex(r, i))


def _dropout(x, training=False, **kw):
    if training:
        raise NotImplementedError("tf_shim: dropout is implemented in inference mode only")
    return x


def install():
    """tf_shim.install(), then the spectrogram U-Net's ops on the same fake `tensorflow` modules."""
    tf = tf_shim.install()
    layers, nn = tf.layers, tf.nn
    tf.log1p = lambda x: T(torch.log1p(x.t))
    tf.abs = lambda x: T(torch.abs(x.t))
    tf.angle = lambda x: T(torch.angle(x.t))
    tf.complex = _complex
    tf.exp = lambda x: T(torch.exp(x.t))
    tf.multiply = lambda a, b: T((a.t if isinstance(a, T) else a) * (b.t if isinstance(b, T) else b))
    tf.pad = _pad
    layers.conv2d = _conv2d_layer
    layers.conv2d_transpose = _conv2d_transpose_layer
    layers.dropout = _dropout
    nn.relu = lambda x: T(torch.relu(x.t))
    contrib = types.ModuleType("tensorflow.contrib")
    signal = types.ModuleType("tensorflow.contrib.signal")
    signal.stft = _stft
    signal.inverse_stft = _inverse_stft
    signal.inverse_stft_window_fn = _inverse_stft_window_fn
    contrib_layers = types.ModuleType("tensorflow.contrib.layers")
    contrib_layers.batch_norm = _batch_norm
    contrib.signal = signal
    contrib.layers = contrib_layers
    tf.contrib = contrib
    python = types.ModuleType("tensorflow.contrib.signal.python")
    ops = types.ModuleType("tensorflow.contrib.signal.python.ops")
    window_ops = types.ModuleType("tensorflow.contrib.signal.python.ops.window_ops")
    window_ops.hann_window = _hann_window
    signal.python, python.ops, ops.window_ops = python, ops, window_ops
    for m in (contrib, signal, contrib_layers, python, ops, window_ops):
        sys.modules[m.__name__] = m
    return tf
