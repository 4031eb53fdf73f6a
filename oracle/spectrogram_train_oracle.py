"""float64 torch restatement of one training step of the spectrogram U-Net baselines (the reference's
Models/UnetSpectrogramSeparator.py get_output with training=True, the loss of Training.py:50-63 and the Adam / UPDATE_OPS
step of :66-77), differentiated by torch autograd.

    per source k, in source_names order, one U-Net on log1p(|X|)[..., :512] (spectrogram_oracle's wiring), with
      batch norm (training): (z - mean) / sqrt(var + 1e-3) + beta, mean and biased var over B*H*W per channel;
        UPDATE_OPS moving -= (moving - batch value) * (1 - 0.999), the variance Bessel-corrected N / max(N - 1, 1)
      dropout(rate 0.5, training) on the concatenation of up steps 0, 1, 2 (levels L-2, L-3, L-4): kept elements x 2
      LeakyReLU tf.maximum(0.2 v, v): slope 0.2 at v = 0 (TF's Maximum gradient sends the tie to its first argument);
      ReLU: slope 0 at 0
    U7  (raw_audio_loss): sum_k mean((target_k - istft(mask_k X))^2) / K
    U7a: sum_k mean|STFTmag(target_k) - mask_k |X|| / K   (d|x|/dx = sign(x), sign(0) = 0 as TF's Abs gradient)

TF 1.8's FusedBatchNorm returns the Bessel-corrected batch variance, with max(N - 1, 1) in the divisor, for the moving
average; that is recalled from its kernel, not read from it (no TensorFlow source is available here), as
wun.KAISER_BEST_* is for resampy.

The dropout keep bits are this project's counter-based hash (csrc/kernels.h spec_dropout_keep; the reference draws them
with TF's stateful RNG, which cannot be reproduced): keep_masks restates it in numpy, so the oracle can run with the masks the
engine used.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from oracle import spectrogram_oracle as S
from oracle.feeder_oracle import M64, mix64

DECAY = 0.999
GOLDEN = 0x9E3779B97F4A7C15


def dropped_levels(num_layers):
    """Concatenation levels tf.layers.dropout acts on: up step i < 3 drops level L - 2 - i."""
    return [d for d in range(num_layers - 1) if d >= num_layers - 4]


def keep_masks(seed, step, source, level, shape):
    """Keep bits (bool, NHWC `shape`) of `level` in the U-Net of `source` at dropout step `step`."""
    key = ((step << 16) & M64) ^ (source << 8) ^ level
    stream = np.uint64(mix64((seed & M64) ^ mix64((key + GOLDEN) & M64)))
    i = np.arange(int(np.prod(shape)), dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = stream + i * np.uint64(GOLDEN)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(63)).astype(bool).reshape(shape)


def level_shape(batch, n_frames, num_layers, num_initial_filters, d):
    """NHWC shape of the concatenation at level d < L - 1."""
    return (batch, n_frames >> (d + 1), 512 >> (d + 1), 2 * num_initial_filters * 2 ** d)


def engine_masks(seed, step, batch, n_frames, num_layers, num_initial_filters, num_sources=2):
    """{(source, level): keep bits} of one call at dropout step `step`."""
    return {(k, d): keep_masks(seed, step, k, d, level_shape(batch, n_frames, num_layers, num_initial_filters, d))
            for k in range(num_sources) for d in dropped_levels(num_layers)}


def trainable(name):
    return not name.endswith(("/moving_mean", "/moving_variance"))


def _names(num_layers, num_sources):
    names = [n for n, _ in S.param_specs(num_layers, 1, num_sources)]
    conv = [n[:-len("/kernel")] for n in names if n.endswith("/kernel") and "transpose" not in n]
    tconv = [n[:-len("/kernel")] for n in names if n.endswith("/kernel") and "transpose" in n]
    bn = [n[:-len("/beta")] for n in names if n.endswith("/beta")]
    return iter(conv), iter(tconv), iter(bn)


def forward_backward(params, mix, targets, num_layers, source_names, raw_audio_loss, masks, bias_scale=None, positive=None,
                     report=None):
    """One training step's loss, gradients and batch statistics.
    params: name -> array; mix [B, T, 1]; targets: list over sources of [B, T, 1]; masks: {(source, level): keep bits}.
    Returns (loss, grads: OrderedDict trainable name -> float64 array, moving: OrderedDict moving-statistic name -> the
    value after this step's update (float64 of the float32 inputs)).
    bias_scale (a dict, optional) receives, per conv bias that feeds batch norm, rstd * sum(|dy| + |mean dy| +
    |xhat mean(dy xhat)|) per channel: the magnitudes whose cancellation makes that bias's gradient (0 in exact
    arithmetic) rounding noise, which bounds it in float32.
    positive (optional): {batch-norm index in creation order: bool NHWC array} - the activation slopes to use there (True:
    slope 1) instead of the oracle's own v > 0, e.g. the engine's; then `report` (a list) receives (index, slopes that
    differ from the oracle's, largest |v| / rms(v) among them) per overridden layer."""
    mix = torch.as_tensor(np.asarray(mix, np.float64))
    T = mix.shape[1]
    X = S.stft(mix[:, :, 0])
    mag = X.abs()
    x0 = torch.log1p(mag)[:, :, :-1].unsqueeze(1)
    P = OrderedDict((n, torch.tensor(np.asarray(a, np.float64), requires_grad=trainable(n))) for n, a in params.items())
    conv_names, tconv_names, bn_names = _names(num_layers, len(source_names))
    moving = OrderedDict()
    n_bn = [0]

    def bn(y, act, bias_name):
        s = next(bn_names)
        index = n_bn[0]
        n_bn[0] += 1
        yt = y.permute(0, 2, 3, 1)                                   # NHWC
        n = yt.shape[0] * yt.shape[1] * yt.shape[2]
        mean = yt.mean(dim=(0, 1, 2))
        var = ((yt - mean) ** 2).mean(dim=(0, 1, 2))
        rstd = 1.0 / torch.sqrt(var + S.BN_EPS)
        xhat = (yt - mean) * rstd
        v = xhat + P[s + "/beta"]
        if bias_scale is not None:
            def hook(dy, xh=xhat.detach(), r=rstd.detach()):
                c1 = dy.mean(dim=(0, 1, 2))
                c2 = (dy * xh).mean(dim=(0, 1, 2))
                bias_scale[bias_name] = (r * (dy.abs() + c1.abs() + (xh * c2).abs()).sum(dim=(0, 1, 2))).numpy()
            v.register_hook(hook)
        with torch.no_grad():
            for key, val in (("/moving_mean", mean), ("/moving_variance", var * n / max(n - 1, 1))):
                old = P[s + key]
                moving[s + key] = (old - (old - val) * (1.0 - DECAY)).numpy()
        pos = v > 0
        if positive is not None and index in positive:
            want = torch.as_tensor(np.asarray(positive[index], bool))
            diff = want != pos
            if report is not None:
                rel = (v.detach().abs() / v.detach().pow(2).mean().sqrt())[diff]
                report.append((index, int(diff.sum()), float(rel.max()) if rel.numel() else 0.0))
            pos = want
        out = torch.where(pos, v, 0.2 * v if act == "lrelu" else torch.zeros_like(v))
        return out.permute(0, 3, 1, 2)

    def drop(x, k, d):
        if (k, d) not in masks:
            return x
        keep = torch.as_tensor(np.asarray(masks[(k, d)])).permute(0, 3, 1, 2).to(torch.float64)
        return x * keep * 2.0

    def tconv(x, s):
        w = P[s + "/kernel"].permute(3, 2, 0, 1)
        H, W = x.shape[2], x.shape[3]
        return F.conv_transpose2d(x, w, P[s + "/bias"], stride=2, padding=1)[:, :, :2 * H, :2 * W]

    L = num_layers
    loss = 0.0
    for k, name in enumerate(source_names):
        cur, enc = x0, []
        for i in range(L):
            s = next(conv_names)
            y = F.conv2d(F.pad(cur, (1, 2, 1, 2)), P[s + "/kernel"].permute(3, 2, 0, 1), P[s + "/bias"], stride=2)
            cur = bn(y, "lrelu", s + "/bias")
            if i < L - 1:
                enc.append(cur)
        for i in range(L - 1):
            s = next(tconv_names)
            cur = bn(tconv(cur, s), "relu", s + "/bias")
            cur = drop(torch.cat([enc[-i - 1], cur], dim=1), k, L - 2 - i)
        mask = F.pad(torch.sigmoid(tconv(cur, next(tconv_names)))[:, 0], (0, 1), value=0.5)    # [B, n, 513]
        tg = torch.as_tensor(np.asarray(targets[k], np.float64))[:, :, 0]
        if raw_audio_loss:
            loss = loss + torch.mean((tg - S.istft(mask * X, T)) ** 2)
        else:
            loss = loss + torch.mean(torch.abs(S.stft(tg).abs() - mask * mag))
    loss = loss / len(source_names)
    loss.backward()
    grads = OrderedDict((n, t.grad.numpy().copy()) for n, t in P.items() if trainable(n))
    return float(loss.detach()), grads, moving


def adam(params, grads, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    """One tf.train.AdamOptimizer step (the `step`-th, 1-based) on the trainables, in float64:
    lr_t = lr sqrt(1 - beta2^step) / (1 - beta1^step); m = b1 m + (1 - b1) g; v = b2 v + (1 - b2) g^2;
    p -= lr_t m / (sqrt(v) + eps).  Returns new (params, m, v) dicts; the moving statistics pass through unchanged."""
    lr_t = lr * np.sqrt(1 - beta2 ** step) / (1 - beta1 ** step)
    P, M, V = OrderedDict(), OrderedDict(), OrderedDict()
    for n, p in params.items():
        p = np.asarray(p, np.float64)
        if n not in grads:
            P[n] = p
            continue
        g = np.asarray(grads[n], np.float64)
        M[n] = beta1 * np.asarray(m[n], np.float64) + (1 - beta1) * g
        V[n] = beta2 * np.asarray(v[n], np.float64) + (1 - beta2) * g * g
        P[n] = p - lr_t * M[n] / (np.sqrt(V[n]) + eps)
    return P, M, V
