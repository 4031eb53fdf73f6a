"""The data-parallel training step of the spectrogram U-Net (wun_spec_forward_backward_dp) restated in float64 torch, for the
CPU and GPU tests: the batch is split into contiguous shards, one per rank, and

    batch norm  takes its statistics from the per-channel sums of every shard, added in rank order: mean = sum z / n,
                var = sum z^2 / n - mean^2 with n = B * H * W of the whole batch (the engine's one-pass formula);
    dropout     hashes element i of a shard as element (first example of the shard) * (elements per example) + i of the batch;
    the loss    of the whole batch is sum_r (B_r / B) * (shard r's mean loss), so its gradient is the sum of the ranks'
                gradients, each scaled by 1 / B.

Otherwise the wiring is oracle/spectrogram_train_oracle.py's, whose whole-batch step these results must reproduce."""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from oracle import spectrogram_oracle as S
from oracle import spectrogram_train_oracle as O
from oracle.feeder_oracle import M64, mix64


def shard_bounds(sizes):
    """[(lo, hi)] of contiguous shards of the given sizes."""
    out, lo = [], 0
    for n in sizes:
        out.append((lo, lo + n))
        lo += n
    return out


def shard_keep_masks(seed, step, source, level, shape, first):
    """O.keep_masks of a shard: its `shape`'s elements hashed as elements first, first + 1, ... of the batch."""
    key = ((step << 16) & M64) ^ (source << 8) ^ level
    stream = np.uint64(mix64((seed & M64) ^ mix64((key + O.GOLDEN) & M64)))
    i = np.arange(int(np.prod(shape)), dtype=np.uint64) + np.uint64(first)
    with np.errstate(over="ignore"):
        z = stream + i * np.uint64(O.GOLDEN)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(63)).astype(bool).reshape(shape)


def shard_masks(seed, step, lo, hi, n_frames, num_layers, num_initial_filters, num_sources=2):
    """{(source, level): keep bits} of the shard [lo, hi) of one data-parallel call at dropout step `step`."""
    out = {}
    for k in range(num_sources):
        for d in O.dropped_levels(num_layers):
            shape = O.level_shape(hi - lo, n_frames, num_layers, num_initial_filters, d)
            per_example = int(np.prod(shape[1:]))
            out[(k, d)] = shard_keep_masks(seed, step, k, d, shape, lo * per_example)
    return out


def sharded_step(params, mix, targets, num_layers, source_names, raw_audio_loss, seed, step, num_initial_filters, bounds):
    """One data-parallel step over the shards `bounds` ([(lo, hi)] covering the batch in order).
    Returns a dict: loss (the whole batch's), shard_losses [per shard], grads (the sum over the ranks; trainable name ->
    array), moving (moving-statistic name -> value after the update), stats ([(mean, biased var)] per batch norm in
    creation order)."""
    mix = torch.as_tensor(np.asarray(mix, np.float64))
    B, T = mix.shape[0], mix.shape[1]
    n_frames = S.stft_frames(T)
    X = [S.stft(mix[lo:hi, :, 0]) for lo, hi in bounds]
    mag = [x.abs() for x in X]
    x0 = [torch.log1p(m)[:, :, :-1].unsqueeze(1) for m in mag]
    masks = [shard_masks(seed, step, lo, hi, n_frames, num_layers, num_initial_filters, len(source_names))
             for lo, hi in bounds]
    P = OrderedDict((n, torch.tensor(np.asarray(a, np.float64), requires_grad=O.trainable(n))) for n, a in params.items())
    conv_names, tconv_names, bn_names = O._names(num_layers, len(source_names))
    moving, stats = OrderedDict(), []

    def bn(ys, act):
        s = next(bn_names)
        yt = [y.permute(0, 2, 3, 1) for y in ys]                     # NHWC
        n = B * yt[0].shape[1] * yt[0].shape[2]
        s1, s2 = 0.0, 0.0
        for y in yt:                                                 # rank order
            s1 = s1 + y.sum(dim=(0, 1, 2))
            s2 = s2 + (y * y).sum(dim=(0, 1, 2))
        mean = s1 / n
        var = torch.clamp(s2 / n - mean * mean, min=0.0)
        stats.append((mean.detach().numpy().copy(), var.detach().numpy().copy()))
        rstd = 1.0 / torch.sqrt(var + S.BN_EPS)
        with torch.no_grad():
            for key, val in (("/moving_mean", mean), ("/moving_variance", var * n / max(n - 1, 1))):
                old = P[s + key]
                moving[s + key] = (old - (old - val) * (1.0 - O.DECAY)).numpy()
        outs = []
        for y in yt:
            v = (y - mean) * rstd + P[s + "/beta"]
            outs.append(torch.where(v > 0, v, 0.2 * v if act == "lrelu" else torch.zeros_like(v)).permute(0, 3, 1, 2))
        return outs

    def drop(xs, k, d):
        if (k, d) not in masks[0]:
            return xs
        return [x * torch.as_tensor(m[(k, d)]).permute(0, 3, 1, 2).to(torch.float64) * 2.0 for x, m in zip(xs, masks)]

    def tconv(x, s):
        w = P[s + "/kernel"].permute(3, 2, 0, 1)
        H, W = x.shape[2], x.shape[3]
        return F.conv_transpose2d(x, w, P[s + "/bias"], stride=2, padding=1)[:, :, :2 * H, :2 * W]

    L, K = num_layers, len(source_names)
    shard_losses = [0.0] * len(bounds)
    for k in range(K):
        cur, enc = x0, []
        for i in range(L):
            s = next(conv_names)
            cur = bn([F.conv2d(F.pad(c, (1, 2, 1, 2)), P[s + "/kernel"].permute(3, 2, 0, 1), P[s + "/bias"], stride=2)
                      for c in cur], "lrelu")
            if i < L - 1:
                enc.append(cur)
        for i in range(L - 1):
            s = next(tconv_names)
            cur = bn([tconv(c, s) for c in cur], "relu")
            cur = drop([torch.cat([e, c], dim=1) for e, c in zip(enc[-i - 1], cur)], k, L - 2 - i)
        s = next(tconv_names)
        for r, (lo, hi) in enumerate(bounds):
            mask = F.pad(torch.sigmoid(tconv(cur[r], s))[:, 0], (0, 1), value=0.5)
            tg = torch.as_tensor(np.asarray(targets[k], np.float64))[lo:hi, :, 0]
            if raw_audio_loss:
                part = torch.mean((tg - S.istft(mask * X[r], T)) ** 2)
            else:
                part = torch.mean(torch.abs(S.stft(tg).abs() - mask * mag[r]))
            shard_losses[r] = shard_losses[r] + part / K
    loss = 0.0
    for (lo, hi), part in zip(bounds, shard_losses):
        loss = loss + part * ((hi - lo) / B)
    loss.backward()
    grads = OrderedDict((n, t.grad.numpy().copy()) for n, t in P.items() if O.trainable(n))
    return {"loss": float(loss.detach()), "shard_losses": [float(x.detach()) for x in shard_losses], "grads": grads,
            "moving": moving, "stats": stats}
