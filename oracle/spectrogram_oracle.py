"""float64 torch restatement of the spectrogram U-Net's inference graph (the reference's
Models/UnetSpectrogramSeparator.py with training=False) and of Test.test's U7a magnitude loss (Test.py:57-71).

    STFT: frame 1024, hop 768, fft 1024, periodic Hann, no end padding -> n = 1 + (T - 1024) // 768 frames of 513 bins
    per source: log1p(|X|)[..., :512] NHWC -> L x (conv2d 5x5/2 'same' + bias + BN + LeakyReLU(0.2))
              -> L-1 x (conv2d_transpose 5x5/2 'same' + bias + BN + ReLU, concat([skip, up]))
              -> conv2d_transpose to 1 channel + sigmoid, bin 512 padded with 0.5 -> mask
    magnitudes mask * |X|; audio inverse_stft(mask * X) with inverse_stft_window_fn(768, hann)
    BN (inference, center only): (x - moving_mean) / sqrt(moving_variance + 1e-3) + beta

TF's 'same' padding of a stride-2, 5-tap conv on an even length is 1 before and 2 after; its transpose feeds output
2i + k - 1 from input i and tap k and drops outputs at or beyond 2N.
"""
import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

FRAME, HOP, BINS = 1024, 768, 513
BN_EPS = 1e-3


def stft_frames(T):
    return 1 + (T - FRAME) // HOP


def hann(n=FRAME):
    j = torch.arange(n, dtype=torch.float64)
    return 0.5 - 0.5 * torch.cos(2 * math.pi * j / n)


def inverse_window():
    """inverse_stft_window_fn(768, hann): w / d with d[j] = sum_m w[j mod 768 + 768 m]^2."""
    w = hann()
    sq = F.pad(w * w, (0, 2 * HOP - FRAME)).view(2, HOP).sum(0)
    return w / sq.repeat(2)[:FRAME]


def stft(x):
    """x [B, T] float64 -> complex128 [B, n, 513]."""
    x = torch.as_tensor(x, dtype=torch.float64)
    frames = x.unfold(-1, FRAME, HOP)
    return torch.fft.rfft(frames * hann(), n=FRAME)


def istft(X, T):
    """complex [B, n, 513] -> [B, T]: irfft, inverse window, overlap-add with hop 768."""
    frames = torch.fft.irfft(X, n=FRAME) * inverse_window()
    B, n = frames.shape[:2]
    out = torch.zeros((B, (n - 1) * HOP + FRAME), dtype=torch.float64)
    for f in range(n):
        out[:, f * HOP:f * HOP + FRAME] += frames[:, f]
    return out[:, :T]


def param_specs(num_layers, num_initial_filters, num_sources=2):
    """[(TF name, shape)] in creation order, the name counters running on across sources."""
    L, Fi = num_layers, num_initial_filters
    out, n_conv, n_tconv, n_bn = [], 0, 0, 0

    def name(base, i):
        return "separator/%s%s" % (base, "" if i == 0 else "_%d" % i)

    def bn(c):
        nonlocal n_bn
        s = name("BatchNorm", n_bn)
        n_bn += 1
        out.extend([(s + "/beta", (c,)), (s + "/moving_mean", (c,)), (s + "/moving_variance", (c,))])

    for _ in range(num_sources):
        cin = 1
        for i in range(L):
            s = name("conv2d", n_conv)
            n_conv += 1
            cout = Fi * 2 ** i
            out.extend([(s + "/kernel", (5, 5, cin, cout)), (s + "/bias", (cout,))])
            bn(cout)
            cin = cout
        for i in range(L - 1):
            s = name("conv2d_transpose", n_tconv)
            n_tconv += 1
            cout = Fi * 2 ** (L - i - 2)
            out.extend([(s + "/kernel", (5, 5, cout, cin)), (s + "/bias", (cout,))])
            bn(cout)
            cin = 2 * cout
        s = name("conv2d_transpose", n_tconv)
        n_tconv += 1
        out.extend([(s + "/kernel", (5, 5, 1, cin)), (s + "/bias", (1,))])
    return out


def random_params(num_layers, num_initial_filters, seed, num_sources=2):
    """Glorot-uniform kernels and non-trivial biases, betas, moving means and moving variances (in [0.5, 2]), float32
    values.  OrderedDict name -> array."""
    rng = np.random.default_rng(seed)
    p = OrderedDict()
    for n, shape in param_specs(num_layers, num_initial_filters, num_sources):
        if n.endswith("/kernel"):
            lim = math.sqrt(6.0 / (shape[0] * shape[1] * (shape[2] + shape[3])))
            a = rng.uniform(-lim, lim, size=shape)
        elif n.endswith("/moving_variance"):
            a = rng.uniform(0.5, 2.0, size=shape)
        else:
            a = rng.uniform(-0.1, 0.1, size=shape)
        p[n] = a.astype(np.float32)
    return p


def _bn(x, params, prefix):
    g = lambda k: torch.as_tensor(np.asarray(params[prefix + k], np.float64))
    return (x - g("/moving_mean")) / torch.sqrt(g("/moving_variance") + BN_EPS) + g("/beta")


def _t(a):
    return torch.as_tensor(np.asarray(a, np.float64))


def forward(params, mix, num_layers, source_names, return_spectrogram=False):
    """mix [B, T, 1] -> OrderedDict name -> float64 numpy: audio [B, T, 1], or magnitudes [B, n, 513]."""
    mix = torch.as_tensor(np.asarray(mix, np.float64))
    assert mix.shape[2] == 1
    T = mix.shape[1]
    X = stft(mix[:, :, 0])
    mag = X.abs()
    x0 = torch.log1p(mag)[:, :, :-1].unsqueeze(1)             # NCHW [B, 1, n, 512]
    names = [n for n, _ in param_specs(num_layers, 1, len(source_names))]
    conv_names = iter(n[:-len("/kernel")] for n in names if n.endswith("/kernel") and "/conv2d" in n
                      and "transpose" not in n)
    tconv_names = iter(n[:-len("/kernel")] for n in names if "conv2d_transpose" in n and n.endswith("/kernel"))
    bn_names = iter(n[:-len("/beta")] for n in names if n.endswith("/beta"))
    out = OrderedDict()
    for name in source_names:
        cur, enc = x0, []
        for i in range(num_layers):
            s = next(conv_names)
            w = _t(params[s + "/kernel"]).permute(3, 2, 0, 1)
            y = F.conv2d(F.pad(cur, (1, 2, 1, 2)), w, _t(params[s + "/bias"]), stride=2)
            y = _bn(y.permute(0, 2, 3, 1), params, next(bn_names)).permute(0, 3, 1, 2)
            cur = torch.maximum(0.2 * y, y)
            if i < num_layers - 1:
                enc.append(cur)
        for i in range(num_layers - 1):
            s = next(tconv_names)
            w = _t(params[s + "/kernel"]).permute(3, 2, 0, 1)          # [Cin, Cout, 5, 5]
            H, W = cur.shape[2], cur.shape[3]
            y = F.conv_transpose2d(cur, w, _t(params[s + "/bias"]), stride=2, padding=1)[:, :, :2 * H, :2 * W]
            y = _bn(y.permute(0, 2, 3, 1), params, next(bn_names)).permute(0, 3, 1, 2)
            cur = torch.cat([enc[-i - 1], torch.relu(y)], dim=1)
        s = next(tconv_names)
        w = _t(params[s + "/kernel"]).permute(3, 2, 0, 1)
        H, W = cur.shape[2], cur.shape[3]
        m = torch.sigmoid(F.conv_transpose2d(cur, w, _t(params[s + "/bias"]), stride=2, padding=1)[:, :, :2 * H, :2 * W])
        mask = F.pad(m[:, 0], (0, 1), value=0.5)                     # [B, n, 513]
        if return_spectrogram:
            out[name] = (mask * mag).numpy()
        else:
            out[name] = istft(mask * X, T).unsqueeze(2).numpy()
    return out


def magnitude_l1(targets, est_mags):
    """Test.py:63-67,71 for one batch: sum_k mean|STFTmag(target_k) - est_k| / K.  targets / est_mags: lists over sources of
    [B, T, 1] audio and [B, n, 513] magnitudes."""
    total = 0.0
    for t, e in zip(targets, est_mags):
        real = stft(torch.as_tensor(np.asarray(t, np.float64))[:, :, 0]).abs()
        total += float(torch.mean(torch.abs(real - torch.as_tensor(np.asarray(e, np.float64)))))
    return total / len(targets)
