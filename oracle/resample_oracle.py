"""numpy restatement of librosa 0.6.2 resample(y, sr_in, sr_out) with res_type='kaiser_best': resampy 0.2's resample_f
loop, then fix_length's zero padding.  resampy itself is not run here; see DESIGN.md §4.6 for what this rests on.

Vectorised over the output frames t; the filter taps run in resampy's order (left wing ascending, then right wing
ascending), each product added in float64 and the float32 output rounded after every addition.  The filter table is an
input, so the loop can be checked apart from the filter design (wun.resample_tables builds kaiser_best's).
Signals are [n][nchan].
"""
import numpy as np


def time_register(n_out, ratio):
    """resampy's time_register for t = 0 .. n_out-1: the sequential float64 sum 0, inc, inc+inc, ... with inc = 1 / ratio
    (np.add.accumulate adds strictly in sequence)."""
    tr = np.zeros(n_out)
    if n_out > 1:
        tr[1:] = np.add.accumulate(np.full(n_out - 1, 1.0 / ratio))
    return tr


def _wing(y, x, first, sign, limit, frac, win, delta, precision, index_step):
    index_frac = frac * precision
    offset = index_frac.astype(np.int64)                         # int(): truncation
    eta = index_frac - offset
    count = np.minimum(limit, (len(win) - offset) // index_step)
    n_in = x.shape[0]
    for i in range(int(count.max(initial=0))):
        f = first + sign * i
        on = (i < count) & (f < n_in)                            # frames past the end read as zero (include/wun.h)
        idx = np.where(on, offset + i * index_step, 0)
        w = win[idx] + eta * delta[idx]
        xs = x[np.where(on, f, 0)].astype(np.float64)
        for c in range(x.shape[1]):
            y[:, c] = np.where(on, (y[:, c].astype(np.float64) + w * xs[:, c]).astype(np.float32), y[:, c])


def resample_f(x, ratio, win, delta, precision, frames=None):
    """resampy's resample_f: float32 [n_in][nchan] -> float32 [int(n_in * ratio)][nchan]; with `frames` (output frame
    indices) only those rows."""
    x = np.asarray(x, np.float32)
    n_in = x.shape[0]
    n_out = int(n_in * ratio)
    scale = min(1.0, ratio)
    index_step = int(scale * precision)
    tr = time_register(n_out, ratio)
    if frames is not None:
        tr = tr[frames]
    n = tr.astype(np.int64)                                      # int(time_register)
    frac = scale * (tr - n)
    y = np.zeros((tr.shape[0], x.shape[1]), np.float32)
    _wing(y, x, n, -1, n + 1, frac, win, delta, precision, index_step)
    _wing(y, x, n + 1, 1, n_in - n - 1, scale - frac, win, delta, precision, index_step)
    return y


def resample(x, sr_in, sr_out, win, delta, precision):
    """librosa.resample(x.T, sr_in, sr_out).T for x float32 [n][nchan]; `win` already scaled by the ratio when
    downsampling and `delta` its difference (wun.resample_tables)."""
    if sr_in == sr_out:
        return x
    ratio = float(sr_out) / sr_in
    n_out = int(np.ceil(x.shape[0] * ratio))
    if int(x.shape[0] * ratio) < 1:
        raise ValueError("input of %d frames too short to resample from %d to %d" % (x.shape[0], sr_in, sr_out))
    y = resample_f(x, ratio, win, delta, precision)
    return np.concatenate([y, np.zeros((n_out - y.shape[0], y.shape[1]), np.float32)])      # fix_length
