"""librosa 0.6.2 / resampy 0.2 kaiser_best resampling without a GPU: the numpy oracle (oracle/resample_oracle.py) against a
literal scalar transcription of resampy's resample_f loop, the filter table (wun.kaiser_best_filter), signals through the
oracle, lengths, an independent cross-check against torchaudio, and Predict.py's WAV reading and writing."""
import math

import numpy as np
import pytest
import scipy.io.wavfile
import scipy.special

import Predict
import wun
from oracle import resample_oracle as R

RATIOS = [(44100, 22050), (22050, 44100), (48000, 22050), (22050, 48000), (44100, 8192), (16000, 22050)]


def literal_resample(x, sr_in, sr_out):
    """librosa.resample(x.T, sr_in, sr_out).T written out as resampy's resample_f loop, one scalar at a time, followed by
    fix_length; float32 output rounded after every addition."""
    win, delta = wun.resample_tables(sr_in, sr_out)
    num_table = wun.KAISER_BEST_PRECISION
    sample_ratio = float(sr_out) / sr_in
    n_orig, n_channels = x.shape
    y = np.zeros((int(n_orig * sample_ratio), n_channels), np.float32)
    scale = min(1.0, sample_ratio)
    time_increment = 1.0 / sample_ratio
    index_step = int(scale * num_table)
    time_register = 0.0
    nwin = win.shape[0]
    for t in range(y.shape[0]):
        n = int(time_register)
        frac = scale * (time_register - n)
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        i_max = min(n + 1, (nwin - offset) // index_step)
        for i in range(i_max):
            weight = float(win[offset + i * index_step]) + eta * float(delta[offset + i * index_step])
            for j in range(n_channels):
                y[t, j] = np.float32(float(y[t, j]) + weight * float(x[n - i, j]))
        frac = scale - frac
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        k_max = min(n_orig - n - 1, (nwin - offset) // index_step)
        for k in range(k_max):
            weight = float(win[offset + k * index_step]) + eta * float(delta[offset + k * index_step])
            for j in range(n_channels):
                y[t, j] = np.float32(float(y[t, j]) + weight * float(x[n + k + 1, j]))
        time_register += time_increment
    n_fix = int(math.ceil(n_orig * sample_ratio))
    return np.concatenate([y, np.zeros((n_fix - y.shape[0], n_channels), np.float32)])


def oracle(x, sr_in, sr_out):
    win, delta = wun.resample_tables(sr_in, sr_out)
    return R.resample(x, sr_in, sr_out, win, delta, wun.KAISER_BEST_PRECISION)


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("sr_in,sr_out", RATIOS)
def test_oracle_matches_literal_transcription(sr_in, sr_out):
    rng = np.random.default_rng(sr_in + sr_out)
    lengths = [n for n in range(1, 401) if int(n * float(sr_out) / sr_in) >= 1]
    lengths = [n for n in lengths if n <= 64 or n % 7 == 0 or n == lengths[-1]]      # every short length, then a stride to 400
    for n in lengths:
        x = (rng.standard_normal((n, 2)) * 0.3).astype(np.float32)
        want = literal_resample(x, sr_in, sr_out)
        assert same_bits(oracle(x, sr_in, sr_out), want), n
        assert same_bits(oracle(x[:, :1].copy(), sr_in, sr_out), want[:, :1].copy()), n       # channels are independent


def test_filter_table():
    win, precision = wun.kaiser_best_filter()
    rolloff, beta = wun.KAISER_BEST_ROLLOFF, wun.KAISER_BEST_BETA
    assert precision == 512 and win.shape == (32769,) and win.dtype == np.float64
    assert win[0] == rolloff
    want_last = rolloff * np.sinc(64 * rolloff) / scipy.special.i0(beta)
    assert abs(win[-1] - want_last) <= 1e-14 * abs(want_last)
    # downsampling scales the table by the ratio; delta is its forward difference with a trailing zero
    w, d = wun.resample_tables(44100, 22050)
    np.testing.assert_array_equal(w, win * 0.5)
    assert d[-1] == 0 and np.array_equal(d[:-1], np.diff(w))
    w, d = wun.resample_tables(22050, 44100)
    np.testing.assert_array_equal(w, win)


def test_filter_response():
    """The full symmetric filter (the table mirrored, 512 taps per input sample): flat to 1e-5 dB up to 0.9 x rolloff x
    Nyquist, at least 140 dB down above 1.03 x Nyquist."""
    win, precision = wun.kaiser_best_filter()
    h = np.concatenate([win[:0:-1], win])
    nfft = 2 ** 22
    mag = np.abs(np.fft.rfft(h, nfft)) / precision
    f = np.arange(mag.size) * precision / nfft                     # cycles per input sample; Nyquist = 0.5
    db = 20 * np.log10(np.maximum(mag, 1e-300))
    assert np.max(np.abs(db[f <= 0.9 * wun.KAISER_BEST_ROLLOFF * 0.5])) < 1e-5
    assert np.max(db[f >= 1.03 * 0.5]) < -140


def test_tone_round_trip():
    """A 1 kHz tone taken 44.1 -> 22.05 -> 44.1 kHz comes back to 1e-5 of its amplitude away from the edges."""
    t = np.arange(2 * 44100) / 44100.0
    x = (0.8 * np.sin(2 * np.pi * 1000 * t)).astype(np.float32)[:, None]
    down = oracle(x, 44100, 22050)
    assert down.shape == (44100, 1)
    back = oracle(down, 22050, 44100)[:x.shape[0]]
    edge = 2000
    assert np.max(np.abs(back[edge:-edge] - x[edge:-edge])) < 1e-5 * 0.8


def test_tone_above_new_nyquist_is_removed():
    t = np.arange(44100) / 44100.0
    x = np.stack([0.5 * np.sin(2 * np.pi * 15000 * t), 0.5 * np.cos(2 * np.pi * 15000 * t)], 1).astype(np.float32)
    y = oracle(x, 44100, 22050)
    edge = 1000
    assert np.max(np.abs(y[edge:-edge])) < 1e-6


@pytest.mark.parametrize("sr_in,sr_out", RATIOS)
def test_lengths_and_zero_padding(sr_in, sr_out):
    rng = np.random.default_rng(1)
    ratio = float(sr_out) / sr_in
    for n in (97, 1000, 4321):
        x = rng.standard_normal((n, 2)).astype(np.float32)
        y = oracle(x, sr_in, sr_out)
        n_valid, n_out = int(n * ratio), int(np.ceil(n * ratio))
        assert y.shape == (n_out, 2) and n_out == wun.resample_frames(n, sr_in, sr_out)
        assert np.all(y[n_valid:] == 0)
    assert ratio == 2 or any(int(n * ratio) < int(np.ceil(n * ratio)) for n in (97, 1000, 4321))


def test_equal_rates_and_short_inputs():
    x = np.ones((10, 2), np.float32)
    assert oracle(x, 22050, 22050) is x
    with pytest.raises(ValueError):
        oracle(x[:1], 44100, 22050)                                   # int(1 * 0.5) == 0
    with pytest.raises(ValueError):
        oracle(x[:5], 44100, 8192)                                    # int(5 * 0.1858) == 0
    assert oracle(x[:2], 44100, 22050).shape == (1, 2)
    assert wun.lib.wun_resample_frames(10, 0, 22050) == wun.WUN_E_INVALID
    assert wun.lib.wun_resample_frames(10, 44100, -1) == wun.WUN_E_INVALID


def test_cross_check_against_torchaudio():
    """torchaudio's kaiser-windowed sinc, built without a table, with the same zero crossings, rolloff and beta: on
    low-passed noise the two resamplers agree within 1e-5 in the interior, and shifting either by one sample breaks it."""
    torch = pytest.importorskip("torch")
    taf = pytest.importorskip("torchaudio.functional")
    rng = np.random.default_rng(5)
    n = 4 * 44100
    spec = np.fft.rfft(rng.standard_normal((2, n)), axis=1)
    spec[:, np.fft.rfftfreq(n, 1 / 44100.0) > 8000] = 0
    x = np.fft.irfft(spec, n, axis=1)
    x = (x * 0.18 / np.sqrt(np.mean(x ** 2))).astype(np.float32)
    want = taf.resample(torch.from_numpy(x).double(), 44100, 22050, lowpass_filter_width=64,
                        rolloff=wun.KAISER_BEST_ROLLOFF, resampling_method="sinc_interp_kaiser",
                        beta=wun.KAISER_BEST_BETA).numpy().T
    got = oracle(np.ascontiguousarray(x.T), 44100, 22050).astype(np.float64)
    assert got.shape == want.shape
    edge = 200
    inner = slice(edge, got.shape[0] - edge)
    assert np.max(np.abs(got[inner] - want[inner])) < 1e-5
    shifted = slice(edge + 1, got.shape[0] - edge + 1)
    assert np.max(np.abs(got[shifted] - want[inner])) > 1e-2
    assert np.max(np.abs(got[inner] - want[shifted])) > 1e-2


def test_wav_read_and_write(tmp_path):
    rng = np.random.default_rng(2)
    pcm = rng.integers(-32768, 32767, size=(1000, 2), dtype=np.int16)
    scipy.io.wavfile.write(str(tmp_path / "pcm.wav"), 44100, pcm)
    rate, audio = Predict.read_wav(str(tmp_path / "pcm.wav"))
    assert rate == 44100 and audio.dtype == np.float32 and audio.shape == (1000, 2)
    assert np.array_equal(audio, pcm.astype(np.float32) / 32768)
    scipy.io.wavfile.write(str(tmp_path / "mono.wav"), 8000, pcm[:, 0])
    rate, audio = Predict.read_wav(str(tmp_path / "mono.wav"))
    assert rate == 8000 and audio.shape == (1000, 1)
    flt = rng.standard_normal((500, 2)).astype(np.float32)
    scipy.io.wavfile.write(str(tmp_path / "f32.wav"), 22050, flt)
    rate, audio = Predict.read_wav(str(tmp_path / "f32.wav"))
    assert rate == 22050 and same_bits(audio, flt)
    for est in (flt, flt[:, :1].copy()):
        Predict.write_wav(str(tmp_path / "est.wav"), est, 44100)
        rate, back = Predict.read_wav(str(tmp_path / "est.wav"))
        assert rate == 44100 and same_bits(back, est)
    scipy.io.wavfile.write(str(tmp_path / "i32.wav"), 44100, pcm.astype(np.int32))
    with pytest.raises(ValueError, match="int32"):
        Predict.read_wav(str(tmp_path / "i32.wav"))
