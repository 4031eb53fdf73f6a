"""Inputs and closed-form checks shared by the BSS Eval tests (tests/test_bsseval.py on the oracle,
tests/test_bsseval_gpu.py on the device)."""
import numpy as np
import scipy.signal

RATE = 44100


def coloured(rng, nsrc, n, nchan, order=4):
    """Independent coloured noise [nsrc, n, nchan] (a random all-pole filter per signal), float32."""
    x = rng.standard_normal((nsrc, n, nchan))
    for k in range(nsrc):
        for c in range(nchan):
            poles = 0.6 * rng.uniform(0.2, 1.0, order // 2) * np.exp(1j * rng.uniform(0.3, 2.8, order // 2))
            a = np.real(np.poly(np.concatenate([poles, np.conj(poles)])))
            x[k, :, c] = scipy.signal.lfilter([1.0], a, x[k, :, c])
    return (x / np.std(x)).astype(np.float32)


def ill_conditioned(rng, nsrc, n, nchan):
    """Low-passed references, source 0 with equal left and right channels: G is singular up to rounding."""
    b, a = scipy.signal.butter(8, 0.25)
    x = scipy.signal.lfilter(b, a, rng.standard_normal((nsrc, n, nchan)), axis=1)
    x[0, :, 1] = x[0, :, 0]
    ref = (x / np.std(x)).astype(np.float32)
    est = (ref + 0.3 * np.roll(ref, 1, axis=0) + 0.2 * rng.standard_normal(ref.shape)).astype(np.float32)
    return ref, est


def frame_energy(x, t, win):
    """sum over the frame's samples and channels of x^2, x [n, nchan]."""
    return float(np.sum(np.asarray(x[t * win:(t + 1) * win], np.float64) ** 2))


def check_closed_forms(score, seconds=20, seed=0):
    """Runs score(ref, est, win, hop) -> (SDR, ISR, SIR, SAR) [nsrc, nwin] on white-noise cases with known answers."""
    rng = np.random.default_rng(seed)
    n, win = seconds * RATE, RATE
    ref = rng.standard_normal((2, n, 2)).astype(np.float32)

    # est_j = g_j r_j: the filters are exact (g at lag 0); SDR = ISR = -20 log10 |g - 1| (image definition)
    g = np.array([0.5, 1.25], np.float32)
    est = (ref * g[:, None, None]).astype(np.float32)
    sdr, isr, sir, sar = score(ref, est, win, win)
    for j in range(2):
        want = -20 * np.log10(abs(float(g[j]) - 1))
        assert np.max(np.abs(isr[j] - want)) < 1e-6, (j, isr[j], want)
        assert np.max(np.abs(sdr[j] - want)) < 1e-6, (j, sdr[j], want)
        assert np.all(sir[j] > 150) and np.all(sar[j] > 150), (sir[j], sar[j])

    # est_j = r_j + alpha r_k: no artifacts, SIR = energy ratio (up to the part of r_k the single-source filter fits)
    alpha = np.float32(0.3)
    est = np.stack([ref[0] + alpha * ref[1], ref[1] + alpha * ref[0]]).astype(np.float32)
    sdr, isr, sir, sar = score(ref, est, win, win)
    assert np.all(sar > 150), sar
    for j, k in ((0, 1), (1, 0)):
        want = [10 * np.log10(frame_energy(ref[j], t, win) / (float(alpha) ** 2 * frame_energy(ref[k], t, win)))
                for t in range(sir.shape[1])]
        assert np.max(np.abs(sir[j] - want)) < 0.05, (j, np.max(np.abs(sir[j] - want)))

    # est_j = r_j + independent noise: SAR = the frame's input SNR
    noise = (0.1 * rng.standard_normal(ref.shape)).astype(np.float32)
    est = (ref + noise).astype(np.float32)
    sdr, isr, sir, sar = score(ref, est, win, win)
    for j in range(2):
        want = [10 * np.log10(frame_energy(ref[j], t, win) / frame_energy(noise[j], t, win)) for t in range(sar.shape[1])]
        assert np.max(np.abs(sar[j] - want)) < 0.1, (j, np.max(np.abs(sar[j] - want)))


def silent_case():
    """Short stereo case with a silent second-frame stretch in reference 1 and estimate 0 equal to reference 0."""
    rng = np.random.default_rng(5)
    win = 2000
    ref = rng.standard_normal((2, 4 * win + 700, 2)).astype(np.float32)
    ref[1, win:2 * win] = 0.0                                        # frame 1: a silent reference -> NaN for every target
    ref[1, 3 * win:4 * win, 1] = -ref[1, 3 * win:4 * win, 0]         # frame 3: channels cancel -> silent as well
    est = ref.copy()
    est[1] += 0.1 * rng.standard_normal(est[1].shape).astype(np.float32)
    est[1, win:2 * win] += 0.5                                       # estimate not silent where the reference is
    return ref, est, win


def check_silent_case(sdr, isr, sir, sar):
    for m in (sdr, isr, sir, sar):
        assert m.shape == (2, 4)
        assert np.all(np.isnan(m[:, 1])) and np.all(np.isnan(m[:, 3]))
        assert not np.any(np.isnan(m[:, [0, 2]]))
    assert np.all(np.isposinf(sdr[0, [0, 2]]))                        # est_0 == r_0: |est - r_0|^2 == 0
    assert np.all(np.isfinite(sdr[1, [0, 2]]))
