"""The closed-form cases of bsseval_cases.check_closed_forms under BSS Eval v3, shared by tests/test_bsseval_v3.py (oracle)
and tests/test_bsseval_v3_gpu.py (device).

Filters solved from one frame fit a share of any signal by chance, about taps / win of it: the single-source filter of
target j has nchan * L taps per estimate channel, so that share of the interference alpha r_k lands in P_j and SIR comes
out -10 log10(1 - nchan L / win) dB (0.10 dB at 1 s, stereo) above the energy ratio; the all-source filter has
nsrc * nchan * L taps, and SAR is above the input SNR by -10 log10(1 - nsrc nchan L / win) (0.21 dB).  v4 fits over the
whole track, where the share is small enough for the ratios themselves.  The first case is exact under both."""
import numpy as np

from bsseval_cases import RATE, frame_energy

L = 512


def check_closed_forms_v3(score, seconds=4, seed=0):
    rng = np.random.default_rng(seed)
    n, win, nchan = seconds * RATE, RATE, 2
    ref = rng.standard_normal((2, n, nchan)).astype(np.float32)

    g = np.array([0.5, 1.25], np.float32)
    sdr, isr, sir, sar = score(ref, (ref * g[:, None, None]).astype(np.float32), win, win)
    for j in range(2):
        want = -20 * np.log10(abs(float(g[j]) - 1))
        assert np.max(np.abs(isr[j] - want)) < 1e-6 and np.max(np.abs(sdr[j] - want)) < 1e-6, (j, isr[j], sdr[j], want)
        assert np.all(sir[j] > 150) and np.all(sar[j] > 150), (sir[j], sar[j])

    alpha = np.float32(0.3)
    est = np.stack([ref[0] + alpha * ref[1], ref[1] + alpha * ref[0]]).astype(np.float32)
    sdr, isr, sir, sar = score(ref, est, win, win)
    assert np.all(sar > 150), sar
    shift = -10 * np.log10(1 - nchan * L / win)
    for j, k in ((0, 1), (1, 0)):
        want = [10 * np.log10(frame_energy(ref[j], t, win) / (float(alpha) ** 2 * frame_energy(ref[k], t, win))) + shift
                for t in range(sir.shape[1])]
        assert np.max(np.abs(sir[j] - want)) < 0.05, (j, np.max(np.abs(sir[j] - want)))

    noise = (0.1 * rng.standard_normal(ref.shape)).astype(np.float32)
    sdr, isr, sir, sar = score(ref, (ref + noise).astype(np.float32), win, win)
    shift = -10 * np.log10(1 - 2 * nchan * L / win)
    for j in range(2):
        want = [10 * np.log10(frame_energy(ref[j], t, win) / frame_energy(noise[j], t, win)) + shift
                for t in range(sar.shape[1])]
        assert np.max(np.abs(sar[j] - want)) < 0.1, (j, np.max(np.abs(sar[j] - want)))
