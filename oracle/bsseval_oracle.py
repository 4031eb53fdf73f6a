"""float64 restatement of BSS Eval v4 (museval 0.2.0 `evaluate(..., mode="v4")`: the "images" decomposition with
512-tap filters solved once over the whole track and applied frame by frame), in stages that the GPU tests can enter
separately.  museval itself is not run here; see DESIGN.md §5 for what this restatement rests on.

Layouts follow include/wun.h: signals [nsrc][N][nchan]; Gram matrix and right-hand sides indexed by (source k, channel c,
delay l); filters C[j][e][k][c][l] for target j and estimate channel e, and Cj[j][e][c][l] for source j alone.
"""
import numpy as np
import scipy.linalg

L = 512
EPS = np.finfo(np.float64).eps       # museval adds numpy's float eps to the Gram matrix' diagonal


def _signals(x):
    """[nsrc][N][nchan] -> [nsrc*nchan][N] float64, rows (k, c)."""
    x = np.asarray(x, np.float64)
    return np.moveaxis(x, 2, 1).reshape(-1, x.shape[1])


def correlations_fft(ref, est, filters_len=L):
    """G [n, n] and D [n, nsrc*nchan] (n = nsrc*nchan*L) from FFT cross-correlations and Toeplitz blocks, the way museval's
    _compute_reference_correlations / _compute_projection_filters build them.  D's column (j, e) is estimate j, channel e."""
    r, s = _signals(ref), _signals(est)
    nref, N = r.shape
    nfft = int(2 ** np.ceil(np.log2(N + filters_len - 1)))
    rf, sf = np.fft.rfft(r, n=nfft), np.fft.rfft(s, n=nfft)
    G = np.zeros((nref, filters_len, nref, filters_len))
    for a in range(nref):
        for b in range(a, nref):
            cc = np.fft.irfft(rf[b] * np.conj(rf[a]), n=nfft)      # cc[tau] = sum_m r_a[m] r_b[m + tau]
            blk = scipy.linalg.toeplitz(np.hstack((cc[0], cc[-1:-filters_len:-1])), r=cc[:filters_len])
            G[b, :, a, :] = blk
            G[a, :, b, :] = blk.T
    D = np.zeros((nref, filters_len, s.shape[0]))
    for a in range(nref):
        for col in range(s.shape[0]):
            cc = np.fft.irfft(rf[a] * np.conj(sf[col]), n=nfft)     # cc[-l] = sum_m r_a[m] est[m + l]
            D[a, :, col] = np.hstack((cc[0], cc[-1:-filters_len:-1]))
    n = nref * filters_len
    return G.reshape(n, n), D.reshape(n, -1)


def correlations_direct(ref, est, filters_len=L):
    """The same G and D as plain inner products of delayed copies S_p x (zero-extended to N + L - 1): small N only."""
    r, s = _signals(ref), _signals(est)
    nref, N = r.shape
    basis = np.zeros((nref * filters_len, N + filters_len - 1))
    for a in range(nref):
        for p in range(filters_len):
            basis[a * filters_len + p, p:p + N] = r[a]
    spad = np.hstack((s, np.zeros((s.shape[0], filters_len - 1))))
    return basis @ basis.T, basis @ spad.T, basis


def solve_filters(G, D, nsrc, nchan, filters_len=L):
    """C_j = (G + eps I)^-1 D_j for every j, and Cj_j = (G[j,j] + eps I)^-1 D_j[j] against source j's diagonal block."""
    n, m = G.shape[0], nchan * filters_len
    X = np.linalg.solve(G + EPS * np.eye(n), D)
    C = X.T.reshape(nsrc, nchan, nsrc, nchan, filters_len)
    Cj = np.zeros((nsrc, nchan, nchan, filters_len))
    for j in range(nsrc):
        blk = slice(j * m, (j + 1) * m)
        Xj = np.linalg.solve(G[blk, blk] + EPS * np.eye(m), D[blk, j * nchan:(j + 1) * nchan])
        Cj[j] = Xj.T.reshape(nchan, nchan, filters_len)
    return C, Cj


def num_frames(N, win, hop):
    return max(0, (N - win + hop) // hop)


def _safe_db(num, den):
    if den == 0:
        return np.inf
    with np.errstate(divide="ignore"):          # a zero numerator is -inf dB
        return 10 * np.log10(num / den)


def _any_source_silent(x):
    """x [nsrc][win][nchan]: some source has sum_c x[n][c] == 0 for every n (museval's _any_source_silent)."""
    return bool(np.any(np.all(np.sum(x, axis=2) == 0, axis=1)))


def framewise(ref, est, C, Cj, win, hop, filters_len=L):
    """metrics [4 (SDR, ISR, SIR, SAR)][nsrc][nwin] from given filters: each frame's slices, zero-extended to
    W = win + L - 1, are filtered into P_all (all sources, C) and P_j (source j, Cj)."""
    ref = np.asarray(ref, np.float64)
    est = np.asarray(est, np.float64)
    nsrc, N, nchan = ref.shape
    nwin, W = num_frames(N, win, hop), win + filters_len - 1
    nfft = int(2 ** np.ceil(np.log2(W)))
    Hf = np.fft.rfft(C.reshape(nsrc, nchan, nsrc * nchan, filters_len), n=nfft)      # [j, e, (k, c), F]
    Hjf = np.fft.rfft(Cj, n=nfft)                                                     # [j, e, c, F]
    out = np.full((4, nsrc, nwin), np.nan)
    for t in range(nwin):
        r, s = ref[:, t * hop:t * hop + win], est[:, t * hop:t * hop + win]
        if _any_source_silent(r) or _any_source_silent(s):
            continue
        Xf = np.fft.rfft(np.moveaxis(r, 2, 1), n=nfft)                                # [k, c, F]
        p_all = np.fft.irfft(np.einsum("jeaf,af->jef", Hf, Xf.reshape(nsrc * nchan, -1)), n=nfft)[..., :W]
        for j in range(nsrc):
            p_j = np.fft.irfft(np.einsum("ecf,cf->ef", Hjf[j], Xf[j]), n=nfft)[:, :W]
            out[:, j, t] = metrics_from_projections(r[j].T, s[j].T, p_j, p_all[j], filters_len)
    return out


def metrics_from_projections(r_j, s_j, p_j, p_all, filters_len=L):
    """(SDR, ISR, SIR, SAR) of one frame and target from s_true = r_j, e_spat = P_j - r_j, e_interf = P_all - P_j and
    e_artif = est - P_all (museval's _bss_decomp_mtifilt + _bss_crit, images version).  r_j, s_j [nchan][win]."""
    pad = ((0, 0), (0, filters_len - 1))
    r, s = np.pad(r_j, pad), np.pad(s_j, pad)
    e_true = np.sum(r ** 2)
    sdr = _safe_db(e_true, np.sum((s - r) ** 2))
    isr = _safe_db(e_true, np.sum((p_j - r) ** 2))
    sir = _safe_db(np.sum(p_j ** 2), np.sum((p_all - p_j) ** 2))
    sar = _safe_db(np.sum(p_all ** 2), np.sum((s - p_all) ** 2))
    return sdr, isr, sir, sar


def pad_or_truncate(est, N):
    """museval padding=True: estimates cut or zero-extended to the references' length."""
    est = np.asarray(est)
    if est.shape[1] >= N:
        return est[:, :N]
    return np.pad(est, ((0, 0), (0, N - est.shape[1]), (0, 0)))


def bss_eval(ref, est, win, hop, filters_len=L):
    """The whole v4 evaluation: returns (metrics [4][nsrc][nwin], C, Cj)."""
    ref = np.asarray(ref, np.float64)
    est = pad_or_truncate(np.asarray(est, np.float64), ref.shape[1])
    nsrc, _, nchan = ref.shape
    G, D = correlations_fft(ref, est, filters_len)
    C, Cj = solve_filters(G, D, nsrc, nchan, filters_len)
    return framewise(ref, est, C, Cj, win, hop, filters_len), C, Cj
