"""float64 restatement of museval 0.2.0's `bss_eval(reference_sources, estimated_sources, window, hop, compute_permutation,
filters_len=512, framewise_filters, bsseval_sources_version)`, the function behind museval.metrics' mir_eval-compatible
bss_eval_sources / bss_eval_images (and their _framewise forms), built from the stages of oracle/bsseval_oracle.py
(correlations_fft, solve_filters' systems, framewise / metrics_from_projections) and the frame slices of
oracle/bsseval_v3_oracle.py.

What this rests on (museval's code as recalled, not run; each point lives here and nowhere else in the oracle):

- Pairs.  With compute_permutation every (reference jtrue, estimate jest) pair is decomposed.  P_all of the pair is
  estimate jest projected on all references (C of estimate jest, the solve against G that v4 already does per estimate);
  P_j is estimate jest projected on reference jtrue alone: Cj solved against the diagonal block G[jtrue, jtrue] with the
  right-hand side D[rows of jtrue, columns of jest] (museval: `_bss_decomp_mtifilt(..., estimated_sources[jest], jtrue,
  C[jest], Cj[jtrue, jest])`).  pair_filters.
- Sources version (`_bss_crit(..., bsseval_sources_version=True)`): the same decomposition, s_filt = P_j;
  SDR = |P_j|^2 / |est - P_j|^2, SIR = |P_j|^2 / |P_all - P_j|^2, SAR = |P_all|^2 / |est - P_all|^2, ISR is NaN.  SIR and
  SAR are the images version's.  pair_metrics_from_projections.
- Selection (`mean_sir[i] = np.mean(sir[perm, dum, :], axis=0)`, `popt = candidates[argmax(mean_sir, axis=0)].T`,
  `sdr[popt, dum, t]` with the pair arrays indexed [jtrue, jest]): the candidates are itertools.permutations(range(nsrc))
  in that order; candidate `perm` pairs estimate j with reference perm[j].  So the returned row j is ESTIMATE j, scored
  against reference popt[j, t]; a frame's mean adds the nsrc pair SIRs in estimate order (numpy adds the rows of an
  axis-0 reduction one after another) and divides by nsrc; argmax takes the first maximum, or the first NaN if there is
  one, so a silent frame (all NaN) keeps the identity.  Without compute_permutation the identity is the only candidate.
  select.
- Silence: the frames _any_source_silent rejects are NaN for every pair and get no filters (v3), as in the oracles above.
"""
import itertools

import numpy as np

from oracle.bsseval_oracle import (EPS, L, _any_source_silent, _safe_db, correlations_fft, metrics_from_projections,
                                   num_frames, solve_filters)
from oracle.bsseval_v3_oracle import frame_slices


def pair_filters(G, D, nsrc, nchan, filters_len=L):
    """C [jest][e][k][c][l] as solve_filters, and Cj [jtrue][jest][e][c][l] = (G[jtrue,jtrue] + eps I)^-1 D[jtrue rows,
    jest columns].  Each (jtrue, jest) is its own solve with nchan right-hand sides, the shape solve_filters uses for the
    diagonal, so Cj[j][j] equals solve_filters' Cj[j] bit for bit."""
    C, _ = solve_filters(G, D, nsrc, nchan, filters_len)
    m = nchan * filters_len
    Cj = np.zeros((nsrc, nsrc, nchan, nchan, filters_len))
    for jt in range(nsrc):
        blk = slice(jt * m, (jt + 1) * m)
        A = G[blk, blk] + EPS * np.eye(m)
        for je in range(nsrc):
            Xj = np.linalg.solve(A, D[blk, je * nchan:(je + 1) * nchan])
            Cj[jt, je] = Xj.T.reshape(nchan, nchan, filters_len)
    return C, Cj


def pair_metrics_from_projections(r_j, s_j, p_j, p_all, sources_version, filters_len=L):
    """(SDR, ISR, SIR, SAR) of one frame and pair; the images version is metrics_from_projections."""
    sdr, isr, sir, sar = metrics_from_projections(r_j, s_j, p_j, p_all, filters_len)
    if sources_version:
        s = np.pad(s_j, ((0, 0), (0, filters_len - 1)))
        sdr, isr = _safe_db(np.sum(p_j ** 2), np.sum((s - p_j) ** 2)), np.nan
    return sdr, isr, sir, sar


def framewise_pairs(ref, est, C, Cj, win, hop, sources_version=False, filters_len=L):
    """pair metrics [4][nsrc (jtrue)][nsrc (jest)][nwin] from given filters (pair_filters' layout), computed as
    bsseval_oracle.framewise computes its diagonal."""
    ref = np.asarray(ref, np.float64)
    est = np.asarray(est, np.float64)
    nsrc, N, nchan = ref.shape
    nwin, W = num_frames(N, win, hop), win + filters_len - 1
    nfft = int(2 ** np.ceil(np.log2(W)))
    Hf = np.fft.rfft(C.reshape(nsrc, nchan, nsrc * nchan, filters_len), n=nfft)      # [jest, e, (k, c), F]
    Hjf = np.fft.rfft(Cj, n=nfft)                                                     # [jtrue, jest, e, c, F]
    out = np.full((4, nsrc, nsrc, nwin), np.nan)
    for t in range(nwin):
        r, s = ref[:, t * hop:t * hop + win], est[:, t * hop:t * hop + win]
        if _any_source_silent(r) or _any_source_silent(s):
            continue
        Xf = np.fft.rfft(np.moveaxis(r, 2, 1), n=nfft)                                # [k, c, F]
        p_all = np.fft.irfft(np.einsum("jeaf,af->jef", Hf, Xf.reshape(nsrc * nchan, -1)), n=nfft)[..., :W]
        for jt in range(nsrc):
            for je in range(nsrc):
                p_j = np.fft.irfft(np.einsum("ecf,cf->ef", Hjf[jt, je], Xf[jt]), n=nfft)[:, :W]
                out[:, jt, je, t] = pair_metrics_from_projections(r[jt].T, s[je].T, p_j, p_all[je], sources_version,
                                                                  filters_len)
    return out


def pairs(ref, est, win, hop, framewise_filters=False, sources_version=False, filters_len=L):
    """The pair stage: (pair metrics [4][nsrc (jtrue)][nsrc (jest)][nwin], C, Cj).  Filters over the whole track (v4), or
    per frame (framewise_filters, v3: leading [nwin] axis, NaN for silent frames)."""
    ref = np.asarray(ref, np.float64)
    est = np.asarray(est, np.float64)
    nsrc, N, nchan = ref.shape
    if not framewise_filters:
        G, D = correlations_fft(ref, est, filters_len)
        C, Cj = pair_filters(G, D, nsrc, nchan, filters_len)
        return framewise_pairs(ref, est, C, Cj, win, hop, sources_version, filters_len), C, Cj
    nwin = num_frames(N, win, hop)
    out = np.full((4, nsrc, nsrc, nwin), np.nan)
    C = np.full((nwin, nsrc, nchan, nsrc, nchan, filters_len), np.nan)
    Cj = np.full((nwin, nsrc, nsrc, nchan, nchan, filters_len), np.nan)
    for t in range(nwin):
        r, s = frame_slices(ref, est, t, win, hop)
        if _any_source_silent(r) or _any_source_silent(s):
            continue
        G, D = correlations_fft(r, s, filters_len)
        C[t], Cj[t] = pair_filters(G, D, nsrc, nchan, filters_len)
        out[..., t] = framewise_pairs(r, s, C[t], Cj[t], win, win, sources_version, filters_len)[..., 0]
    return out, C, Cj


def candidates(nsrc, compute_permutation=True):
    """The candidate permutations [ncand][nsrc], in itertools order (the identity alone without compute_permutation)."""
    if not compute_permutation:
        return np.arange(nsrc)[None, :]
    return np.array(list(itertools.permutations(range(nsrc))))


def mean_sir(pair, compute_permutation=True):
    """[ncand][nwin]: per candidate perm, sum over estimates j in order of SIR(jtrue = perm[j], jest = j), over nsrc."""
    sir = pair[2]
    nsrc = sir.shape[0]
    out = []
    for perm in candidates(nsrc, compute_permutation):
        s = sir[perm[0], 0]
        for j in range(1, nsrc):
            s = s + sir[perm[j], j]
        out.append(s / nsrc)
    return np.array(out)


def select(pair, compute_permutation=True):
    """The selection stage: (metrics [4][nsrc][nwin], popt int64 [nsrc][nwin]); row j is estimate j, scored against
    reference popt[j, t]."""
    nsrc, nwin = pair.shape[1], pair.shape[3]
    cand = candidates(nsrc, compute_permutation)
    popt = cand[np.argmax(mean_sir(pair, compute_permutation), axis=0)].T.astype(np.int64)
    return pair[:, popt, np.arange(nsrc)[:, None], np.arange(nwin)[None, :]], popt


def bss_eval(ref, est, win, hop, compute_permutation=False, framewise_filters=False, sources_version=False,
             filters_len=L):
    """museval's bss_eval on arrays [nsrc][nsampl][nchan] of equal shape: (metrics [4 (SDR, ISR, SIR, SAR)][nsrc][nwin],
    popt [nsrc][nwin], pair metrics [4][nsrc][nsrc][nwin]).  The pairs are all computed either way; without
    compute_permutation only the diagonal is read."""
    pair = pairs(ref, est, win, hop, framewise_filters, sources_version, filters_len)[0]
    metrics, popt = select(pair, compute_permutation)
    return metrics, popt, pair
