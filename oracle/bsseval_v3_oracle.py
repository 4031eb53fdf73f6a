"""float64 restatement of BSS Eval v3 (museval 0.2.0 `evaluate(..., mode="v3")`): the decomposition of
oracle/bsseval_oracle.py with the 512-tap filters solved again for every frame, from that frame's samples only.  Built
from the v4 oracle's stages (correlations_fft, solve_filters, framewise / metrics_from_projections) applied per frame.

museval's mode="v3" is bss_eval(..., framewise_filters=True, compute_permutation=False, bsseval_sources_version=False)
(recalled, not run; DESIGN.md §4.12): G and the filters come from the frame slices, and only for frames that pass
_any_source_silent; Cj solves against the frame's G[j,j] (solve_filters).
"""
import numpy as np

from oracle.bsseval_oracle import (L, _any_source_silent, correlations_fft, framewise, num_frames, pad_or_truncate,
                                   solve_filters)


def frame_slices(ref, est, t, win, hop):
    """Frame t's slices [nsrc][win][nchan] of the references and the estimates."""
    return ref[:, t * hop:t * hop + win], est[:, t * hop:t * hop + win]


def frame_correlations(ref, est, t, win, hop, filters_len=L):
    """G and D of frame t: correlations_fft of its slices, which it zero-extends."""
    return correlations_fft(*frame_slices(np.asarray(ref), np.asarray(est), t, win, hop), filters_len)


def bss_eval_v3(ref, est, win, hop, filters_len=L):
    """The whole v3 evaluation: returns (metrics [4][nsrc][nwin], C [nwin][...], Cj [nwin][...]) with C and Cj of each
    frame in the layout of bsseval_oracle.solve_filters; silent frames are NaN in all three."""
    ref = np.asarray(ref, np.float64)
    est = pad_or_truncate(np.asarray(est, np.float64), ref.shape[1])
    nsrc, N, nchan = ref.shape
    nwin = num_frames(N, win, hop)
    out = np.full((4, nsrc, nwin), np.nan)
    C = np.full((nwin, nsrc, nchan, nsrc, nchan, filters_len), np.nan)
    Cj = np.full((nwin, nsrc, nchan, nchan, filters_len), np.nan)
    for t in range(nwin):
        r, s = frame_slices(ref, est, t, win, hop)
        if _any_source_silent(r) or _any_source_silent(s):
            continue
        G, D = correlations_fft(r, s, filters_len)
        C[t], Cj[t] = solve_filters(G, D, nsrc, nchan, filters_len)
        out[:, :, t] = framewise(r, s, C[t], Cj[t], win, win, filters_len)[:, :, 0]
    return out, C, Cj
