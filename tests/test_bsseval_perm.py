"""museval's bss_eval switches without a GPU: the permutation search and the "sources" decomposition of the float64 oracle
(oracle/bsseval_perm_oracle.py) against direct projections and against the v4 / v3 oracles; the selection rule; the
Evaluate wrappers (bss_eval, bss_eval_sources / _images and their _framewise forms) with the device call replaced; and the
C ABI's argument checks for wun_bss_eval_ex."""
import ctypes

import numpy as np
import pytest

import Evaluate
import wun
from bsseval_cases import coloured, silent_case
from oracle import bsseval_oracle as B
from oracle import bsseval_perm_oracle as P
from oracle import bsseval_v3_oracle as V3

FRAMEWISE, PERMUTATION, SOURCES = wun.BSS_FRAMEWISE_FILTERS, wun.BSS_PERMUTATION, wun.BSS_SOURCES


def case(seed, nsrc, n, nchan, shuffle=None):
    """References and estimates; estimate j is mostly reference shuffle[j] (the identity by default)."""
    rng = np.random.default_rng(seed)
    ref = coloured(rng, nsrc, n, nchan)
    order = np.arange(nsrc) if shuffle is None else np.asarray(shuffle)
    est = (ref[order] + 0.3 * np.roll(ref, 1, axis=0)[order] + 0.1 * rng.standard_normal(ref.shape)).astype(np.float32)
    return ref, est


@pytest.mark.parametrize("sources_version", [False, True])
def test_pairs_equal_direct_projections(sources_version):
    nsrc, nchan, n = 2, 2, 2600
    ref, est = case(1, nsrc, n, nchan)
    pair, C, Cj = P.pairs(ref, est, n, n, sources_version=sources_version)
    G, _, basis = B.correlations_direct(ref, est)
    s = np.hstack((np.moveaxis(np.asarray(est, np.float64), 2, 1).reshape(nsrc * nchan, n), np.zeros((nsrc * nchan, B.L - 1))))
    m = nchan * B.L
    for je in range(nsrc):
        sj = s[je * nchan:(je + 1) * nchan]
        p_all = basis.T @ np.linalg.solve(G + B.EPS * np.eye(G.shape[0]), basis @ sj.T)
        for jt in range(nsrc):
            Bj = basis[jt * m:(jt + 1) * m]
            x = np.linalg.solve(Bj @ Bj.T + B.EPS * np.eye(m), Bj @ sj.T)
            assert np.allclose(x.T.reshape(nchan, nchan, B.L), Cj[jt, je], rtol=0, atol=1e-7 * np.abs(x).max())
            want = P.pair_metrics_from_projections(ref[jt].T.astype(np.float64), est[je].T.astype(np.float64),
                                                   (Bj.T @ x).T, p_all.T, sources_version)
            got = pair[:, jt, je, 0]
            assert np.array_equal(np.isnan(got), np.isnan(want))
            f = ~np.isnan(got)
            assert np.max(np.abs(got[f] - np.asarray(want)[f])) < 1e-7, (jt, je, got, want)
    if sources_version:
        assert np.all(np.isnan(pair[1]))


@pytest.mark.parametrize("framewise", [False, True])
def test_diagonal_equals_v4_and_v3_oracles_exactly(framewise):
    ref, est = case(2, 3, 5000, 2)
    win, hop = 2000, 1400
    want = (V3.bss_eval_v3 if framewise else B.bss_eval)(ref, est, win, hop)[0]
    images = P.pairs(ref, est, win, hop, framewise)[0]
    sources = P.pairs(ref, est, win, hop, framewise, sources_version=True)[0]
    diag = lambda x: np.stack([x[:, j, j] for j in range(3)], axis=1)   # noqa: E731
    assert np.array_equal(diag(images), want)
    assert np.array_equal(diag(sources)[2:], want[2:])                   # SIR and SAR
    assert np.all(np.isnan(sources[1]))
    assert not np.allclose(diag(sources)[0], want[0])                    # SDR: |P_j|^2 / |est - P_j|^2, not the image SDR
    m, popt, _ = P.bss_eval(ref, est, win, hop, framewise_filters=framewise)
    assert np.array_equal(m, want) and np.array_equal(popt, np.tile(np.arange(3)[:, None], (1, m.shape[2])))


@pytest.mark.parametrize("shuffle", [(2, 0, 1), (1, 0, 2), (0, 1, 2)])
def test_shuffled_estimates_give_the_shuffle(shuffle):
    ref, est = case(3, 3, 6000, 1, shuffle)
    for framewise in (False, True):
        m, popt, pair = P.bss_eval(ref, est, 2000, 2000, compute_permutation=True, framewise_filters=framewise)
        assert np.array_equal(popt, np.tile(np.asarray(shuffle)[:, None], (1, 3)))
        for j in range(3):
            assert np.array_equal(m[:, j], pair[:, shuffle[j], j])
        m0 = P.bss_eval(ref, est, 2000, 2000, framewise_filters=framewise)[0]
        if shuffle != (0, 1, 2):
            assert np.nanmean(m[2]) > np.nanmean(m0[2]) + 10                 # the identity scores far worse


def test_silent_frames_are_nan_with_the_identity():
    ref, est, win = silent_case()
    est = est[::-1].copy()                                               # estimate 0 is mostly reference 1
    m, popt, pair = P.bss_eval(ref, est, win, win, compute_permutation=True, framewise_filters=True)
    assert np.all(np.isnan(pair[:, :, :, [1, 3]])) and np.all(np.isnan(m[:, :, [1, 3]]))
    assert np.array_equal(popt[:, [1, 3]], [[0, 0], [1, 1]])
    assert np.array_equal(popt[:, [0, 2]], [[1, 1], [0, 0]])


def test_selection_rule():
    nsrc, nwin = 3, 4
    pair = np.zeros((4, nsrc, nsrc, nwin))
    pair[0] = np.arange(nsrc * nsrc * nwin).reshape(nsrc, nsrc, nwin)   # SDR tags each pair
    sir = pair[2]
    sir[:, :, 0] = 1.0                                                   # every candidate ties: the first (the identity)
    sir[:, :, 1] = [[0, 0, 5], [5, 0, 0], [0, 5, 0]]                     # pairs (1,0), (2,1), (0,2): candidate (1, 2, 0)
    sir[:, :, 2] = [[0, 0, 5], [5, 0, 0], [0, 5, 0]]
    sir[2, 2, 2] = np.nan                                                # a NaN mean wins: first candidate with jt=2 for j=2
    sir[:, :, 3] = [[np.inf, 0, 0], [0, -np.inf, 0], [0, 0, 0]]          # inf - inf: NaN for the identity and (0, 2, 1)...
    cands = [tuple(c) for c in P.candidates(nsrc)]
    assert cands == [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]
    m, popt = P.select(pair)
    assert list(popt[:, 0]) == [0, 1, 2] and list(popt[:, 1]) == [1, 2, 0]
    assert list(popt[:, 2]) == [0, 1, 2]                                 # (0, 1, 2) has sir[2, 2]: NaN, first
    assert list(popt[:, 3]) == [0, 1, 2]                                 # inf + -inf = NaN, first
    for j in range(nsrc):
        assert np.array_equal(m[0, j], pair[0, popt[j], j, np.arange(nwin)])
    m1, popt1 = P.select(pair, compute_permutation=False)
    assert np.array_equal(popt1, np.tile(np.arange(nsrc)[:, None], (1, nwin)))


def _oracle_device(calls):
    def fake(ref, est, win, hop, compute_permutation, framewise_filters, sources_version):
        calls.append(dict(shape=ref.shape, win=win, hop=hop, perm=compute_permutation, framewise=framewise_filters,
                          sources=sources_version))
        m, popt, _ = P.bss_eval(ref, est, win, hop, compute_permutation, framewise_filters, sources_version)
        return m, popt
    return fake


def test_bss_eval_sources_is_one_frame_of_the_framewise_form(monkeypatch):
    calls = []
    monkeypatch.setattr(Evaluate, "_device_bss_eval_ex", _oracle_device(calls))
    ref, est = case(4, 3, 3000, 1, (1, 2, 0))
    ref2, est2 = ref[:, :, 0], est[:, :, 0]                              # 2-D inputs
    whole = Evaluate.bss_eval_sources(ref2, est2)
    frames = Evaluate.bss_eval_sources_framewise(ref2, est2, window=3000, hop=3000, compute_permutation=True)
    assert len(whole) == 4 and all(x.shape == (3, 1) for x in whole)
    for a, b in zip(whole, frames):
        assert np.array_equal(a, b)
    assert list(whole[3][:, 0]) == [1, 2, 0]
    v4 = P.bss_eval(ref, est, 3000, 3000, compute_permutation=True, sources_version=True)[0]
    assert np.allclose(np.stack(whole[:3]), v4[[0, 2, 3]], rtol=1e-10, atol=0)
    assert calls[0] == dict(shape=(3, 3000, 1), win=3000, hop=3000, perm=True, framewise=True, sources=True)


def _shape_device(calls):
    def fake(ref, est, win, hop, compute_permutation, framewise_filters, sources_version):
        calls.append((win, hop, compute_permutation, framewise_filters, sources_version))
        nsrc, nwin = ref.shape[0], B.num_frames(ref.shape[1], win, hop)
        return np.zeros((4, nsrc, nwin)), np.tile(np.arange(nsrc)[:, None], (1, nwin))
    return fake


def test_evaluate_wrappers_shapes_and_defaults(monkeypatch):
    calls = []
    monkeypatch.setattr(Evaluate, "_device_bss_eval_ex", _shape_device(calls))
    rate, n = 44100, 61 * 44100
    ref = np.zeros((2, n, 2), np.float32)
    out = Evaluate.bss_eval_sources(ref, ref)
    assert len(out) == 4 and all(x.shape == (2, 1) for x in out)
    out = Evaluate.bss_eval_images(ref[:, :, 0], ref[:, :, 0], compute_permutation=False)
    assert len(out) == 5 and all(x.shape == (2, 1) for x in out)
    out = Evaluate.bss_eval_sources_framewise(ref, ref)
    assert len(out) == 4 and all(x.shape == (2, 3) for x in out)        # 30 s frames every 15 s over 61 s
    out = Evaluate.bss_eval_images_framewise(ref, ref, compute_permutation=True)
    assert len(out) == 5 and all(x.shape == (2, 3) for x in out)
    out = Evaluate.bss_eval(ref, ref)
    assert len(out) == 5 and all(x.shape == (2, 40) for x in out)       # museval's 2 s / 1.5 s default framing
    assert calls == [(n, n, True, True, True), (n, n, False, True, False), (30 * rate, 15 * rate, False, True, True),
                     (30 * rate, 15 * rate, True, True, False), (2 * rate, int(1.5 * rate), False, False, False)]
    with pytest.raises(ValueError, match="shape"):
        Evaluate.bss_eval(ref, ref[:, :-1])
    with pytest.raises(ValueError, match="filters_len"):
        Evaluate.bss_eval(ref, ref, filters_len=256)
    with pytest.raises(ValueError, match="nsrc"):
        Evaluate.bss_eval(ref[0, :, 0], ref[0, :, 0])


def test_wun_bss_eval_option_checks():
    with pytest.raises(ValueError, match="pair_metrics"):
        wun.bss_eval(None, None, 1000, 1000, pair_metrics=True)


def test_c_abi_workspace_sizes_ex():
    ws = wun.lib.wun_bss_eval_ex_workspace_bytes
    args = (4, 2, 44100 * 3, 44100, 44100)
    assert ws(*args, 0, 1) == wun.lib.wun_bss_eval_workspace_bytes(*args) == ws(*args, 0, 0) == ws(*args, SOURCES, 7) - \
        (ws(*args, SOURCES, 1) - ws(*args, 0, 1))
    for fpp in (1, 2, 3):
        assert ws(*args, FRAMEWISE, fpp) == wun.lib.wun_bss_eval_v3_workspace_bytes(*args, fpp)
    # the pairs: nsrc times the Cj columns, nsrc times the energies, and the pair metrics
    assert ws(*args, PERMUTATION, 1) - ws(*args, 0, 1) >= 8 * (3 * 8 * 1024 + 4 * 16 * 3)
    one, two = ws(*args, FRAMEWISE | PERMUTATION, 1), ws(*args, FRAMEWISE | PERMUTATION, 2)
    assert two - one == (ws(*args, FRAMEWISE, 2) - ws(*args, FRAMEWISE, 1)) + 8 * 3 * 8 * 1024
    for bad in [8, -1, 16 | PERMUTATION]:
        assert ws(*args, bad, 1) == wun.WUN_E_INVALID, bad
    assert ws(*args, FRAMEWISE, 0) == wun.WUN_E_INVALID
    assert ws(0, 2, 100, 10, 10, PERMUTATION, 1) == wun.WUN_E_INVALID


def test_c_abi_argument_checks_ex():
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    call = wun.lib.wun_bss_eval_ex
    for flags in (0, FRAMEWISE, PERMUTATION, FRAMEWISE | PERMUTATION | SOURCES):
        good = wun.lib.wun_bss_eval_ex_workspace_bytes(2, 1, 100, 10, 10, flags, 1)
        perm = p if flags & PERMUTATION else None
        assert call(p, p, 2, 1, 100, 10, 10, flags | 8, p, perm, None, None, p, good, None) == wun.WUN_E_INVALID
        assert call(p, p, 9, 1, 100, 10, 10, flags, p, perm, None, None, p, good, None) == wun.WUN_E_INVALID
        assert call(None, p, 2, 1, 100, 10, 10, flags, p, perm, None, None, p, good, None) == wun.WUN_E_INVALID
        assert call(p, p, 2, 1, 100, 10, 10, flags, None, perm, None, None, p, good, None) == wun.WUN_E_INVALID
        assert call(p, p, 2, 1, 100, 10, 10, flags, p, perm, None, None, p, good - 8, None) == wun.WUN_E_INVALID
        assert call(p, p, 2, 1, 100, 10, 10, flags, p, perm, None, None, None, good, None) == wun.WUN_E_INVALID
        if flags & PERMUTATION:                                          # perm is required when there are frames
            assert call(p, p, 2, 1, 100, 10, 10, flags, p, None, p, None, p, good, None) == wun.WUN_E_INVALID
        else:                                                            # and only written with the permutation search
            assert call(p, p, 2, 1, 100, 10, 10, flags, p, p, None, None, p, good, None) == wun.WUN_E_INVALID
            assert call(p, p, 2, 1, 100, 10, 10, flags, p, None, p, None, p, good, None) == wun.WUN_E_INVALID


def test_c_abi_ex_without_device_is_nogpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    for flags in (0, FRAMEWISE | PERMUTATION, PERMUTATION | SOURCES):
        good = wun.lib.wun_bss_eval_ex_workspace_bytes(2, 1, 100, 10, 10, flags, 1)
        buf = ctypes.create_string_buffer(good + 256)
        p = (ctypes.addressof(buf) + 255) // 256 * 256
        perm = p if flags & PERMUTATION else None
        assert wun.lib.wun_bss_eval_ex(p, p, 2, 1, 100, 10, 10, flags, p, perm, None, None, p, good, None) == wun.WUN_E_NOGPU
