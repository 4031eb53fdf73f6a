"""museval's bss_eval switches on the GPU (wun_bss_eval_ex; wun.bss_eval(..., permutation=, sources_version=)) against the
float64 oracle (oracle/bsseval_perm_oracle.py): flags 0 and WUN_BSS_FRAMEWISE_FILTERS give wun_bss_eval's and
wun_bss_eval_v3's bits; pair metrics, selected metrics, the permutation and the filters on the framings of
test_bsseval_v3_gpu.py; permuted estimates; bits across repeats and frames per pass; 3-minute 4-source tracks."""
import numpy as np
import pytest
import torch

import Evaluate
import wun
from bsseval_cases import coloured, silent_case
from oracle import bsseval_perm_oracle as P
from oracle import bsseval_v3_oracle as V3

pytestmark = pytest.mark.gpu

FRAMINGS = [(2, 2, 24000, 8000, 4000), (3, 1, 26000, 6000, 9000), (1, 2, 20500, 8000, 8000), (4, 2, 30000, 12000, 9000)]


def case(seed, nsrc, nchan, n, shuffle=None):
    rng = np.random.default_rng(seed)
    ref = coloured(rng, nsrc, n, nchan)
    order = np.arange(nsrc) if shuffle is None else np.asarray(shuffle)
    est = (ref[order] + 0.3 * np.roll(ref, 1, axis=0)[order] + 0.1 * rng.standard_normal(ref.shape)).astype(np.float32)
    return ref, est


def gpu(ref, est, win, hop, **kw):
    out = wun.bss_eval(torch.from_numpy(np.ascontiguousarray(ref)).cuda(), torch.from_numpy(np.ascontiguousarray(est)).cuda(),
                       win, hop, **kw)
    return [t.cpu().numpy() for t in out]


def bits(x):
    return np.ascontiguousarray(x).view(np.uint64)


def max_db_diff(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isinf(a), np.isinf(b))
    f = np.isfinite(a)
    return float(np.max(np.abs(a[f] - b[f]))) if f.any() else 0.0


def rel_norm(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def legacy(ref, est, win, hop, v3):
    """metrics and filters from wun_bss_eval / wun_bss_eval_v3 called directly."""
    r, e = torch.from_numpy(ref).cuda(), torch.from_numpy(est).cuda()
    nsrc, n, nchan = ref.shape
    nwin = (n - win) // hop + 1
    if v3:
        nbytes = wun.lib.wun_bss_eval_v3_workspace_bytes(nsrc, nchan, n, win, hop, 2)
    else:
        nbytes = wun.lib.wun_bss_eval_workspace_bytes(nsrc, nchan, n, win, hop)
    metrics = torch.empty((4, nsrc, nwin), dtype=torch.float64, device="cuda")
    filt = torch.empty((nwin if v3 else 1) * nsrc * nchan * (nsrc * nchan + nchan) * 512, dtype=torch.float64, device="cuda")
    ws = torch.empty((nbytes + 255) // 256 * 32, dtype=torch.float64, device="cuda")
    call = wun.lib.wun_bss_eval_v3 if v3 else wun.lib.wun_bss_eval
    rc = call(r.data_ptr(), e.data_ptr(), nsrc, nchan, n, win, hop, metrics.data_ptr(), filt.data_ptr(), ws.data_ptr(),
              ws.numel() * 8, torch.cuda.current_stream().cuda_stream)
    assert rc == wun.WUN_OK
    return metrics.cpu().numpy(), filt.cpu().numpy()


@pytest.mark.parametrize("mode", ["v4", "v3"])
@pytest.mark.parametrize("nsrc,nchan,n,win,hop", [FRAMINGS[0], FRAMINGS[1]])
def test_flags_without_pairs_give_the_bits_of_the_existing_calls(mode, nsrc, nchan, n, win, hop):
    ref, est = case(20 + nsrc, nsrc, nchan, n)
    ref[0, win:win + hop] = 0                                            # a silent frame as well
    metrics, filt = legacy(ref, est, win, hop, mode == "v3")
    *got, C, Cj = gpu(ref, est, win, hop, filters=True, mode=mode, max_workspace_bytes=0)
    assert np.array_equal(bits(np.stack(got)), bits(metrics))
    lead = C.shape[0] if mode == "v3" else 1
    assert np.array_equal(bits(np.concatenate([C.reshape(lead, -1), Cj.reshape(lead, -1)], axis=1).ravel()), bits(filt))


@pytest.mark.parametrize("nsrc,nchan,n,win,hop", FRAMINGS)
@pytest.mark.parametrize("mode,sources_version", [("v4", False), ("v3", True)])
def test_pairs_selection_and_filters_match_oracle(nsrc, nchan, n, win, hop, mode, sources_version):
    shuffle = np.roll(np.arange(nsrc), 1)
    ref, est = case(10 + nsrc, nsrc, nchan, n, shuffle)
    want_pair, C, Cj = P.pairs(ref, est, win, hop, mode == "v3", sources_version)
    want, want_popt = P.select(want_pair)
    m = gpu(ref, est, win, hop, mode=mode, permutation=True, sources_version=sources_version, pair_metrics=True, filters=True)
    got, popt, pair, gC, gCj = np.stack(m[:4]), m[4], m[5], m[6], m[7]
    assert gC.shape == C.shape and gCj.shape == Cj.shape
    for t in range(C.shape[0] if mode == "v3" else 1):
        a, b = (gC[t], gCj[t]) if mode == "v3" else (gC, gCj)
        c, d = (C[t], Cj[t]) if mode == "v3" else (C, Cj)
        assert rel_norm(a, c) < 1e-8 and rel_norm(b, d) < 1e-8, (t, rel_norm(a, c), rel_norm(b, d))
    assert max_db_diff(pair, want_pair) < 1e-6
    assert np.array_equal(popt, want_popt) and np.array_equal(popt[:, 0], shuffle)
    assert max_db_diff(got, want) < 1e-6


def test_permuted_estimates_give_the_same_metrics():
    nsrc, nchan, n, win, hop = 4, 2, 30000, 12000, 9000
    tau = np.array([2, 0, 3, 1])
    ref, est = case(31, nsrc, nchan, n, tau)
    for mode in ("v4", "v3"):
        for sources_version in (False, True):
            base = gpu(ref, est, win, hop, mode=mode, permutation=True, sources_version=sources_version)
            assert np.array_equal(base[4], np.tile(tau[:, None], (1, base[4].shape[1])))
            for sigma in ([1, 0, 2, 3], [3, 2, 1, 0], [1, 2, 3, 0]):
                other = gpu(ref, np.ascontiguousarray(est[sigma]), win, hop, mode=mode, permutation=True,
                            sources_version=sources_version)
                for a, b in zip(other[:4], base[:4]):
                    assert np.array_equal(bits(a), bits(b[sigma]))
                assert np.array_equal(other[4], base[4][sigma])


def test_silent_frames_nan_with_the_identity_gpu():
    ref, est, win = silent_case()
    est = np.ascontiguousarray(est[::-1])
    for mode in ("v4", "v3"):
        got = gpu(ref, est, win, win, mode=mode, permutation=True)
        assert np.all(np.isnan(np.stack(got[:4])[:, :, [1, 3]]))
        assert np.array_equal(got[4], [[1, 0, 1, 0], [0, 1, 0, 1]])


def test_repeats_and_frames_per_pass_give_the_same_bits():
    ref, est = case(32, 3, 2, 40000, [1, 2, 0])
    ref[1, 8000:17000] = 0                                           # silent frames 2 and 3: fewer frames than slots
    runs = [gpu(ref, est, 5000, 4000, mode="v3", permutation=True, sources_version=s, pair_metrics=True, filters=True,
                max_workspace_bytes=b) for s in (False, True) for b in (0, 0, 1 << 40, 3 * 90 << 20)]
    assert runs[0][0].shape[1] == 9 and np.isnan(runs[0][0][:, 2:4]).all()
    for k in (0, 4):
        for other in runs[k + 1:k + 4]:
            for x, y in zip(runs[k], other):
                assert np.array_equal(bits(x), bits(y))
    again = gpu(ref, est, 5000, 4000, mode="v4", permutation=True, pair_metrics=True, filters=True)
    for x, y in zip(again, gpu(ref, est, 5000, 4000, mode="v4", permutation=True, pair_metrics=True, filters=True)):
        assert np.array_equal(bits(x), bits(y))


@pytest.mark.parametrize("sources_version", [False, True])
def test_full_size_four_sources_three_minutes_sampled_frames(sources_version):
    rng = np.random.default_rng(50)
    n, rate, nsrc = 7938000, 44100, 4
    tau = np.array([3, 1, 0, 2])
    ref = coloured(rng, nsrc, n, 2)
    ref[0, 10 * rate:12 * rate + 500] = 0                            # NaN frames 10 and 11
    est = (ref[tau] + 0.25 * np.roll(ref, 1, axis=0)[tau] + 0.05 * rng.standard_normal(ref.shape)).astype(np.float32)
    m = gpu(ref, est, rate, rate, mode="v3", permutation=True, sources_version=sources_version, pair_metrics=True)
    got, popt, pair = np.stack(m[:4]), m[4], m[5]
    assert got.shape == (4, nsrc, 180) and pair.shape == (4, nsrc, nsrc, 180)
    assert np.all(np.isnan(got[:, :, 10:12])) and np.array_equal(popt[:, 10], np.arange(nsrc))
    keep = np.delete(np.arange(180), [10, 11])
    assert np.array_equal(popt[:, keep], np.tile(tau[:, None], (1, keep.size)))
    for t in (0, 61, 179):
        r, e = V3.frame_slices(ref, est, t, rate, rate)
        want_pair = P.pairs(r, e, rate, rate, True, sources_version)[0]
        want, want_popt = P.select(want_pair)
        assert max_db_diff(pair[..., t], want_pair[..., 0]) < 1e-4, t
        assert max_db_diff(got[:, :, t], want[:, :, 0]) < 1e-4 and np.array_equal(popt[:, t], want_popt[:, 0]), t


def test_evaluate_wrappers_on_the_device():
    ref, est = case(33, 3, 1, 20000, [2, 0, 1])
    sdr, sir, sar, perm = Evaluate.bss_eval_sources(ref[:, :, 0], est[:, :, 0])
    assert sdr.shape == (3, 1) and list(perm[:, 0]) == [2, 0, 1]
    want, popt, _ = P.bss_eval(ref, est, 20000, 20000, compute_permutation=True, sources_version=True)
    assert max_db_diff(np.stack([sdr, sir, sar]), want[[0, 2, 3]]) < 1e-6 and np.array_equal(perm, popt)
    out = Evaluate.bss_eval_images_framewise(ref, est, window=8000, hop=6000)
    assert len(out) == 5 and out[0].shape == (3, 3) and np.array_equal(out[4], np.tile(np.arange(3)[:, None], (1, 3)))
