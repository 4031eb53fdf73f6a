"""BSS Eval v4 without a GPU: the float64 oracle (oracle/bsseval_oracle.py) against its own direct form and closed-form
cases, Evaluate's scenario / JSON / averaging logic with the device call replaced by the oracle, and the C ABI's
argument checks."""
import ctypes
import json

import numpy as np
import pytest

import Evaluate
import wun
from bsseval_cases import check_closed_forms, check_silent_case, coloured, silent_case
from oracle import bsseval_oracle as B


def rel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def oracle_score(ref, est, win, hop):
    return B.bss_eval(ref, est, win, hop)[0]


def test_fft_correlations_equal_direct_inner_products():
    rng = np.random.default_rng(0)
    ref = coloured(rng, 2, 3000, 2)
    est = (ref[::-1] * 0.5 + 0.1 * rng.standard_normal(ref.shape)).astype(np.float32)
    G, D = B.correlations_fft(ref, est)
    Gd, Dd, _ = B.correlations_direct(ref, est)
    assert rel(G, Gd) < 1e-13 and rel(D, Dd) < 1e-13


def test_whole_track_residual_is_orthogonal_to_delayed_references():
    rng = np.random.default_rng(1)
    ref = coloured(rng, 2, 6000, 2)
    est = (ref[0] + 0.4 * ref[1] + 0.2 * rng.standard_normal(ref.shape[1:])).astype(np.float32)[None].repeat(2, 0)
    G, D, basis = B.correlations_direct(ref, est)
    C, _ = B.solve_filters(G, D, 2, 2)
    spad = np.hstack((B._signals(est), np.zeros((4, B.L - 1))))
    for j in range(2):
        for e in range(2):
            resid = spad[j * 2 + e] - basis.T @ C[j, e].reshape(-1)
            assert np.max(np.abs(basis @ resid)) < 1e-9 * np.max(np.abs(D))


def test_closed_forms_oracle():
    check_closed_forms(lambda r, e, w, h: oracle_score(r, e, w, h))


def test_silent_frames_nan_and_zero_denominator_inf():
    ref, est, win = silent_case()
    check_silent_case(*oracle_score(ref, est, win, win))


@pytest.mark.parametrize("n,win,hop,want", [(10, 12, 5, 0), (12, 12, 5, 1), (16, 12, 5, 1), (17, 12, 5, 2),
                                            (100, 10, 10, 10), (109, 10, 10, 10), (5, 12, 1, 0)])
def test_number_of_frames_is_the_floor(n, win, hop, want):
    assert B.num_frames(n, win, hop) == want
    assert B.framewise(np.ones((1, n, 1)), np.ones((1, n, 1)), np.zeros((1, 1, 1, 1, B.L)),
                       np.zeros((1, 1, 1, B.L)), win, hop).shape == (4, 1, want)


def test_estimates_are_truncated_or_padded(monkeypatch):
    seen = []

    def fake(ref, est, win, hop):
        seen.append(est.copy())
        return np.stack(oracle_score(ref, est, win, hop))

    monkeypatch.setattr(Evaluate, "_device_bss_eval", fake)
    rng = np.random.default_rng(2)
    ref = rng.standard_normal((2, 5000, 1)).astype(np.float32)
    long_est = rng.standard_normal((2, 5300, 1)).astype(np.float32)
    sdr, isr, sir, sar = Evaluate.evaluate(ref, long_est, 2000, 1000)
    assert sdr.shape == (2, 4) and np.array_equal(seen[-1], long_est[:, :5000])
    Evaluate.evaluate(ref, long_est[:, :4200], 2000, 1000)
    assert seen[-1].shape == (2, 5000, 1) and not np.any(seen[-1][:, 4200:]) and np.array_equal(seen[-1][:, :4200], long_est[:, :4200])
    assert np.array_equal(B.pad_or_truncate(long_est[:, :4200], 5000), seen[-1])


def _fake_device(calls):
    def fake(ref, est, win, hop):
        calls.append(ref.shape[0])
        return np.stack(oracle_score(ref, est, win, hop))
    return fake


@pytest.mark.parametrize("names,scored,calls", [
    (["vocals", "accompaniment"], ["vocals", "accompaniment"], [2]),
    (["bass", "drums", "other", "vocals"], ["bass", "drums", "other", "vocals"], [4]),
    (["vocals", "accompaniment", "drums"], ["drums", "vocals", "accompaniment"], [2, 2]),
    (["vocals"], [], []),
    (["drums"], [], []),
])
def test_eval_track_scenarios_and_json(monkeypatch, tmp_path, names, scored, calls):
    seen = []
    monkeypatch.setattr(Evaluate, "_device_bss_eval", _fake_device(seen))
    rate = 1000
    rng = np.random.default_rng(3)
    refs = {n: rng.standard_normal((3 * rate + 100, 2)).astype(np.float32) for n in names}
    refs[names[0]][rate:2 * rate] = 0                              # a silent second: NaN frame
    ests = {n: (refs[n] + 0.1 * rng.standard_normal(refs[n].shape)).astype(np.float32)[:3 * rate + 50] for n in names}
    ests["unrelated"] = ests[names[0]]                             # only names in both dicts are scored
    scores = Evaluate.eval_track(refs, ests, rate, output_dir=str(tmp_path), track_name="song")
    assert seen == calls
    assert [t["name"] for t in scores["targets"]] == scored
    with open(tmp_path / "song.json") as f:
        js = json.load(f)
    assert js == json.loads(json.dumps(scores))
    for t in js["targets"]:
        assert len(t["frames"]) == 3
        assert [f["time"] for f in t["frames"]] == [0.0, 1.0, 2.0] and all(f["duration"] == 1.0 for f in t["frames"])
        assert sorted(t["frames"][0]["metrics"]) == ["ISR", "SAR", "SDR", "SIR"]
        assert all(np.isnan(v) for v in t["frames"][1]["metrics"].values())
        assert all(np.isfinite(v) for v in t["frames"][0]["metrics"].values())
    if scored:
        means = Evaluate.compute_mean_metrics(str(tmp_path), metric="SIR")
        frames = Evaluate.compute_mean_metrics(str(tmp_path), compute_averages=False, metric="SIR")
        assert len(means) == len(scored)
        for (med, mad, mean, sd), vals, t in zip(means, frames, js["targets"]):
            want = np.array([t["frames"][i]["metrics"]["SIR"] for i in (0, 2)])
            assert len(vals) == 3 and np.isnan(vals[1])
            assert np.isclose(med, np.median(want)) and np.isclose(mean, np.mean(want)) and np.isclose(sd, np.std(want))
            assert np.isclose(mad, np.median(np.abs(want - np.median(want))))


def test_c_abi_argument_checks():
    ws = wun.lib.wun_bss_eval_workspace_bytes
    assert ws(2, 2, 44100, 44100, 44100) > 0
    for bad in [(0, 2, 100, 10, 10), (9, 2, 100, 10, 10), (2, 3, 100, 10, 10), (2, 0, 100, 10, 10),
                (2, 2, 0, 10, 10), (2, 2, 100, 0, 10), (2, 2, 100, 10, 0)]:
        assert ws(*bad) == wun.WUN_E_INVALID, bad
    buf = ctypes.create_string_buffer(1024)
    p = ctypes.addressof(buf)
    good = ws(1, 1, 100, 10, 10)
    call = wun.lib.wun_bss_eval
    assert call(p, p, 0, 1, 100, 10, 10, p, None, p, good, None) == wun.WUN_E_INVALID
    assert call(p, p, 1, 2, 100, 10, 0, p, None, p, good, None) == wun.WUN_E_INVALID
    assert call(None, p, 1, 1, 100, 10, 10, p, None, p, good, None) == wun.WUN_E_INVALID
    assert call(p, p, 1, 1, 100, 10, 10, None, None, p, good, None) == wun.WUN_E_INVALID     # frames but no metrics
    assert call(p, p, 1, 1, 100, 10, 10, p, None, p, good - 8, None) == wun.WUN_E_INVALID    # workspace too small
    assert call(p, p, 1, 1, 100, 10, 10, p, None, None, good, None) == wun.WUN_E_INVALID


def test_c_abi_without_device_is_nogpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    good = wun.lib.wun_bss_eval_workspace_bytes(1, 1, 100, 10, 10)
    buf = ctypes.create_string_buffer(good + 256)
    p = (ctypes.addressof(buf) + 255) // 256 * 256
    assert wun.lib.wun_bss_eval(p, p, 1, 1, 100, 10, 10, p, None, p, good, None) == wun.WUN_E_NOGPU
