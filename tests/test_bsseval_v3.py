"""BSS Eval v3 (museval mode="v3": the filters solved again for every frame) without a GPU: the float64 oracle
(oracle/bsseval_v3_oracle.py) against direct inner products, against v4 on a single frame, frame locality and the
closed-form cases; the `mode` / `bss_mode` plumbing of Evaluate and Predict with the device call replaced by the oracle;
and the C ABI's argument checks."""
import ctypes
import json

import numpy as np
import pytest

import Config
import Evaluate
import Predict
import wun
from bsseval_cases import check_silent_case, coloured, silent_case
from bsseval_v3_cases import check_closed_forms_v3
from oracle import bsseval_oracle as B
from oracle import bsseval_v3_oracle as V3


def rel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def case(seed, nsrc, n, nchan):
    rng = np.random.default_rng(seed)
    ref = coloured(rng, nsrc, n, nchan)
    est = (ref + 0.3 * np.roll(ref, 1, axis=0) + 0.1 * rng.standard_normal(ref.shape)).astype(np.float32)
    return ref, est


# overlapping frames, gaps between frames, and a ragged end (samples after the last frame)
@pytest.mark.parametrize("n,win,hop", [(2900, 1000, 600), (3500, 800, 1300), (2345, 1000, 1000)])
def test_frame_correlations_equal_direct_inner_products_of_the_slice(n, win, hop):
    ref, est = case(1, 2, n, 2)
    for t in range(B.num_frames(n, win, hop)):
        G, D = V3.frame_correlations(ref, est, t, win, hop)
        Gd, Dd, _ = B.correlations_direct(*V3.frame_slices(ref, est, t, win, hop))
        assert rel(G, Gd) < 1e-13 and rel(D, Dd) < 1e-13, t


@pytest.mark.parametrize("nsrc,nchan", [(2, 2), (3, 1)])
def test_one_frame_over_the_whole_track_equals_v4(nsrc, nchan):
    ref, est = case(2, nsrc, 6000, nchan)
    m3, C3, Cj3 = V3.bss_eval_v3(ref, est, 6000, 6000)
    m4, C4, Cj4 = B.bss_eval(ref, est, 6000, 6000)
    assert m3.shape == m4.shape == (4, nsrc, 1)
    assert rel(m3, m4) < 1e-12 and rel(C3[0], C4) < 1e-12 and rel(Cj3[0], Cj4) < 1e-12


def _sweep():
    rng = np.random.default_rng(3)
    cases = []
    for nsrc, nchan in [(1, 1), (1, 2), (2, 1), (2, 2), (3, 1), (3, 2), (4, 1), (4, 2)]:
        win = int(rng.integers(600, 1500))
        hop = int(rng.integers(win // 2, 3 * win // 2))
        cases.append((nsrc, nchan, win, hop))
    return cases


@pytest.mark.parametrize("nsrc,nchan,win,hop", _sweep())
def test_frame_locality(nsrc, nchan, win, hop):
    n = win + 2 * hop + 137                                             # three frames and a ragged end
    ref, est = case(4 + nsrc, nsrc, n, nchan)
    t = 1
    m3 = V3.bss_eval_v3(ref, est, win, hop)[0]
    m4 = B.bss_eval(ref, est, win, hop)[0]
    outside = np.ones(n, bool)
    outside[t * hop:t * hop + win] = False
    ref2, est2 = ref.copy(), est.copy()
    rng = np.random.default_rng(9)
    ref2[:, outside] += (0.5 * rng.standard_normal(ref2[:, outside].shape)).astype(np.float32)
    est2[:, outside] *= np.float32(-0.7)
    n3 = V3.bss_eval_v3(ref2, est2, win, hop)[0]
    n4 = B.bss_eval(ref2, est2, win, hop)[0]
    assert np.array_equal(m3[:, :, t], n3[:, :, t])
    assert not np.allclose(m4[:, :, t], n4[:, :, t], rtol=0, atol=1e-6)


def test_closed_forms_oracle_v3():
    check_closed_forms_v3(lambda r, e, w, h: V3.bss_eval_v3(r, e, w, h)[0])


def test_silent_frames_v3_nan_and_no_filters():
    ref, est, win = silent_case()
    m, C, Cj = V3.bss_eval_v3(ref, est, win, win)
    check_silent_case(*m)
    for t in (1, 3):
        assert np.all(np.isnan(C[t])) and np.all(np.isnan(Cj[t]))
    assert np.all(np.isfinite(C[[0, 2]])) and np.all(np.isfinite(Cj[[0, 2]]))


def _fake_device(calls):
    def fake(ref, est, win, hop, mode="v4"):
        calls.append(mode)
        return np.stack((V3.bss_eval_v3 if mode == "v3" else B.bss_eval)(ref, est, win, hop)[0])
    return fake


@pytest.mark.parametrize("mode", ["v4", "v3"])
def test_eval_track_mode_reaches_the_device_and_json_layout(monkeypatch, tmp_path, mode):
    seen = []
    monkeypatch.setattr(Evaluate, "_device_bss_eval", _fake_device(seen))
    rate = 1000
    rng = np.random.default_rng(5)
    refs = {n: rng.standard_normal((3 * rate + 100, 2)).astype(np.float32) for n in ("vocals", "accompaniment")}
    ests = {n: (refs[n] + 0.1 * rng.standard_normal(refs[n].shape)).astype(np.float32) for n in refs}
    scores = Evaluate.eval_track(refs, ests, rate, output_dir=str(tmp_path), track_name="song", mode=mode)
    assert seen == [mode]
    with open(tmp_path / "song.json") as f:
        js = json.load(f)
    assert js == json.loads(json.dumps(scores))
    assert [t["name"] for t in js["targets"]] == ["vocals", "accompaniment"]
    for t in js["targets"]:
        assert [f["time"] for f in t["frames"]] == [0.0, 1.0, 2.0]
        assert all(sorted(f) == ["duration", "metrics", "time"] for f in t["frames"])
        assert all(sorted(f["metrics"]) == ["ISR", "SAR", "SDR", "SIR"] for f in t["frames"])
    assert len(Evaluate.compute_mean_metrics(str(tmp_path), metric="SDR")) == 2


def test_evaluate_v3_scores_each_frame_alone(monkeypatch):
    monkeypatch.setattr(Evaluate, "_device_bss_eval", _fake_device([]))
    ref, est = case(6, 2, 3000, 2)
    got = np.stack(Evaluate.evaluate(ref, est[:, :2900], 1000, 1000, mode="v3"))
    assert np.array_equal(got, V3.bss_eval_v3(ref, B.pad_or_truncate(est[:, :2900], 3000), 1000, 1000)[0])


def test_unknown_mode_is_an_error(monkeypatch):
    monkeypatch.setattr(Evaluate, "_device_bss_eval", _fake_device([]))
    ref = np.ones((2, 3000, 1), np.float32)
    with pytest.raises(ValueError, match="mode"):
        Evaluate.evaluate(ref, ref, 1000, 1000, mode="v2")
    with pytest.raises(ValueError, match="mode"):
        Evaluate.eval_track({"vocals": ref[0]}, {"vocals": ref[0]}, 1000, mode="sources")
    with pytest.raises(ValueError, match="mode"):
        wun.bss_eval(None, None, 1000, 1000, mode="V3")


def test_predict_bss_mode_options():
    assert Predict.scoring_options() == (False, "v4")
    assert Predict.scoring_options("refs", "out") == (True, "v4")
    assert Predict.scoring_options("refs", "out", "v3") == (True, "v3")
    assert Predict.scoring_options("refs", "out", "V4") == (True, "v4")
    with pytest.raises(ValueError, match="bss_mode=v5"):
        Predict.scoring_options("refs", "out", "v5")
    for refs, out in ((None, None), ("refs", None), (None, "out")):
        with pytest.raises(ValueError, match="references_path"):
            Predict.scoring_options(refs, out, "v3")


def test_predict_main_passes_bss_mode(monkeypatch, tmp_path):
    cfg = Config.build_config(["baseline_stereo"], {}, experiment_id=0)
    rate = cfg["model_config"]["expected_sr"]
    rng = np.random.default_rng(7)
    mix = rng.standard_normal((3 * rate, 2)).astype(np.float32)
    np.save(tmp_path / "song.npy", mix)
    np.savez(tmp_path / "refs.npz", **{n: mix for n in cfg["model_config"]["source_names"]})
    monkeypatch.setattr(Evaluate, "produce_source_estimates",
                        lambda mc, path, m: {n: m for n in mc["source_names"]})
    seen = []
    monkeypatch.setattr(Evaluate, "eval_track", lambda *a, **k: seen.append(k["mode"]))
    Predict.main(cfg, None, str(tmp_path / "song.npy"), references_path=str(tmp_path / "refs.npz"),
                 results_dir=str(tmp_path / "res"), bss_mode="v3")
    Predict.main(cfg, None, str(tmp_path / "song.npy"), references_path=str(tmp_path / "refs.npz"),
                 results_dir=str(tmp_path / "res"))
    assert seen == ["v3", "v4"]
    with pytest.raises(ValueError, match="bss_mode"):
        Predict.main(cfg, None, str(tmp_path / "song.npy"), bss_mode="v3")


def test_c_abi_argument_checks_v3():
    ws = wun.lib.wun_bss_eval_v3_workspace_bytes
    one = ws(2, 2, 44100 * 3, 44100, 44100, 1)
    assert one > 0
    per_frame = ws(2, 2, 44100 * 3, 44100, 44100, 2) - one
    assert per_frame >= 8 * (2048 * 2048 + 2 * 1024 * 1024)            # G and the G[j,j] of one frame
    assert ws(2, 2, 44100 * 3, 44100, 44100, 3) == one + 2 * per_frame
    assert ws(2, 2, 44100 * 3, 44100, 44100, 50) == ws(2, 2, 44100 * 3, 44100, 44100, 3)   # never more than nwin
    for bad in [(0, 2, 100, 10, 10, 1), (9, 2, 100, 10, 10, 1), (2, 3, 100, 10, 10, 1), (2, 0, 100, 10, 10, 1),
                (2, 2, 0, 10, 10, 1), (2, 2, 100, 0, 10, 1), (2, 2, 100, 10, 0, 1), (2, 2, 100, 10, 10, 0)]:
        assert ws(*bad) == wun.WUN_E_INVALID, bad
    buf = ctypes.create_string_buffer(1024)
    p = ctypes.addressof(buf)
    good = ws(1, 1, 100, 10, 10, 1)
    call = wun.lib.wun_bss_eval_v3
    assert call(p, p, 0, 1, 100, 10, 10, p, None, p, good, None) == wun.WUN_E_INVALID
    assert call(p, p, 1, 2, 100, 10, 0, p, None, p, good, None) == wun.WUN_E_INVALID
    assert call(None, p, 1, 1, 100, 10, 10, p, None, p, good, None) == wun.WUN_E_INVALID
    assert call(p, p, 1, 1, 100, 10, 10, None, None, p, good, None) == wun.WUN_E_INVALID     # frames but no metrics
    assert call(p, p, 1, 1, 100, 10, 10, p, None, p, good - 8, None) == wun.WUN_E_INVALID    # not even one frame fits
    assert call(p, p, 1, 1, 100, 10, 10, p, None, None, good, None) == wun.WUN_E_INVALID


def test_c_abi_v3_without_device_is_nogpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    good = wun.lib.wun_bss_eval_v3_workspace_bytes(1, 1, 100, 10, 10, 1)
    buf = ctypes.create_string_buffer(good + 256)
    p = (ctypes.addressof(buf) + 255) // 256 * 256
    assert wun.lib.wun_bss_eval_v3(p, p, 1, 1, 100, 10, 10, p, None, p, good, None) == wun.WUN_E_NOGPU
