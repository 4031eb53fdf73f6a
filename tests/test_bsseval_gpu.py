"""BSS Eval v4 on the GPU (wun.bss_eval, csrc/kernels_bsseval.cu) against the float64 oracle (oracle/bsseval_oracle.py),
stage by stage: the filters against the oracle's solve, the framewise stage fed the GPU's own filters, and whole calls."""
import os

import numpy as np
import pytest
import torch

import Config
import Evaluate
import Predict
import Training
import wun
from Models.UnetAudioSeparator import UnetAudioSeparator
from bsseval_cases import check_closed_forms, check_silent_case, coloured, ill_conditioned, silent_case
from oracle import bsseval_oracle as B
from oracle import wave_unet_oracle as O

pytestmark = pytest.mark.gpu


def gpu(ref, est, win, hop, filters=False):
    out = wun.bss_eval(torch.from_numpy(np.ascontiguousarray(ref)).cuda(), torch.from_numpy(np.ascontiguousarray(est)).cuda(),
                       win, hop, filters=filters)
    return [t.cpu().numpy() for t in out]


def max_db_diff(a, b):
    """max |a - b| over frames finite in both; the NaN / inf patterns must agree."""
    a, b = np.asarray(a), np.asarray(b)
    assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isinf(a), np.isinf(b))
    f = np.isfinite(a)
    return float(np.max(np.abs(a[f] - b[f]))) if f.any() else 0.0


def rel_norm(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def coloured_case(seed, nsrc, nchan, seconds, rate=8000):
    rng = np.random.default_rng(seed)
    ref = coloured(rng, nsrc, seconds * rate, nchan)
    mix = np.roll(ref, 1, axis=0)
    est = (ref + 0.3 * mix + 0.1 * rng.standard_normal(ref.shape)).astype(np.float32)
    return ref, est, rate


@pytest.mark.parametrize("nsrc,nchan,seconds", [(2, 2, 6), (3, 1, 5), (8, 1, 2)])
def test_filters_and_metrics_match_oracle(nsrc, nchan, seconds):
    ref, est, rate = coloured_case(10 + nsrc, nsrc, nchan, seconds)
    G, D = B.correlations_fft(ref, est)
    cond = np.linalg.cond(G)
    assert cond < 1e6, cond
    C, Cj = B.solve_filters(G, D, nsrc, nchan)
    want = B.framewise(ref, est, C, Cj, rate, rate // 2)
    *got, gC, gCj = gpu(ref, est, rate, rate // 2, filters=True)
    assert gC.shape == C.shape and gCj.shape == Cj.shape
    assert rel_norm(gC, C) < 1e-8 and rel_norm(gCj, Cj) < 1e-8, (rel_norm(gC, C), rel_norm(gCj, Cj))
    assert max_db_diff(np.stack(got), want) < 1e-6
    # the framewise stage alone: the oracle fed the GPU's filters
    assert max_db_diff(np.stack(got), B.framewise(ref, est, gC, gCj, rate, rate // 2)) < 1e-9


def test_framewise_stage_ill_conditioned():
    rng = np.random.default_rng(20)
    ref, est = ill_conditioned(rng, 2, 5 * 8000, 2)
    *got, gC, gCj = gpu(ref, est, 8000, 8000, filters=True)
    assert np.max(np.abs(gC)) > 1e3                                  # the filters are large and not unique here
    assert max_db_diff(np.stack(got), B.framewise(ref, est, gC, gCj, 8000, 8000)) < 1e-6


def test_closed_forms_gpu():
    check_closed_forms(lambda r, e, w, h: gpu(r, e, w, h))


def test_silent_frames_gpu():
    ref, est, win = silent_case()
    got = gpu(ref, est, win, win)
    check_silent_case(*got)
    got, want = np.stack(got), B.bss_eval(ref, est, win, win)[0]
    exact = (got > 150) & (want > 150)          # est_0 == r_0: rounding sets the value of these, not the algorithm
    assert max_db_diff(np.where(exact, 0, got), np.where(exact, 0, want)) < 1e-6


def test_two_calls_same_bits():
    ref, est, rate = coloured_case(30, 3, 2, 3)
    a = gpu(ref, est, rate, rate // 4, filters=True)
    b = gpu(ref, est, rate, rate // 4, filters=True)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint64), y.view(np.uint64))


@pytest.mark.parametrize("nsrc", [2, 4])
def test_full_size_three_minutes(nsrc):
    rng = np.random.default_rng(40 + nsrc)
    n = 7938000                                                      # 3 minutes at 44.1 kHz (predict_3min_44k)
    ref = coloured(rng, nsrc, n, 2)
    ref[0, 10 * 44100:12 * 44100 + 500] = 0                          # silent stretches: NaN frames 10 and 11
    ref[nsrc - 1, 100 * 44100 + 7:101 * 44100 + 7] = 0               # not a whole frame: scored
    est = (ref + 0.25 * np.roll(ref, 1, axis=0) + 0.05 * rng.standard_normal(ref.shape)).astype(np.float32)
    got = np.stack(gpu(ref, est, 44100, 44100))
    assert got.shape == (4, nsrc, 180)
    want = B.bss_eval(ref, est, 44100, 44100)[0]
    assert np.all(np.isnan(got[:, :, 10:12])) and np.isfinite(got[:, :, 100]).all()
    assert max_db_diff(got, want) < 1e-4


def test_predict_scores_against_references(tmp_path):
    cfg = Config.build_config(["baseline_stereo"], dict(num_layers=3, num_frames=64), experiment_id=0)
    mc = cfg["model_config"]
    t_in, _ = O.get_padding(mc, 64)
    sep = UnetAudioSeparator(mc)
    sep.load_variables(O.init_params(mc, seed=3), input_frames=t_in)
    model = Training.save_checkpoint(str(tmp_path / "model.npz"), sep)
    rate = mc["expected_sr"]
    rng = np.random.default_rng(6)
    refs = {n: coloured(rng, 1, 3 * rate + 123, 2)[0] for n in mc["source_names"]}
    mix = sum(refs.values()).astype(np.float32)
    np.save(tmp_path / "song.npy", mix)
    np.savez(tmp_path / "refs.npz", **refs)
    Predict.main(cfg, model, str(tmp_path / "song.npy"), references_path=str(tmp_path / "refs.npz"),
                 results_dir=str(tmp_path / "results"))
    assert os.path.exists(tmp_path / "results" / "song.json")
    means = Evaluate.compute_mean_metrics(str(tmp_path / "results"), metric="SDR")
    assert len(means) == len(Evaluate.eval_track(refs, {n: refs[n] for n in refs}, rate)["targets"])
    assert all(np.isfinite(m).all() for m in means)
