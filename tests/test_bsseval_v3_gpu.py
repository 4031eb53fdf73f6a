"""BSS Eval v3 on the GPU (wun.bss_eval(..., mode="v3"), wun_bss_eval_v3) against the float64 oracle
(oracle/bsseval_v3_oracle.py): per-frame filters and metrics on overlapping, gapped and ragged framings, 3-minute tracks on
sampled frames, bits independent of the frames per pass, silent frames, and Predict.py with bss_mode=v3."""
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
from bsseval_cases import check_silent_case, coloured, silent_case
from bsseval_v3_cases import check_closed_forms_v3
from oracle import bsseval_v3_oracle as V3
from oracle import wave_unet_oracle as O

pytestmark = pytest.mark.gpu


def gpu(ref, est, win, hop, filters=False, **kw):
    out = wun.bss_eval(torch.from_numpy(np.ascontiguousarray(ref)).cuda(), torch.from_numpy(np.ascontiguousarray(est)).cuda(),
                       win, hop, filters=filters, mode="v3", **kw)
    return [t.cpu().numpy() for t in out]


def max_db_diff(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isinf(a), np.isinf(b))
    f = np.isfinite(a)
    return float(np.max(np.abs(a[f] - b[f]))) if f.any() else 0.0


def rel_norm(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def coloured_case(seed, nsrc, nchan, n):
    rng = np.random.default_rng(seed)
    ref = coloured(rng, nsrc, n, nchan)
    est = (ref + 0.3 * np.roll(ref, 1, axis=0) + 0.1 * rng.standard_normal(ref.shape)).astype(np.float32)
    return ref, est


# overlapping (hop < win), gapped (hop > win) and ragged (samples after the last frame) framings
@pytest.mark.parametrize("nsrc,nchan,n,win,hop", [(2, 2, 24000, 8000, 4000), (3, 1, 26000, 6000, 9000),
                                                  (1, 2, 20500, 8000, 8000), (4, 2, 30000, 12000, 9000)])
def test_filters_and_metrics_match_oracle(nsrc, nchan, n, win, hop):
    ref, est = coloured_case(10 + nsrc, nsrc, nchan, n)
    want, C, Cj = V3.bss_eval_v3(ref, est, win, hop)
    *got, gC, gCj = gpu(ref, est, win, hop, filters=True)
    assert gC.shape == C.shape and gCj.shape == Cj.shape and C.shape[0] >= 2
    for t in range(C.shape[0]):
        assert rel_norm(gC[t], C[t]) < 1e-8 and rel_norm(gCj[t], Cj[t]) < 1e-8, (t, rel_norm(gC[t], C[t]))
    assert max_db_diff(np.stack(got), want) < 1e-6


def test_closed_forms_gpu_v3():
    check_closed_forms_v3(lambda r, e, w, h: gpu(r, e, w, h), seconds=6)


def test_silent_frames_gpu_v3():
    ref, est, win = silent_case()
    *got, gC, gCj = gpu(ref, est, win, win, filters=True)
    check_silent_case(*got)
    want = V3.bss_eval_v3(ref, est, win, win)[0]
    got = np.stack(got)
    exact = (got > 150) & (want > 150)
    assert max_db_diff(np.where(exact, 0, got), np.where(exact, 0, want)) < 1e-6
    assert np.all(np.isnan(gC[[1, 3]])) and np.all(np.isnan(gCj[[1, 3]]))   # never solved
    assert np.all(np.isfinite(gC[[0, 2]])) and np.all(np.isfinite(gCj[[0, 2]]))


def test_frames_per_pass_and_repeat_give_the_same_bits():
    ref, est = coloured_case(30, 3, 2, 40000)
    ref[1, 8000:17000] = 0                                           # silent frames 2 and 3: fewer frames than slots
    runs = [gpu(ref, est, 5000, 4000, filters=True, max_workspace_bytes=b) for b in (0, 0, 1 << 40, 3 * 84 << 20)]
    nwin = runs[0][0].shape[1]
    assert nwin == 9 and np.isnan(runs[0][0][:, 2:4]).all()
    for other in runs[1:]:
        for x, y in zip(runs[0], other):
            assert np.array_equal(x.view(np.uint64), y.view(np.uint64))


@pytest.mark.parametrize("nsrc", [2, 4])
def test_full_size_three_minutes_sampled_frames(nsrc):
    rng = np.random.default_rng(40 + nsrc)
    n, rate = 7938000, 44100
    ref = coloured(rng, nsrc, n, 2)
    ref[0, 10 * rate:12 * rate + 500] = 0                            # NaN frames 10 and 11
    est = (ref + 0.25 * np.roll(ref, 1, axis=0) + 0.05 * rng.standard_normal(ref.shape)).astype(np.float32)
    got = np.stack(gpu(ref, est, rate, rate))
    assert got.shape == (4, nsrc, 180)
    assert np.all(np.isnan(got[:, :, 10:12])) and np.isfinite(np.delete(got, [10, 11], axis=2)).all()
    for t in (0, 12, 61, 117, 179):
        r, e = V3.frame_slices(ref, est, t, rate, rate)
        want = V3.bss_eval_v3(r, e, rate, rate)[0][:, :, 0]
        assert max_db_diff(got[:, :, t], want) < 1e-4, t


def test_predict_bss_mode_v3_writes_json(tmp_path):
    cfg = Config.build_config(["baseline_stereo"], dict(num_layers=3, num_frames=64), experiment_id=0)
    mc = cfg["model_config"]
    t_in, _ = O.get_padding(mc, 64)
    sep = UnetAudioSeparator(mc)
    sep.load_variables(O.init_params(mc, seed=3), input_frames=t_in)
    model = Training.save_checkpoint(str(tmp_path / "model.npz"), sep)
    rate = mc["expected_sr"]
    rng = np.random.default_rng(6)
    refs = {n: coloured(rng, 1, 3 * rate + 123, 2)[0] for n in mc["source_names"]}
    np.save(tmp_path / "song.npy", sum(refs.values()).astype(np.float32))
    np.savez(tmp_path / "refs.npz", **refs)
    Predict.main(cfg, model, str(tmp_path / "song.npy"), references_path=str(tmp_path / "refs.npz"),
                 results_dir=str(tmp_path / "results"), bss_mode="v3")
    assert os.path.exists(tmp_path / "results" / "song.json")
    means = Evaluate.compute_mean_metrics(str(tmp_path / "results"), metric="SIR")
    assert means and all(np.isfinite(m).all() for m in means)
