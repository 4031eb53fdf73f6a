"""The spectrogram U-Net's training step without a GPU: the float64 oracle (oracle/spectrogram_train_oracle.py) against the
fixtures of the reference's own get_output(training=True) and against finite differences, the dropout hash, the FLOP closed
form, the trainable set, checkpoints with Adam slots for the trainables only, and Training.train's refusal of data
parallelism."""
import json
import os

import numpy as np
import pytest
import torch

import Config
import TFCheckpoint
import Training
import wun
from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator
from oracle import spectrogram_oracle as S
from oracle import spectrogram_train_oracle as O
from wun import parallel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spectrogram_train")
TRAIN_CASES = ["train_l2_u7", "train_l3_u7a", "train_l5_u7"]
PRESET_FRAMES = 768 * 127 + 1024


def mc(named="unet_spectrogram", **kw):
    return Config.build_config([named], kw, experiment_id=0)["model_config"]


def load_case(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = json.loads(str(z["cfg_json"]))
    params = {k[len("param/"):]: z[k].astype(np.float32) for k in z.files if k.startswith("param/")}
    mix = z["mix_pcm16"].astype(np.float32) / np.float32(32768)
    targets = [z["target_pcm16"][k].astype(np.float32) / np.float32(32768) for k in range(2)]
    masks = {}
    for k in z.files:
        if k.startswith("keep/"):
            _, src, lev = k.split("/")
            masks[(int(src), int(lev))] = np.unpackbits(z[k])[:int(np.prod(z["keep_shape/%s/%s" % (src, lev)]))] \
                .reshape(tuple(z["keep_shape/%s/%s" % (src, lev)])).astype(bool)
    return z, cfg, params, mix, targets, masks


@pytest.mark.parametrize("name", TRAIN_CASES)
def test_oracle_matches_reference_training_fixtures(name):
    z, cfg, params, mix, targets, masks = load_case(name)
    loss, grads, moving = O.forward_backward(params, mix, targets, cfg["num_layers"], cfg["source_names"],
                                             cfg["raw_audio_loss"], masks)
    assert abs(loss - float(z["loss"])) <= 1e-12 * abs(float(z["loss"])), (loss, float(z["loss"]))
    for n, g in grads.items():
        want = z["grad/" + n].astype(np.float64)                 # stored rounded to float32
        err = np.abs(g - want).max()
        # relative to the tensor's largest value; a conv bias that feeds batch norm has gradient 0 plus float64 noise
        assert err <= 1e-6 * np.abs(want).max() or err <= 1e-15, (name, n, err)
    for n, v in moving.items():
        assert np.allclose(v, z["moving/" + n], rtol=1e-12, atol=1e-15), (name, n)
    assert set(grads) == {k[len("grad/"):] for k in z.files if k.startswith("grad/")}


@pytest.mark.parametrize("name", TRAIN_CASES)
def test_fixture_masks_are_the_engine_hash(name):
    z, cfg, _, mix, _, masks = load_case(name)
    want = O.engine_masks(int(z["dropout_seed"]), int(z["dropout_step"]), mix.shape[0], S.stft_frames(mix.shape[1]),
                          cfg["num_layers"], cfg["num_initial_filters"])
    assert set(want) == set(masks) and all(np.array_equal(want[k], masks[k]) for k in want)


def test_fixtures_have_dropped_and_undropped_levels():
    z, cfg, _, _, _, masks = load_case("train_l5_u7")
    assert cfg["num_layers"] == 5 and sorted({d for _, d in masks}) == [1, 2, 3]    # level 0 is not dropped
    assert cfg["num_initial_filters"] <= 2 and z["mix_pcm16"].shape[1] == 1024 + 768 * 31


def test_oracle_gradient_matches_finite_differences():
    L, Fi, n, B = 2, 2, 4, 1
    T = 1024 + 768 * (n - 1)
    params = S.random_params(L, Fi, seed=3)
    rng = np.random.default_rng(1)
    mix = rng.uniform(-0.5, 0.5, (B, T, 1)).astype(np.float32)
    targets = [rng.uniform(-0.3, 0.3, (B, T, 1)).astype(np.float32) for _ in range(2)]
    masks = O.engine_masks(1337, 4, B, n, L, Fi)
    for raw in (True, False):
        _, grads, _ = O.forward_backward(params, mix, targets, L, ["accompaniment", "vocals"], raw, masks)
        for name in ("separator/conv2d_1/kernel", "separator/conv2d_transpose/kernel", "separator/BatchNorm_1/beta",
                     "separator/conv2d_transpose_3/bias"):
            idx = np.unravel_index(int(np.argmax(np.abs(grads[name]))), grads[name].shape)
            h = 1e-6
            p = {k: np.asarray(v, np.float64).copy() for k, v in params.items()}
            p[name][idx] += h
            up = O.forward_backward(p, mix, targets, L, ["accompaniment", "vocals"], raw, masks)[0]
            p[name][idx] -= 2 * h
            down = O.forward_backward(p, mix, targets, L, ["accompaniment", "vocals"], raw, masks)[0]
            fd = (up - down) / (2 * h)
            assert abs(fd - grads[name][idx]) <= 1e-5 * abs(grads[name][idx]), (raw, name, fd, grads[name][idx])


def test_dropout_hash_keeps_half_and_differs_across_step_source_and_level():
    shape = (2, 16, 64, 32)
    base = O.keep_masks(1337, 10, 0, 2, shape)
    assert abs(base.mean() - 0.5) < 0.01
    for other in (O.keep_masks(1337, 11, 0, 2, shape), O.keep_masks(1337, 10, 1, 2, shape),
                  O.keep_masks(1337, 10, 0, 3, shape), O.keep_masks(1338, 10, 0, 2, shape)):
        agree = (other == base).mean()
        assert abs(agree - 0.5) < 0.01, agree
    assert np.array_equal(base, O.keep_masks(1337, 10, 0, 2, shape))


def test_dropped_levels():
    assert O.dropped_levels(1) == [] and O.dropped_levels(2) == [0] and O.dropped_levels(3) == [0, 1]
    assert O.dropped_levels(6) == [2, 3, 4]


def engine(cfg, T):
    return wun.SpecEngine(wun.spec_config_from_model_config(cfg), num_frames=T)


def test_train_flops_closed_form_at_the_preset():
    eng = engine(mc("unet_spectrogram"), PRESET_FRAMES)
    assert eng.train_flops(1) == 9017753600.0
    assert eng.train_flops(4) == 4 * 9017753600.0
    assert eng.train_flops(4) == 3 * eng.forward_flops(4) - 2 * 2 * (64 * 256 * 25 * 16) * 4
    assert eng.train_workspace_bytes(4) > eng.workspace_bytes(4)


def test_trainable_set_of_the_parameter_table():
    eng = engine(mc("unet_spectrogram"), PRESET_FRAMES)
    names = [n for n, _, _, _ in eng.param_table]
    trainable = [n for n, _, _ in eng.trainable_ranges]
    assert trainable == [n for n in names if n.rsplit("/", 1)[1] in ("kernel", "bias", "beta")]
    assert len(trainable) == 2 * (6 * 3 + 5 * 3 + 2) and len(names) - len(trainable) == 2 * 11 * 2
    assert [(o, c) for _, o, c in eng.trainable_ranges] == [(o, c) for n, _, o, c in eng.param_table if n in trainable]


def test_checkpoint_round_trip_has_adam_slots_for_trainables_only(tmp_path):
    T = 1024 + 768 * 7
    cfg = mc("unet_spectrogram_l1", num_layers=3, num_initial_filters=3, num_frames=T)
    sep = UnetSpectrogramSeparator(cfg)
    sep.load_variables(S.random_params(3, 3, seed=4), device=torch.device("cpu"), num_frames=T)
    sep._ensure_training_state()
    rng = np.random.default_rng(0)
    trainable = sep.trainable_variable_names()
    for n, _, o, c in sep.param_table():
        if n in trainable:
            sep.adam_m[o:o + c] = torch.from_numpy(rng.uniform(-1, 1, c).astype(np.float32))
            sep.adam_v[o:o + c] = torch.from_numpy(rng.uniform(0, 1, c).astype(np.float32))
    sep.global_step = 12
    path = TFCheckpoint.save_separator(str(tmp_path / "u7a-12"), sep)
    names = [n for n, _, _ in TFCheckpoint.list_variables(path)]
    slots = sorted(n for n in names if n.endswith(("/Adam", "/Adam_1")))
    want = sorted("%s/%s/%s" % (TFCheckpoint.SOLVER_SCOPE, n, s) for n in trainable for s in ("Adam", "Adam_1"))
    assert slots == want
    fresh = UnetSpectrogramSeparator(cfg)
    fresh.engine(num_frames=T)
    TFCheckpoint.restore_separator(path, fresh, T)
    assert fresh.global_step == 12
    for a, b in ((fresh.params, sep.params), (fresh.adam_m, sep.adam_m), (fresh.adam_v, sep.adam_v)):
        assert np.array_equal(a.numpy().view(np.uint32), b.numpy().view(np.uint32))
    assert int(fresh._dropout_step.item()) == 12                 # the dropout masks resume with the step


def test_training_refuses_data_parallel_spectrogram(monkeypatch):
    monkeypatch.setattr(parallel, "world", lambda: (0, 2))
    with pytest.raises(ValueError, match="one GPU"):
        Training.train(mc("unet_spectrogram_l1"), 0)
