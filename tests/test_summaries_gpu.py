"""The reference's TensorBoard summaries on the GPU: Training.train's per-step `sep_loss` for the Wave-U-Net and the
spectrogram U-Nets (U7, U7a) against a run of the same seed that reads every step's loss on the host, resumed epochs,
wall times, Test.test's `test_loss`, and Training.run(dataset="musdb") writing both into log_dir/<experiment_id>."""
import glob
import os
import time

import numpy as np
import pytest
import torch

import Config
import Datasets
import Summaries
import Test
import Training
from dataset_fixtures import TEST, TRAIN, write_ccmixter, write_musdb
from Models.UnetAudioSeparator import UnetAudioSeparator
from oracle import wave_unet_oracle as O

pytestmark = pytest.mark.gpu

SPEC_T = 1024 + 768 * 7
NETWORKS = {
    "wave_u_net": ("baseline_stereo", dict(num_layers=3, num_frames=40, batch_size=4)),
    "u7": ("unet_spectrogram", dict(num_layers=2, num_initial_filters=4, num_frames=SPEC_T, batch_size=2)),
    "u7a": ("unet_spectrogram_l1", dict(num_layers=2, num_initial_filters=4, num_frames=SPEC_T, batch_size=2)),
}


def f32_bits(x):
    return np.float32(x).tobytes()


def events_files(logdir):
    return sorted(glob.glob(os.path.join(str(logdir), "*tfevents*")))


def host_read_losses(cfg, load_model=None):
    """Training.train's steps with the same seeds, each step's loss read on the host right after it."""
    dev = torch.device("cuda", 0)
    sep = Training.separator_class(cfg)(cfg)
    in_shape, _ = sep.get_padding(np.array([cfg["batch_size"], cfg["num_frames"], 0]))
    t_in = int(in_shape[1])
    eng = sep.engine(input_frames=t_in)
    if load_model is not None:
        Training.load_checkpoint(load_model, sep, t_in)
    sep._ensure_params(eng, dev, create=True)
    sep._ensure_training_state()
    feeder = Training._device_feeder(cfg, sep, eng, dev, 0, 1, int(in_shape[0]))
    losses = []
    for _ in range(cfg["epoch_it"]):
        mix, tg = feeder.next_batch()
        losses.append(float(sep.loss_and_gradients(mix, tg).item()))
        sep.adam_step(cfg["init_sup_sep_lr"])
    return losses


def check_epoch(path, first_step, want, t0, t1):
    records = Summaries.read_records(path)
    first = Summaries.decode_event(records[0])
    assert first["file_version"] == "brain.Event:2" and first["values"] == []
    got = Summaries.read_scalars(path)
    assert len(records) == 1 + len(want)
    assert [(s, tag) for _, s, tag, _ in got] == [(first_step + i, "sep_loss") for i in range(len(want))]
    for i, ((_, _, _, v), w) in enumerate(zip(got, want)):
        assert f32_bits(v) == f32_bits(w), (i, v, w)
    walls = [t for t, _, _, _ in got]
    assert all(a <= b for a, b in zip(walls, walls[1:])), walls
    assert t0 <= walls[0] and walls[-1] <= t1, (t0, walls, t1)


@pytest.mark.parametrize("net", sorted(NETWORKS))
def test_train_writes_sep_loss_per_step_and_resumes(tmp_path, net):
    named, kw = NETWORKS[net]
    cfg = Config.build_config([named], dict(kw, epoch_it=12, model_base_dir=str(tmp_path / "ck"),
                                            log_dir=str(tmp_path / "logs")), experiment_id=42)["model_config"]
    logdir = tmp_path / "logs" / "42"
    t0 = time.time()
    path, sep = Training.train(dict(cfg), 42, log_every=0, summaries=True)
    t1 = time.time()
    (first,) = events_files(logdir)
    check_epoch(first, 0, host_read_losses(dict(cfg)), t0, t1)
    # a resumed run continues at the checkpoint's step, in a new file
    t0 = time.time()
    path2, sep2 = Training.train(dict(cfg), 42, load_model=path, log_every=0, summaries=True)
    t1 = time.time()
    assert sep2.global_step == 24
    (second,) = [p for p in events_files(logdir) if p != first]
    check_epoch(second, 12, host_read_losses(dict(cfg), load_model=path), t0, t1)


@pytest.fixture(scope="module")
def tiny_dataset(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("ds"))
    return write_musdb(os.path.join(root, "musdb")), write_ccmixter(root)


def test_test_writes_one_test_loss_at_the_global_step(tiny_dataset, tmp_path):
    musdb, xml = tiny_dataset
    cfg = Config.build_config(["baseline_stereo"], dict(num_layers=2, num_frames=40, batch_size=4,
                                                        log_dir=str(tmp_path / "logs")), experiment_id=0)["model_config"]
    ds = Datasets.load_musdb(cfg, 151, 41, musdb, xml, valid_tracks=2)
    sep = UnetAudioSeparator(cfg)
    sep.load_variables(O.init_params(cfg, seed=5), input_frames=151)
    sep.global_step = 17
    quiet = Test.test(cfg, "valid", "run", None, dataset=ds, separator=sep)
    assert not os.path.exists(str(tmp_path / "logs"))                 # the default writes nothing
    for part in ("valid", "test"):
        before = events_files(tmp_path / "logs" / "run")
        loss = Test.test(cfg, part, "run", None, dataset=ds, separator=sep, summaries=True)
        (path,) = [p for p in events_files(tmp_path / "logs" / "run") if p not in before]
        ((_, step, tag, value),) = Summaries.read_scalars(path)
        assert (step, tag) == (17, "test_loss") and f32_bits(value) == f32_bits(loss)
        if part == "valid":
            assert loss == quiet


def test_training_run_on_musdb_writes_sep_loss_and_test_loss(tmp_path):
    stereo = lambda spec: {n: (rate, frames, 2, fmt) for n, (rate, frames, _, fmt) in spec.items()}
    musdb = write_musdb(str(tmp_path / "musdb"), stereo(TRAIN), stereo(TEST))
    xml = write_ccmixter(str(tmp_path))
    cfg = Config.build_config(["baseline_stereo"], dict(
        num_layers=2, num_frames=40, batch_size=2, epoch_it=3, worse_epochs=1, musdb_path=musdb,
        model_base_dir=str(tmp_path / "ck"), log_dir=str(tmp_path / "logs"), estimates_path=str(tmp_path / "est")),
        experiment_id=7)
    path, loss = Training.run(cfg, max_epochs=2, dataset="musdb", ccmixter_xml=xml, valid_tracks=2)
    files = events_files(tmp_path / "logs" / "7")
    scalars = sorted((x for p in files for x in Summaries.read_scalars(p)), key=lambda x: x[0])
    sep_loss = [(s, v) for _, s, tag, v in scalars if tag == "sep_loss"]
    test_loss = [(s, v) for _, s, tag, v in scalars if tag == "test_loss"]
    assert len(files) == 2 + 3                          # one file per epoch, one per validation, one for the final test
    assert [s for s, _ in sep_loss] == list(range(6)) and all(np.isfinite(v) for _, v in sep_loss)
    assert [s for s, _ in test_loss[:2]] == [3, 6]       # a validation after each epoch
    best_step = int(path.rsplit("-", 1)[1])
    assert test_loss[2][0] == best_step and f32_bits(test_loss[2][1]) == f32_bits(loss)
