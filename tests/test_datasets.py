"""Dataset layer without a GPU: track discovery, the valid split, stem checks, the accompaniment, the snippet positions of
Test.test against a transcription of take_all_snippets, and the command-line extras (Datasets.py, Training.py)."""
import os

import numpy as np
import pytest
import scipy.io.wavfile

import Config
import Datasets
import Training
from dataset_fixtures import TEST, TRAIN, write_ccmixter, write_musdb
from oracle import dataset_oracle as D


def mc(named=("baseline_stereo",), **kw):
    kw.setdefault("num_layers", 2)
    kw.setdefault("num_frames", 40)
    return Config.build_config(list(named), kw, experiment_id=0)["model_config"]


@pytest.fixture
def musdb(tmp_path):
    return write_musdb(str(tmp_path / "musdb"))


def test_discovery_is_sorted_and_complete(musdb):
    train = Datasets.musdb_tracks(musdb, "train")
    assert [t["name"] for t in train] == sorted(TRAIN)
    test = Datasets.musdb_tracks(musdb, "test")
    assert [t["name"] for t in test] == sorted(TEST)
    t = train[0]
    assert t["mix"] == os.path.join(musdb, "train", "a_track", "mixture.wav")
    assert all(t[s] == os.path.join(musdb, "train", "a_track", s + ".wav") for s in Datasets.MUSDB_STEMS)
    with pytest.raises(FileNotFoundError):
        Datasets.musdb_tracks(musdb, "valid")
    os.remove(os.path.join(musdb, "test", "t_mid", "drums.wav"))
    with pytest.raises(FileNotFoundError, match="drums.wav"):
        Datasets.musdb_tracks(musdb, "test")


def test_ccmixter_xml(tmp_path):
    xml = write_ccmixter(str(tmp_path))
    tracks = Datasets.ccmixter_tracks(xml)
    assert [t["name"] for t in tracks] == ["cc_one", "cc_two"]
    db = os.path.join(str(tmp_path), "ccmixter")
    assert tracks[0]["mix"] == db + os.sep + os.path.join("cc_one", "mix.wav")
    assert tracks[0]["vocals"].endswith("source-02.wav") and tracks[0]["accompaniment"].endswith("source-01.wav")
    assert Datasets.probe_track(tracks[1], mc()) == (22050, 650)


def test_split_is_deterministic_and_disjoint(musdb):
    train = Datasets.musdb_tracks(musdb, "train")
    a_train, a_valid = Datasets.split_valid(train, 2)
    b_train, b_valid = Datasets.split_valid(train, 2)
    assert [t["name"] for t in a_valid] == [t["name"] for t in b_valid]
    assert [t["name"] for t in a_train] == [t["name"] for t in b_train]
    names_t, names_v = {t["name"] for t in a_train}, {t["name"] for t in a_valid}
    assert not names_t & names_v and names_t | names_v == set(TRAIN) and len(names_v) == 2
    idx = np.random.RandomState(1337).choice(len(train), 2, replace=False)
    assert [t["name"] for t in a_valid] == [train[i]["name"] for i in idx]
    for n in (len(train), len(train) + 3):
        with pytest.raises(ValueError, match="valid_tracks"):
            Datasets.split_valid(train, n)


def test_stem_mismatch_errors_name_the_files(musdb):
    cfg = mc()
    track = Datasets.musdb_tracks(musdb, "train")[0]
    assert Datasets.probe_track(track, cfg) == (44100, 1234)
    rate, data = scipy.io.wavfile.read(track["vocals"])
    for bad in (lambda: scipy.io.wavfile.write(track["vocals"], rate, data[:-1]),          # length
                lambda: scipy.io.wavfile.write(track["vocals"], 22050, data),              # rate
                lambda: scipy.io.wavfile.write(track["vocals"], rate, data[:, 0])):        # channels
        bad()
        with pytest.raises(ValueError) as e:
            Datasets.probe_track(track, cfg)
        assert track["vocals"] in str(e.value) and track["mix"] in str(e.value)
        scipy.io.wavfile.write(track["vocals"], rate, data)


@pytest.mark.parametrize("named,task", [("baseline_stereo", "voice"), ("baseline_context", "voice"),
                                        ("full_multi_instrument", "multi_instrument")])
def test_read_track_accompaniment_and_channels(musdb, named, task):
    cfg = mc((named,))
    assert cfg["task"] == task
    for track in Datasets.musdb_tracks(musdb, "train"):
        rate, audio = Datasets.read_track(track, cfg)
        raw = {k: D.read(track[k])[1] for k in ("mix",) + Datasets.MUSDB_STEMS}
        if task == "voice":
            raw["accompaniment"] = np.clip(raw["bass"] + raw["drums"] + raw["other"], -1.0, 1.0)
        assert list(audio) == cfg["source_names"] + ["mix"]
        for k, a in audio.items():
            want = raw[k]
            if cfg["mono_downmix"]:
                want = np.mean(want, axis=1, keepdims=True)
            elif want.shape[1] == 1:
                want = np.tile(want, [1, 2])
            assert a.dtype == np.float32 and np.array_equal(a, want), (track["name"], k)


def test_oracle_staging_pads_both_ends(musdb):
    cfg = mc()
    import wun
    track = Datasets.musdb_tracks(musdb, "train")[0]
    tables = lambda a, b: wun.resample_tables(a, b) + (wun.KAISER_BEST_PRECISION,)
    staged = D.stage_track({k: track[k] for k in ("mix",) + Datasets.MUSDB_STEMS}, cfg["source_names"], False, 22050,
                           151, 41, tables)
    n = wun.resample_frames(1234, 44100, 22050)
    for k, a in staged.items():
        assert a.shape == (n + 110, 2) and not a[:55].any() and not a[-55:].any()


def transcribed_positions(lengths, t_in, t_out, batch):
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    snippets = [o + s for o, l in zip(offsets, lengths) for s in D.take_all_snippets(int(l), t_in, t_out)]
    return [p for b in D.batch_and_drop_remainder(snippets, batch) for p in b]


@pytest.mark.parametrize("lengths,batch", [
    ([151, 150, 100], 1),                # L - T_in <= 0: no snippet
    ([151 + 41 * 3], 2),                 # L - T_in an exact multiple of T_out: the last start is excluded
    ([152 + 41 * 3], 2),                 # one frame more: that start is included
    ([400, 151, 333, 1000, 90, 700], 4),  # batches that cross tracks, remainder dropped
    ([5000], 7),
])
def test_snippet_positions_match_take_all_snippets(lengths, batch):
    lengths = np.array(lengths, np.int64)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64)
    want = transcribed_positions(lengths, 151, 41, batch)
    if not want:
        with pytest.raises(ValueError, match="fewer than one batch"):
            Datasets.snippet_positions(offsets, lengths, 151, 41, batch)
        return
    got = Datasets.snippet_positions(offsets, lengths, 151, 41, batch)
    assert got.dtype == np.int64 and got.tolist() == want and len(got) % batch == 0


def test_exact_multiple_excludes_the_last_start():
    assert Datasets.snippet_starts(151 + 41 * 3, 151, 41).tolist() == [0, 41, 82]
    assert Datasets.snippet_starts(152 + 41 * 3, 151, 41).tolist() == [0, 41, 82, 123]
    assert Datasets.snippet_starts(151, 151, 41).tolist() == [] and Datasets.snippet_starts(20, 151, 41).tolist() == []


def test_too_few_snippets_for_one_batch():
    with pytest.raises(ValueError, match="3 snippets .* fewer than one batch of 4"):
        Datasets.snippet_positions(np.array([0]), np.array([151 + 41 * 2 + 1]), 151, 41, 4)
    with pytest.raises(ValueError):
        Datasets.snippet_positions(np.zeros(0, np.int64), np.zeros(0, np.int64), 151, 41, 1)


def test_cli_dataset_extras():
    cfg, extras = Config.parse_command_line(["with", "cfg.full", "model_config.musdb_path=/data/musdb18", "dataset=musdb",
                                             "ccmixter_xml=/data/CCMixter.xml", "valid_tracks=10", "max_epochs=3"])
    assert cfg["model_config"]["musdb_path"] == "/data/musdb18"
    assert extras == {"dataset": "musdb", "ccmixter_xml": "/data/CCMixter.xml", "valid_tracks": 10, "max_epochs": 3}
    assert Training.dataset_options(extras) == {"dataset": "musdb", "ccmixter_xml": "/data/CCMixter.xml", "valid_tracks": 10}
    _, extras = Config.parse_command_line(["with", "cfg.full", "dataset=musdb"])
    assert Training.dataset_options(extras) == {"dataset": "musdb", "valid_tracks": 25}
    _, extras = Config.parse_command_line(["with", "cfg.baseline_context", "max_epochs=1"])
    assert Training.dataset_options(extras) == {}
    with pytest.raises(ValueError, match="only dataset=musdb"):
        Training.dataset_options({"dataset": "dsd100"})
    with pytest.raises(ValueError, match="need dataset=musdb"):
        Training.dataset_options({"valid_tracks": 3})


def test_layout_paths_live_in_one_place():
    assert Datasets.estimate_path("/e", "test", "t", "vocals") == os.path.join("/e", "test", "t", "vocals.wav")
    assert Datasets.museval_json_dir("/e", "train") == os.path.join("/e", "train")
