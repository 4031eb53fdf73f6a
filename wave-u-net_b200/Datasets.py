"""From a dataset directory to partition pools in HBM: the reference's Datasets.py (getMUSDB, getCCMixter, write_records,
the partition split and take_all_snippets) over WAV files, without TFRecords.

    ds = Datasets.load_musdb(model_config, t_in, t_out, musdb_path, ccmixter_xml=None, valid_tracks=25)
    ds.partitions["train" | "valid" | "test"]     # Partition: pool [K + 1, frames, C] on the device, offsets, lengths
    ds.train_feeder(engine, batch, ...)           # wun.feeder.DeviceFeeder over the train pool
    ds.positions("valid", batch)                  # device int64 snippet frames for Test.test, built once per batch size

Tracks come from the MUSDB18 WAV layout <musdb_path>/{train,test}/<track>/{mixture,bass,drums,other,vocals}.wav (the
decoded and HQ releases), sorted by name, and for the voice task optionally from an XML of the reference's CCMixter schema
(train only, Datasets.py:150-155).  Every stem is staged as write_records prepares it (Datasets.py:43-93): read (Predict.
read_wav), for the voice task accompaniment = clip(bass + drums + other, -1, 1) (Datasets.py:259-262), the mono downmix or
the tiling to stereo of Evaluate._model_channels, upload, kaiser_best resampling to expected_sr on the GPU (wun.resample),
and a copy into the zero-initialised pool at offset + (T_in - T_out) // 2, which gives the zero padding at both ends.

Not reproduced: the reference's PCM16 round trip of every stem through soundfile.write, its TFRecord cache, the shuffle
buffer, and its own validation draw, which depends on sacred's seeding and musdb's listing order.
"""
import os
import xml.etree.ElementTree as ET

import numpy as np
import scipy.io.wavfile

# The MUSDB18 WAV layout and the musdb / museval output layout, as recalled from those packages (neither is read here).
MUSDB_SUBSETS = ("train", "test")
MUSDB_STEMS = ("bass", "drums", "other", "vocals")
MUSDB_FILES = dict(mix="mixture", bass="bass", drums="drums", other="other", vocals="vocals")
ACCOMPANIMENT_STEMS = ("bass", "drums", "other")            # summed in this order (Datasets.py:259-262)


def estimate_path(estimates_path, subset, track, source):
    """musdb's estimates_dir layout: <estimates_path>/<subset>/<track>/<source>.wav."""
    return os.path.join(estimates_path, subset, track, "%s.wav" % source)


def museval_json_dir(estimates_path, subset):
    """museval's output_dir layout: one <track>.json per track in <estimates_path>/<subset>."""
    return os.path.join(estimates_path, subset)


VALID_SEED = 1337               # the reference experiment's seed (Training.py:21)


# ---- discovery ----------------------------------------------------------------------------------------------------------
def musdb_tracks(musdb_path, subset):
    """[{"name", "mix", "bass", "drums", "other", "vocals"}] (file paths) of <musdb_path>/<subset>/*/, sorted by name."""
    root = os.path.join(musdb_path, subset)
    if not os.path.isdir(root):
        raise FileNotFoundError("%s: no MUSDB18 %s directory (expected <musdb_path>/{train,test}/<track>/mixture.wav ...)"
                                % (root, subset))
    tracks = []
    for name in sorted(os.listdir(root)):
        d = os.path.join(root, name)
        if not os.path.isdir(d):
            continue
        t = {"name": name}
        for key, stem in MUSDB_FILES.items():
            path = os.path.join(d, stem + ".wav")
            if not os.path.isfile(path):
                raise FileNotFoundError("%s: missing (a MUSDB18 WAV track has %s.wav)" % (path, ".wav, ".join(MUSDB_FILES.values())))
            t[key] = path
        tracks.append(t)
    return tracks


def ccmixter_tracks(xml_path):
    """[{"name", "mix", "accompaniment", "vocals"}] from an XML of the reference's CCMixter schema (Datasets.py:279-295):
    databaseFolderPath + each instrument's relativeFilepath, instruments Mix, Instrumental and Voice."""
    root = ET.parse(xml_path).getroot()
    db_path = root.find("./databaseFolderPath").text
    tracks = []
    for i, track in enumerate(root.findall(".//track")):
        t = {}
        for key, inst in (("mix", "Mix"), ("accompaniment", "Instrumental"), ("vocals", "Voice")):
            node = track.find(".//instrument[instrumentName='%s']" % inst)
            if node is None:
                raise ValueError("%s: track %d has no %s instrument" % (xml_path, i, inst))
            t[key] = db_path + os.path.sep + node.find("./relativeFilepath").text
        t["name"] = os.path.basename(os.path.dirname(t["mix"])) or "ccmixter_%d" % i
        tracks.append(t)
    return tracks


def split_valid(train_tracks, valid_tracks=25, seed=VALID_SEED):
    """(train, valid): `valid_tracks` of the sorted MUSDB train tracks drawn with RandomState(seed).choice(n, valid_tracks,
    replace=False), in drawn order (Datasets.py:139-148); the rest, in their order, is the train partition."""
    n = len(train_tracks)
    if valid_tracks >= n:
        raise ValueError("valid_tracks = %d leaves no training track out of %d MUSDB train tracks" % (valid_tracks, n))
    idx = np.random.RandomState(seed).choice(n, int(valid_tracks), replace=False)
    chosen = set(int(i) for i in idx)
    valid = [train_tracks[int(i)] for i in idx]
    print("Validation with MUSDB training songs: " + ", ".join(t["name"] for t in valid))
    return [t for i, t in enumerate(train_tracks) if i not in chosen], valid


# ---- host side of staging -----------------------------------------------------------------------------------------------
def _files(track, model_config):
    """The files a track is read from for the model's sources: key -> path (the accompaniment of a MUSDB track is summed)."""
    names = list(model_config["source_names"]) + ["mix"]
    if "accompaniment" in names and "accompaniment" not in track:
        names = [n for n in names if n != "accompaniment"] + list(ACCOMPANIMENT_STEMS)
    return {n: track[n] for n in dict.fromkeys(names)}


def probe_track(track, model_config):
    """(rate, frames) of a track from its WAV headers; raises ValueError naming the files when its stems differ in rate,
    length or channel count (Datasets.py:79-83)."""
    info = {}
    for key, path in _files(track, model_config).items():
        rate, data = scipy.io.wavfile.read(path, mmap=True)
        info[path] = (int(rate), int(data.shape[0]), 1 if data.ndim == 1 else int(data.shape[1]))
        del data
    if len(set(info.values())) != 1:
        raise ValueError("track %s: stems differ in rate, length or channels: %s" % (
            track.get("name"), "; ".join("%s (%d Hz, %d frames, %d ch)" % ((p,) + v) for p, v in info.items())))
    rate, frames, _ = next(iter(info.values()))
    return rate, frames


def read_track(track, model_config):
    """(rate, {key: float32 [frames, C]}) for key in source_names + ["mix"] at the file's rate: stems read with
    Predict.read_wav, the accompaniment of a MUSDB track summed and clipped, then Evaluate._model_channels."""
    import Evaluate
    from Predict import read_wav
    files = _files(track, model_config)
    raw = {}
    rate = None
    for key, path in files.items():
        rate, raw[key] = read_wav(path)
    if "accompaniment" in model_config["source_names"] and "accompaniment" not in track:
        acc = raw[ACCOMPANIMENT_STEMS[0]]
        for s in ACCOMPANIMENT_STEMS[1:]:
            acc = acc + raw[s]
        raw["accompaniment"] = np.clip(acc, -1.0, 1.0)
    return rate, {k: Evaluate._model_channels(model_config, raw[k])
                  for k in list(model_config["source_names"]) + ["mix"]}


def snippet_starts(length, t_in, t_out):
    """take_all_snippets' start frames in a padded track of `length` frames: range(0, length - t_in, t_out)."""
    return np.arange(0, max(int(length) - int(t_in), 0), int(t_out), dtype=np.int64)


def snippet_positions(offsets, lengths, t_in, t_out, batch):
    """Absolute pool frames of every snippet of a partition, in track order, cut to floor(n / batch) * batch
    (batch_and_drop_remainder, Datasets.py:213).  Raises ValueError when there is not one full batch: the reference's
    Test.test would return 0.0 there, which early stopping would read as a perfect model."""
    pos = [int(o) + snippet_starts(l, t_in, t_out) for o, l in zip(offsets, lengths)]
    pos = np.concatenate(pos) if pos else np.zeros(0, np.int64)
    n = (len(pos) // int(batch)) * int(batch)
    if n == 0:
        raise ValueError("%d snippets of %d frames (hop %d) in the partition, fewer than one batch of %d"
                         % (len(pos), t_in, t_out, batch))
    return pos[:n].astype(np.int64)


# ---- device pools ----------------------------------------------------------------------------------------------------
class Partition(object):
    """One staged partition: `pool` float32 CUDA [K + 1, total_frames, C] (sources in source_names order, then the mix),
    `offsets` / `lengths` int64 numpy arrays (first pool frame and padded length of each track), `names` of the tracks."""

    def __init__(self, pool, offsets, lengths, names):
        self.pool, self.offsets, self.lengths, self.names = pool, offsets, lengths, names


def stage_partition(tracks, model_config, t_in, t_out, device="cuda", timings=None):
    """Stage `tracks` into one zero-initialised device pool, allocated once at its final size.  With a dict `timings`, the
    seconds spent reading WAV files ("read"), uploading ("upload") and resampling + copying ("resample") are added to it
    (the device phases are then synchronised to be timed)."""
    import time
    import torch
    import wun
    sr = int(model_config["expected_sr"])
    C = int(model_config["num_channels"])
    keys = list(model_config["source_names"]) + ["mix"]
    pad = (int(t_in) - int(t_out)) // 2
    lengths = []
    for t in tracks:
        rate, frames = probe_track(t, model_config)
        lengths.append((wun.resample_frames(frames, rate, sr) if rate != sr else frames) + 2 * pad)
    lengths = np.array(lengths, np.int64)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64) if len(tracks) else np.zeros(0, np.int64)
    total = int(lengths.sum())
    device = torch.device(device)
    nbytes = len(keys) * total * C * 4
    free, _ = torch.cuda.mem_get_info(device)
    if nbytes > free:
        raise MemoryError("staging %d tracks needs a pool of %d bytes; %s has %d bytes free" % (len(tracks), nbytes, device, free))
    pool = torch.zeros((len(keys), total, C), dtype=torch.float32, device=device)

    def clock(phase, t0, sync=False):
        if timings is not None:
            if sync:
                torch.cuda.synchronize(device)
            timings[phase] = timings.get(phase, 0.0) + time.perf_counter() - t0
        return time.perf_counter()

    for t, off, length in zip(tracks, offsets, lengths):
        t0 = time.perf_counter()
        rate, audio = read_track(t, model_config)
        t0 = clock("read", t0)
        for k, key in enumerate(keys):
            x = torch.from_numpy(np.ascontiguousarray(audio[key])).to(device)
            t0 = clock("upload", t0, sync=True)
            y = wun.resample(x, rate, sr)
            pool[k, off + pad:off + pad + y.shape[0]].copy_(y)
            t0 = clock("resample", t0, sync=True)
        assert y.shape[0] + 2 * pad == length
    return Partition(pool, offsets, lengths, [t["name"] for t in tracks])


class Dataset(object):
    """Staged train / valid / test partitions and the snippet positions Test.test replays, built once per batch size."""

    def __init__(self, partitions, model_config, t_in, t_out):
        self.partitions = partitions
        self.source_names = list(model_config["source_names"])
        self.t_in, self.t_out = int(t_in), int(t_out)
        self._positions = {}

    def positions(self, partition, batch):
        key = (partition, int(batch))
        if key not in self._positions:
            import torch
            p = self.partitions[partition]
            self._positions[key] = torch.from_numpy(
                snippet_positions(p.offsets, p.lengths, self.t_in, self.t_out, batch)).to(p.pool.device)
        return self._positions[key]

    def train_feeder(self, engine, batch, augmentation=True, seed=1337):
        """wun.feeder.DeviceFeeder over the train pool.  A track whose padded length is at most T_in is left out with a
        warning (the reference's tf.random_uniform would fail on it); no track left raises ValueError."""
        from wun.feeder import DeviceFeeder
        p = self.partitions["train"]
        keep = p.lengths > engine.T_in
        for name, length in zip(p.names, p.lengths):
            if length <= engine.T_in:
                print("WARNING: train track %s has %d padded frames, no more than T_in = %d; it is left out"
                      % (name, length, engine.T_in))
        if not keep.any():
            raise ValueError("the train partition has no track longer than T_in = %d frames" % engine.T_in)
        return DeviceFeeder.from_pool(engine, p.pool, p.offsets[keep], p.lengths[keep], self.source_names, batch,
                                      augmentation=augmentation, seed=seed)


def load_musdb(model_config, t_in, t_out, musdb_path=None, ccmixter_xml=None, valid_tracks=25, device="cuda"):
    """The reference's partitions (Datasets.py:137-155) staged on `device`: train = the MUSDB train tracks not drawn for
    valid (plus CCMixter's for the voice task when `ccmixter_xml` is given), valid = `valid_tracks` drawn ones, test = the
    MUSDB test subset."""
    musdb_path = musdb_path or model_config["musdb_path"]
    train, valid = split_valid(musdb_tracks(musdb_path, "train"), valid_tracks)
    test = musdb_tracks(musdb_path, "test")
    if ccmixter_xml and model_config["task"] == "voice":
        train = train + ccmixter_tracks(ccmixter_xml)
    parts = {}
    for name, tracks in (("train", train), ("valid", valid), ("test", test)):
        print("Staging %s partition: %d tracks" % (name, len(tracks)))
        parts[name] = stage_partition(tracks, model_config, t_in, t_out, device)
    return Dataset(parts, model_config, t_in, t_out)
