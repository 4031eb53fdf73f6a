"""Device-side training-batch feeder (SURVEY 8(f) N4).

Replaces the reference's tf.data pipeline for the training partition - TFRecords -> take_random_snippets ->
random_amplify -> crop_sample -> shuffle -> batch (/root/reference/Datasets.py:16-19,196-214, Utils.py:26-42) - with a
track pool that lives in HBM and ONE kernel per batch (csrc/kernels_feed.cu, C-ABI wun_feed_batch).  The batch counter
is a device scalar the call advances itself, so `next_batch()` can be captured into the CUDA graph of a training step
and still produce a fresh batch on every replay.  There is no host fallback: without CUDA the constructor raises.
"""
import numpy as np


def synthetic_tracks(source_names, num_channels, n_tracks, frames, seed=0):
    """Random stand-in for a MUSDB-style dataset (no network / no audio files here): per track one float32 [frames, C]
    array per source plus the recorded mixture "mix" = sum of the sources (what Datasets.write_records stores)."""
    rng = np.random.default_rng(seed)
    tracks = []
    for _ in range(n_tracks):
        n = int(frames) if np.isscalar(frames) else int(rng.integers(frames[0], frames[1] + 1))
        t = {s: (rng.uniform(-1.0, 1.0, size=(n, num_channels)) / len(source_names)).astype(np.float32) for s in source_names}
        mix = np.zeros((n, num_channels), np.float32)
        for s in source_names:
            mix = mix + t[s]
        t["mix"] = mix
        tracks.append(t)
    return tracks


def build_pool(tracks, source_names):
    """[K + 1][total_frames][C] float32 pool (sources in source_names order, then "mix") + int64 offsets / lengths."""
    lengths = np.array([t["mix"].shape[0] for t in tracks], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64)
    keys = list(source_names) + ["mix"]
    pool = np.stack([np.concatenate([np.asarray(t[k], np.float32) for t in tracks], axis=0) for k in keys])
    return np.ascontiguousarray(pool), offsets, lengths


class DeviceFeeder(object):
    """feeder = DeviceFeeder(engine, tracks, source_names, batch, augmentation, seed, device)
    mix, targets = feeder.next_batch()      # CUDA tensors [B, T_in, C], [K, B, T_out, C]; re-used buffers

    `tracks`: list of {source_name: [frames, C] float32, ..., "mix": [frames, C]} (every track >= T_in + 1 frames)."""

    def __init__(self, engine, tracks, source_names, batch, augmentation=True, seed=1337, device="cuda", record_choice=False):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("DeviceFeeder needs a CUDA device: the feeder has no host fallback")
        pool, offsets, lengths = build_pool(tracks, list(source_names))
        self._setup(engine, torch.from_numpy(pool).to(torch.device(device)), offsets, lengths, source_names, batch,
                    augmentation, seed, record_choice)

    @classmethod
    def from_pool(cls, engine, pool, offsets, lengths, source_names, batch, augmentation=True, seed=1337, record_choice=False):
        """A feeder over an already staged device pool (Datasets.stage_partition): `pool` a float32 CUDA tensor
        [K + 1, total_frames, C], `offsets` / `lengths` int64 arrays of the tracks to draw from (each > T_in frames)."""
        self = cls.__new__(cls)
        self._setup(engine, pool, np.asarray(offsets, np.int64), np.asarray(lengths, np.int64), source_names, batch,
                    augmentation, seed, record_choice)
        return self

    def _setup(self, engine, pool, offsets, lengths, source_names, batch, augmentation, seed, record_choice):
        import torch
        self.eng, self.batch, self.augmentation, self.seed = engine, int(batch), bool(augmentation), int(seed)
        self.source_names = list(source_names)
        if len(lengths) == 0 or int(lengths.min()) <= engine.T_in:
            raise ValueError("every track needs more than T_in = %d frames (Datasets.py:18 draws start < length - T_in)" % engine.T_in)
        self.device = pool.device
        self.pool = pool
        self.track_offset = torch.from_numpy(offsets).to(self.device)
        self.track_length = torch.from_numpy(lengths).to(self.device)
        K, C = len(self.source_names), pool.shape[2]
        self.step_state = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.mix = torch.empty((self.batch, engine.T_in, C), dtype=torch.float32, device=self.device)
        self.targets = torch.empty((K, self.batch, engine.T_out, C), dtype=torch.float32, device=self.device)
        self.chosen = torch.zeros((self.batch, 2), dtype=torch.int64, device=self.device) if record_choice else None

    def next_batch(self):
        """Enqueue the feeder kernel on the current stream; returns the (re-used) mix / targets buffers."""
        self.eng.feed_batch(self.pool, self.track_offset, self.track_length, self.batch, self.augmentation, self.seed,
                            self.step_state, self.mix, self.targets, self.chosen)
        return self.mix, self.targets

    def bytes_per_batch(self):
        """Algorithmic HBM bytes of one batch: K source snippets (or the mix alone without augmentation... the sources are
        still read for the targets' centre part) read, mix + cropped targets written."""
        K, B, C = len(self.source_names), self.batch, self.mix.shape[2]
        t_in, t_out = self.eng.T_in, self.eng.T_out
        read = (K * t_in if self.augmentation else (t_in + K * t_out)) * C * 4 * B
        return read + (t_in + K * t_out) * C * 4 * B
