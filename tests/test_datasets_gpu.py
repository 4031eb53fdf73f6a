"""Dataset layer on the GPU: staged pools against the numpy oracle bit for bit, wun_snippet_batch and wun_eval_batch_loss
(csrc/kernels_eval.cu) eager and graph-replayed, Test.test against a per-batch composition and the oracle forward, and
Training.run(dataset="musdb") end to end on a tiny MUSDB-layout dataset."""
import glob
import math
import os
import struct

import numpy as np
import pytest
import torch

import Config
import Datasets
import Evaluate
import Test
import Training
import wun
from dataset_fixtures import TEST, TRAIN, write_ccmixter, write_musdb
from Models.UnetAudioSeparator import UnetAudioSeparator
from oracle import dataset_oracle as D
from oracle import wave_unet_oracle as O

pytestmark = pytest.mark.gpu

T_IN, T_OUT = 151, 41


def mc(named="baseline_stereo", **kw):
    kw.setdefault("num_layers", 2)
    kw.setdefault("num_frames", 40)
    return Config.build_config([named], kw, experiment_id=0)["model_config"]


def tables(a, b):
    return wun.resample_tables(a, b) + (wun.KAISER_BEST_PRECISION,)


def oracle_paths(track):
    return {k: track[k] for k in track if k != "name"}


@pytest.mark.parametrize("named", ["baseline_stereo", "baseline_context", "full_multi_instrument"])
def test_staged_pool_equals_oracle(tmp_path, named):
    cfg = mc(named)
    musdb = write_musdb(str(tmp_path / "musdb"))
    tracks = Datasets.musdb_tracks(musdb, "train") + Datasets.musdb_tracks(musdb, "test")
    if cfg["task"] == "voice":
        tracks += Datasets.ccmixter_tracks(write_ccmixter(str(tmp_path)))
    timings = {}
    part = Datasets.stage_partition(tracks, cfg, T_IN, T_OUT, timings=timings)
    assert set(timings) == {"read", "upload", "resample"}
    pool = part.pool.cpu().numpy()
    keys = cfg["source_names"] + ["mix"]
    assert pool.shape == (len(keys), int(part.lengths.sum()), cfg["num_channels"])
    for t, off, length in zip(tracks, part.offsets, part.lengths):
        want = D.stage_track(oracle_paths(t), cfg["source_names"], cfg["mono_downmix"], cfg["expected_sr"], T_IN, T_OUT, tables)
        for k, key in enumerate(keys):
            assert want[key].shape[0] == length
            assert np.array_equal(pool[k, off:off + length].view(np.uint32), want[key].view(np.uint32)), (t["name"], key)


def make_pool(K, C, frames, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand((K + 1, frames, C), generator=g).sub_(0.5).cuda()


@pytest.mark.parametrize("K,C,B", [(2, 2, 3), (4, 1, 2), (2, 1, 5)])
def test_snippet_batch_is_bit_exact_with_counter_and_graph(K, C, B):
    pool = make_pool(K, C, 4000, seed=K * 10 + C)
    rng = np.random.default_rng(B)
    n_batches = 4
    pos_np = rng.integers(0, 4000 - T_IN, size=n_batches * B).astype(np.int64)
    pos = torch.from_numpy(pos_np).cuda()
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    mix = torch.empty((B, T_IN, C), device="cuda")
    tg = torch.empty((K, B, T_OUT, C), device="cuda")
    p = pool.cpu().numpy()
    crop = (T_IN - T_OUT) // 2

    def want(i):
        s = pos_np[(i % n_batches) * B:(i % n_batches + 1) * B]
        return (np.stack([p[K, f:f + T_IN] for f in s]),
                np.stack([np.stack([p[k, f + crop:f + crop + T_OUT] for f in s]) for k in range(K)]))

    for i in range(n_batches + 1):                       # the counter wraps to batch 0 after the last one
        wun.snippet_batch(pool, pos, B, counter, mix, tg)
        m, t = want(i)
        assert np.array_equal(mix.cpu().numpy(), m) and np.array_equal(tg.cpu().numpy(), t), i
        assert int(counter.item()) == i + 1
    counter.zero_()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g = torch.cuda.CUDAGraph()
        g.capture_begin()
        wun.snippet_batch(pool, pos, B, counter, mix, tg)
        g.capture_end()
    torch.cuda.current_stream().wait_stream(side)
    for i in range(n_batches):
        g.replay()
        torch.cuda.synchronize()
        m, t = want(i)
        assert np.array_equal(mix.cpu().numpy(), m) and np.array_equal(tg.cpu().numpy(), t), ("replay", i)
    assert int(counter.item()) == n_batches
    with pytest.raises(wun.WunError):                    # positions must be whole batches
        wun.snippet_batch(pool, pos[:-1], B, counter, mix, tg)


def fsum_loss(out, tg):
    o, t = out.cpu().numpy().astype(np.float64), tg.cpu().numpy().astype(np.float64)
    K = o.shape[0]
    return math.fsum(math.fsum(((t[k] - o[k]) ** 2).ravel()) / o[k].size for k in range(K)) / K


def bits(x):
    return struct.pack("<d", float(x))


@pytest.mark.parametrize("shape", [(2, 16, 16389, 2), (4, 3, 41, 1), (1, 1, 7, 1), (2, 5, 1000, 2)])
def test_eval_batch_loss_matches_fsum_and_repeats_bits(shape):
    g = torch.Generator().manual_seed(sum(shape))
    out = torch.rand(shape, generator=g).cuda()
    tg = torch.rand(shape, generator=g).mul_(2).sub_(1).cuda()
    K = shape[0]
    ws = torch.empty(K * wun.EVAL_LOSS_CTAS, dtype=torch.float64, device="cuda")
    state = torch.zeros(2, dtype=torch.float64, device="cuda")
    curr = torch.zeros(1, dtype=torch.float64, device="cuda")
    wun.eval_batch_loss(out, tg, state, ws, curr)
    want = fsum_loss(out, tg)
    got = float(curr.item())
    assert abs(got - want) <= 1e-12 * abs(want), (got, want)
    assert float(state[0].item()) == got and float(state[1].item()) == 1.0
    ref_bits = bits(got)
    for _ in range(3):
        state.zero_()
        wun.eval_batch_loss(out, tg, state, ws, curr)
        assert bits(curr.item()) == ref_bits and bits(state[0].item()) == ref_bits
    # graph-replayed: the running mean over n identical batches stays at curr up to the update's rounding; compare with
    # the same recurrence evaluated in Python doubles (no FMA)
    state.zero_()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        gr = torch.cuda.CUDAGraph()
        gr.capture_begin()
        wun.eval_batch_loss(out, tg, state, ws, curr)
        gr.capture_end()
    torch.cuda.current_stream().wait_stream(side)
    total = 0.0
    for n in range(1, 6):
        gr.replay()
        total = total + (1.0 / float(n)) * (got - total)
    torch.cuda.synchronize()
    assert bits(curr.item()) == ref_bits and bits(state[0].item()) == bits(total) and float(state[1].item()) == 5.0


@pytest.fixture(scope="module")
def tiny_dataset(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("ds"))
    return write_musdb(os.path.join(root, "musdb")), write_ccmixter(root)


@pytest.mark.parametrize("named,B", [("baseline_stereo", 4), ("baseline_context", 3)])
def test_test_equals_per_batch_composition_and_oracle(tiny_dataset, named, B):
    musdb, xml = tiny_dataset
    cfg = mc(named, batch_size=B)
    ds = Datasets.load_musdb(cfg, T_IN, T_OUT, musdb, xml, valid_tracks=2)
    params = O.init_params(cfg, seed=5)
    sep = UnetAudioSeparator(cfg)
    sep.load_variables(params, input_frames=T_IN)
    for part in ("valid", "test"):
        got = Test.test(cfg, part, "0", None, dataset=ds, separator=sep)
        again = Test.test(cfg, part, "0", None, dataset=ds, separator=sep)
        assert bits(got) == bits(again)
        print("partition loss %s %s: %r (%s)" % (named, part, got, bits(got).hex()))
        p = ds.partitions[part]
        pos = Datasets.snippet_positions(p.offsets, p.lengths, T_IN, T_OUT, B)
        pool = p.pool.cpu().numpy()
        crop = (T_IN - T_OUT) // 2
        eng = sep.engine(input_frames=T_IN)
        total = 0.0
        for n, b0 in enumerate(range(0, len(pos), B), start=1):
            s = pos[b0:b0 + B]
            mix = np.stack([pool[-1, f:f + T_IN] for f in s])
            tg = np.stack([np.stack([pool[k, f + crop:f + crop + T_OUT] for f in s]) for k in range(len(cfg["source_names"]))])
            out = eng.forward(sep.params, torch.from_numpy(mix).cuda(), False).cpu().numpy()
            curr = sum(np.mean((tg[k].astype(np.float64) - out[k]) ** 2) for k in range(len(tg))) / len(tg)
            total = total + (1.0 / n) * (curr - total)
        assert abs(got - total) <= 1e-12 * abs(total), (part, got, total)
        # the oracle: staged tracks, take_all_snippets, drop-remainder batching, float32 CPU forward
        tracks = [D.stage_track(oracle_paths(t), cfg["source_names"], cfg["mono_downmix"], cfg["expected_sr"], T_IN, T_OUT,
                                tables) for t in _partition_tracks(musdb, xml, part)]
        batches = D.partition_batches(tracks, cfg["source_names"], T_IN, T_OUT, B)
        assert len(batches) == len(pos) // B
        want = D.test_loss(batches, lambda m: O.forward_np(cfg, params, m, False), cfg["source_names"])
        assert abs(got - want) <= 1e-5 * abs(want), (part, got, want)


def _partition_tracks(musdb, xml, part):
    train, valid = Datasets.split_valid(Datasets.musdb_tracks(musdb, "train"), 2)
    return valid if part == "valid" else Datasets.musdb_tracks(musdb, "test")


def test_test_rejects_a_partition_without_one_batch(tiny_dataset):
    musdb, xml = tiny_dataset
    cfg = mc(batch_size=64)
    ds = Datasets.load_musdb(cfg, T_IN, T_OUT, musdb, None, valid_tracks=1)
    sep = UnetAudioSeparator(cfg)
    sep.load_variables(O.init_params(cfg, seed=1), input_frames=T_IN)
    with pytest.raises(ValueError, match="fewer than one batch"):
        Test.test(cfg, "valid", "0", None, dataset=ds, separator=sep)


def test_training_run_on_musdb_end_to_end(tmp_path, capsys):
    # MUSDB18 is stereo: every stem of this dataset is, so that the stereo model's estimates can be scored against them
    stereo = lambda spec: {n: (rate, frames, 2, fmt) for n, (rate, frames, _, fmt) in spec.items()}
    musdb = write_musdb(str(tmp_path / "musdb"), stereo(TRAIN), stereo(TEST))
    xml = write_ccmixter(str(tmp_path))
    cfg = Config.build_config(["baseline_stereo"], dict(
        num_layers=2, num_frames=40, batch_size=2, epoch_it=3, worse_epochs=1, musdb_path=musdb,
        model_base_dir=str(tmp_path / "ck"), log_dir=str(tmp_path / "logs"), estimates_path=str(tmp_path / "est")),
        experiment_id=7)
    path, loss = Training.run(cfg, max_epochs=2, dataset="musdb", ccmixter_xml=xml, valid_tracks=2)
    out = capsys.readouterr().out
    assert "TRAINING FINISHED - TESTING WITH BEST MODEL" in out
    assert np.isfinite(loss) and loss > 0
    assert os.path.exists(path + ".index") and os.path.dirname(path) == str(tmp_path / "ck" / "7")
    assert cfg["model_config"]["batch_size"] == 4                      # the fine-tuning stage doubled it
    est = str(tmp_path / "est")
    for subset in ("train", "test"):
        names = [t["name"] for t in Datasets.musdb_tracks(musdb, subset)]
        for name in names:
            for s in cfg["model_config"]["source_names"]:
                assert os.path.exists(Datasets.estimate_path(est, subset, name, s)), (subset, name, s)
        jsons = sorted(os.path.basename(p) for p in glob.glob(os.path.join(Datasets.museval_json_dir(est, subset), "*.json")))
        assert jsons == sorted(n + ".json" for n in names)
        metrics = Evaluate.compute_mean_metrics(Datasets.museval_json_dir(est, subset))
        assert len(metrics) == 2
        if subset == "test":                                           # t_long is scored over one whole second
            assert all(np.isfinite(m[0]) for m in metrics), metrics
    assert sorted(TEST) == sorted(t["name"] for t in Datasets.musdb_tracks(musdb, "test"))
