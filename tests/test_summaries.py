"""TensorBoard event files (wave-u-net_b200/Summaries.py) without a GPU: byte equality with TensorBoard's own
EventFileWriter, TensorBoard's loader reading our files, the reader's CRC checks, unique file names, and the whole-batch
loss history that data-parallel training logs (wun/parallel.py batch_loss_history) at world size 2 on gloo."""
import glob
import os
import socket
import struct
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import Summaries

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def events_files(logdir):
    return sorted(glob.glob(os.path.join(str(logdir), "*tfevents*")))


def first_record_length(data):
    return 12 + struct.unpack_from("<Q", data, 0)[0] + 4


def test_scalar_event_known_bytes():
    assert Summaries.encode_event(1.5, 7, tag="sep_loss", value=0.25).hex() == \
        "09000000000000f83f10072a110a0f0a087365705f6c6f7373150000803e"
    e = Summaries.decode_event(Summaries.encode_event(1.5, 7, tag="sep_loss", value=0.25))
    assert (e["wall_time"], e["step"], e["file_version"], e["values"]) == (1.5, 7, None, [("sep_loss", 0.25)])


def test_value_is_rounded_to_float32_and_step_zero_round_trips(tmp_path):
    v = 0.1 + 1e-12                                      # float64, not a float32 value
    with Summaries.EventFileWriter(str(tmp_path)) as w:
        w.add_scalar("test_loss", v, 0, wall_time=2.0)
        w.add_scalar("test_loss", v, -3, wall_time=3.0)
    got = Summaries.read_scalars(w.path)
    assert [(t, s, tag) for t, s, tag, _ in got] == [(2.0, 0, "test_loss"), (3.0, -3, "test_loss")]
    assert all(np.float32(x).tobytes() == np.float32(v).tobytes() for _, _, _, x in got)


CASES = [(1.5, 7, "sep_loss", 0.25), (1700000000.123456, 0, "sep_loss", 0.0), (1700000001.5, 123456789012, "test_loss", 3.0e-7),
         (2.25, 1, "sep_loss", float("inf")), (1e9, 2 ** 40 + 3, "a/b", -1.75)]


def test_files_equal_tensorboards_event_file_writer_byte_for_byte(tmp_path):
    pytest.importorskip("tensorboard")
    from tensorboard.compat.proto import event_pb2, summary_pb2
    from tensorboard.summary.writer.event_file_writer import EventFileWriter
    tb_dir, our_dir = tmp_path / "tb", tmp_path / "ours"
    tb = EventFileWriter(str(tb_dir))
    with Summaries.EventFileWriter(str(our_dir)) as ours:
        for wall, step, tag, value in CASES:
            s = summary_pb2.Summary(value=[summary_pb2.Summary.Value(tag=tag, simple_value=value)])
            tb.add_event(event_pb2.Event(wall_time=wall, step=step, summary=s))
            ours.add_scalar(tag, value, step, wall)
    tb.close()
    (tb_path,), (our_path,) = events_files(tb_dir), events_files(our_dir)
    tb_data, our_data = open(tb_path, "rb").read(), open(our_path, "rb").read()
    # after the file_version record: the same records, framing included
    n_tb, n_ours = first_record_length(tb_data), first_record_length(our_data)
    assert our_data[n_ours:] == tb_data[n_tb:]
    assert len(our_data[n_ours:]) > 0
    # the file_version records differ only in the wall time each writer stamps - and in the source_metadata (Event field
    # 10) that TensorBoard's writer adds to name itself, which TensorFlow 1's FileWriter does not write
    tb_first = event_pb2.Event.FromString(Summaries.read_records(tb_path)[0])
    our_first = event_pb2.Event.FromString(Summaries.read_records(our_path)[0])
    assert tb_first.file_version == our_first.file_version == "brain.Event:2"
    tb_first.ClearField("source_metadata")
    assert Summaries.encode_event(tb_first.wall_time, file_version="brain.Event:2") == tb_first.SerializeToString()
    assert not our_first.HasField("source_metadata") and our_first.step == 0
    assert abs(our_first.wall_time - tb_first.wall_time) < 60


def test_tensorboards_loader_reads_our_files_and_our_reader_checks_crcs(tmp_path):
    pytest.importorskip("tensorboard")
    from tensorboard.backend.event_processing import event_file_loader
    from tensorboard.util import tensor_util
    with Summaries.EventFileWriter(str(tmp_path)) as w:
        for wall, step, tag, value in CASES:
            w.add_scalar(tag, value, step, wall)
    events = list(event_file_loader.EventFileLoader(w.path).Load())
    assert events[0].file_version == "brain.Event:2" and len(events) == 1 + len(CASES)
    tb = []
    for e in events[1:]:
        (v,) = e.summary.value
        x = v.simple_value if v.WhichOneof("value") == "simple_value" else float(tensor_util.make_ndarray(v.tensor))
        tb.append((e.wall_time, e.step, v.tag, x))
    want = [(wall, step, tag, float(np.float32(value))) for wall, step, tag, value in CASES]
    assert tb == want
    assert Summaries.read_scalars(w.path) == want
    data = bytearray(open(w.path, "rb").read())
    n0 = first_record_length(data)
    for at in (3, 9, n0 + 14, len(data) - 1):              # length, its CRC, a payload byte, the last payload CRC byte
        bad = bytearray(data)
        bad[at] ^= 0x01
        p = tmp_path / ("bad_%d" % at)
        p.write_bytes(bytes(bad))
        with pytest.raises(Summaries.EventFileError):
            Summaries.read_scalars(str(p))
    p = tmp_path / "truncated"
    p.write_bytes(bytes(data[:-2]))
    with pytest.raises(Summaries.EventFileError, match="truncated"):
        Summaries.read_scalars(str(p))


def test_two_writers_in_the_same_second_write_two_files(tmp_path):
    a = Summaries.EventFileWriter(str(tmp_path))
    b = Summaries.EventFileWriter(str(tmp_path))
    a.add_scalar("sep_loss", 1.0, 0, 1.0)
    b.add_scalar("sep_loss", 2.0, 0, 1.0)
    a.close(); b.close()
    assert a.path != b.path and events_files(tmp_path) == sorted([a.path, b.path])
    name = os.path.basename(a.path).split(".")
    assert name[:3] == ["events", "out", "tfevents"] and len(name[3]) == 10
    assert ".".join(name[4:-2]) == socket.gethostname() and name[-2] == str(os.getpid())
    assert [x[3] for x in Summaries.read_scalars(a.path)] == [1.0] and [x[3] for x in Summaries.read_scalars(b.path)] == [2.0]


def test_write_scalar_is_one_file_with_one_event(tmp_path):
    path = Summaries.write_scalar(str(tmp_path / "new" / "dir"), "test_loss", 0.5, 12)
    assert events_files(tmp_path / "new" / "dir") == [path]
    ((wall, step, tag, value),) = Summaries.read_scalars(path)
    assert (step, tag, value) == (12, "test_loss", 0.5) and wall > 1e9


# ---- data parallel: the logged sep_loss is the whole batch's loss ----------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _batch_loss(cfg, params, mix, targets):
    from oracle import wave_unet_oracle as O
    out = O.forward_np(cfg, params, mix, True, dtype=torch.float64)
    return sum(np.mean((targets[k].astype(np.float64) - out[k]) ** 2) for k in cfg["source_names"]) / len(cfg["source_names"])


def _worker(rank, world, port, out):
    sys.path.insert(0, REPO); sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
    import Config
    from oracle import wave_unet_oracle as O
    from wun import parallel
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.set_num_threads(2)
        cfg = Config.build_config(["baseline_stereo"], dict(num_layers=3, num_initial_filters=8), experiment_id=0)["model_config"]
        t_in, t_out = O.get_padding(cfg, 40)
        params = O.init_params(cfg, seed=5)
        B = 5                                           # uneven split: ranks get 3 and 2 examples
        lo, hi = parallel.shard_range(B, rank, world)
        local, whole = [], []
        for step in range(3):
            mix, targets = O.synthetic_batch(cfg, B, t_in, t_out, seed=20 + step)
            local.append(_batch_loss(cfg, params, mix[lo:hi], {k: v[lo:hi] for k, v in targets.items()}))
            whole.append(_batch_loss(cfg, params, mix, targets))
        h64 = parallel.batch_loss_history(torch.tensor(local, dtype=torch.float64), hi - lo, B)
        h32 = parallel.batch_loss_history(torch.tensor(local, dtype=torch.float32), hi - lo, B)
        out.put((rank, (lo, hi), local, h64.tolist(), h32.tolist(), whole))
    finally:
        dist.destroy_process_group()


def test_data_parallel_loss_history_is_the_whole_batch_loss_gloo():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    res = sorted(q.get(timeout=5) for _ in range(world))
    assert [r[1] for r in res] == [(0, 3), (3, 5)]
    whole = np.array(res[0][5])
    assert res[0][2] != res[1][2]                           # the shards' own losses differ from each other
    for _, _, _, h64, h32, _ in res:                        # every rank ends with the whole batch's losses
        assert np.allclose(h64, whole, rtol=1e-12, atol=0), (h64, whole)
        assert np.allclose(h32, whole, rtol=1e-6, atol=0), (h32, whole)
    assert res[0][3] == res[1][3] and res[0][4] == res[1][4]


def test_batch_loss_history_is_the_identity_without_a_process_group():
    from wun import parallel
    h = torch.tensor([0.5, 0.25], dtype=torch.float64)
    assert parallel.batch_loss_history(h, 3, 5) is h and h.tolist() == [0.5, 0.25]
