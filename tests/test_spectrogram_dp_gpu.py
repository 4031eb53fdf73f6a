"""Data-parallel training of the spectrogram U-Net on one H100: wun_spec_forward_backward_dp at one rank against
wun_spec_forward_backward bit for bit, two processes on cuda:0 (gloo) against one process on the whole batch, and a CUDA
graph of a step through the gather callback.

Multi-GPU NCCL runs are not covered here (tools/spectrogram_dp_check.py is for a box with several GPUs).  Tolerances of the
two-process comparison: the ranks' per-channel sums are regrouped float64 sums of the one-process sums, so batch and moving
statistics (float32) agree to 1 ulp; the forward then differs in float32 rounding only, and the gradients, all-reduced in
float32, are held to test_spectrogram_train_gpu.py's bound: 1e-3 of each tensor's largest value, and for the biases that feed
batch norm (zero in exact arithmetic) 64 u times the oracle's magnitude bound of their cancelling sums."""
import multiprocessing
import os
import socket

import numpy as np
import pytest
import torch

from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator
from oracle import spectrogram_oracle as S
from oracle import spectrogram_train_oracle as O
from spectrogram_dp_ranks import model_config, one_step, problem, run_rank, step_state, train_three

pytestmark = pytest.mark.gpu

TOL = 1e-3
U = 2.0 ** -24


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)


def ulps(a, b):
    """Largest distance in float32 units in the last place (same-sign values)."""
    return int(np.abs(bits(a).astype(np.int64) - bits(b).astype(np.int64)).max())


class OneRank(object):
    """A one-rank shard whose gather is a device copy on the engine's stream."""

    def __init__(self, batch):
        self.rank, self.world, self.global_batch, self.sample_offset, self.local_batch = 0, 1, batch, 0, batch

    def gather(self, local, gathered, stream):
        with torch.cuda.stream(stream):
            gathered.copy_(local)


@pytest.mark.parametrize("preset", ["unet_spectrogram", "unet_spectrogram_l1"])
def test_one_rank_is_the_single_device_step_bit_for_bit(preset):
    L, Fi, B, T = 4, 3, 3, 1024 + 768 * 15
    cfg = model_config(preset, L, Fi, T)
    params, mix, targets = problem(L, Fi, B, T, seed=31)
    want = one_step(cfg, params, mix, targets)
    sep = UnetSpectrogramSeparator(cfg)
    sep.load_variables(params, device=torch.device("cuda", 0), num_frames=T)
    sep.loss_and_gradients(torch.from_numpy(mix).cuda(), torch.from_numpy(np.stack(targets)).cuda(),
                           sync_batch_norm=OneRank(B))
    torch.cuda.synchronize()
    got = step_state(sep, cfg, B, T)
    assert set(got) == set(want)
    for k in want:
        assert np.array_equal(bits(got[k]) if got[k].dtype != np.uint8 else got[k],
                              bits(want[k]) if want[k].dtype != np.uint8 else want[k]), k


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run_two_ranks(case, tmp):
    """Both ranks in spawned processes; always joined, and a straggler is terminated, whatever happens."""
    ctx = multiprocessing.get_context("spawn")
    port = free_port()
    procs = [ctx.Process(target=run_rank, args=(r, 2, port, case, str(tmp))) for r in range(2)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(600)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    assert [p.exitcode for p in procs] == [0, 0], [p.exitcode for p in procs]
    return [np.load(os.path.join(str(tmp), "rank%d_step.npz" % r)) for r in range(2)], \
        [np.load(os.path.join(str(tmp), "rank%d_train.npz" % r)) for r in range(2)]


def bn_fed_biases(table, L):
    """Flat slices of the conv biases that feed batch norm (every conv but the mask's)."""
    out = {}
    for n, _, o, c in table:
        if n.endswith("/bias") and c > 1:
            out[n] = (o, c)
    return out


CASES = [
    # (label, preset, layers, filters, T, shard sizes, seed)
    ("l3_u7_2+2", "unet_spectrogram", 3, 4, 1024 + 768 * 15, (2, 2), 5),
    ("l2_u7a_3+1", "unet_spectrogram_l1", 2, 4, 1024 + 768 * 7, (3, 1), 6),
]


@pytest.mark.parametrize("label,preset,L,Fi,T,sizes,seed", CASES, ids=[c[0] for c in CASES])
def test_two_ranks_take_the_one_process_step(tmp_path, label, preset, L, Fi, T, sizes, seed):
    B = sum(sizes)
    case = (preset, L, Fi, T, sizes, seed)
    ranks, trained = run_two_ranks(case, tmp_path)
    cfg = model_config(preset, L, Fi, T, batch_size=B)
    params, mix, targets = problem(L, Fi, B, T, seed)
    one = one_step(cfg, params, mix, targets)
    bounds = [(0, sizes[0]), (sizes[0], B)]

    # dropout masks: each shard's are the whole batch's of its examples
    for key in [k for k in one if k.startswith("keep/")]:
        for r, (lo, hi) in enumerate(bounds):
            assert np.array_equal(ranks[r][key], one[key][lo:hi]), (label, key, r)
    # batch statistics (the last source's) and moving statistics (all of them, in params)
    for key in [k for k in one if k.startswith("stats/")]:
        for r in range(2):
            assert ulps(ranks[r][key], one[key]) <= 1, (label, key, r, ulps(ranks[r][key], one[key]))
    eng = UnetSpectrogramSeparator(cfg).engine(num_frames=T)
    moving = [(n, o, c) for n, _, o, c in eng.param_table if not O.trainable(n)]
    for n, o, c in moving:
        for r in range(2):
            assert ulps(ranks[r]["params"][o:o + c], one["params"][o:o + c]) <= 1, (label, n, r)
    # the loss: the shards' means weighted by B_r / B
    loss = sum(float(ranks[r]["loss"][0]) * (hi - lo) / B for r, (lo, hi) in enumerate(bounds))
    assert abs(loss - float(one["loss"][0])) <= 1e-5 * abs(float(one["loss"][0])), (label, loss, one["loss"])
    # activation slopes that differ from the one-process step's (pre-activations within rounding of zero)
    flips = sum(int(((ranks[r]["level/%d" % d] > 0) != (one["level/%d" % d][lo:hi] > 0)).sum())
                for r, (lo, hi) in enumerate(bounds) for d in range(L))
    # gradients after the all-reduce: identical on both ranks, and the one-process gradients to test_spectrogram_train_gpu's
    # bound
    assert np.array_equal(bits(ranks[0]["grads"]), bits(ranks[1]["grads"]))
    scale = {}
    O.forward_backward(params, mix, targets, L, cfg["source_names"], cfg["raw_audio_loss"],
                       O.engine_masks(1337, 0, B, S.stft_frames(T), L, Fi), bias_scale=scale)
    fed = bn_fed_biases(eng.param_table, L)
    worst = {}
    for n, _, o, c in eng.param_table:
        if not O.trainable(n):
            continue
        got, want = ranks[0]["grads"][o:o + c].astype(np.float64), one["grads"][o:o + c].astype(np.float64)
        if n in fed:
            worst[n] = float(np.max(np.abs(got - want) / (2 * 64 * U * scale[n]))) * TOL
        else:
            worst[n] = float(np.abs(got - want).max() / np.abs(want).max())
    name = max(worst, key=worst.get)
    print("%s: %d activation slopes differ from the one-process step's; worst gradient %.2e (%s)"
          % (label, flips, worst[name], name))
    assert worst[name] < TOL, (label, name, worst[name], "slope flips", flips)

    # three Training.train steps: every rank holds the same state, close to the one-process run's
    for key in ("params", "adam_m", "adam_v", "adam_state"):
        assert np.array_equal(bits(trained[0][key]), bits(trained[1][key])), (label, key)
    single = train_three(cfg, params, T, str(tmp_path), 1)
    p0 = np.concatenate([np.asarray(params[n], np.float32).reshape(-1) for n, _, _, _ in eng.param_table])
    trainable = np.zeros(p0.size, bool)
    for n, _, o, c in eng.param_table:
        if O.trainable(n) and n not in fed:
            trainable[o:o + c] = True
    d_dp = trained[0]["params"][trainable].astype(np.float64) - p0[trainable]
    d_one = single["params"][trainable].astype(np.float64) - p0[trainable]
    rel = float(np.linalg.norm(d_dp - d_one) / np.linalg.norm(d_one))
    print("%s: 3 steps, update differs from the one-process run's by %.2e of its norm" % (label, rel))
    assert rel < 1e-2, (label, rel)
    for n, o, c in moving:
        assert np.allclose(trained[0]["params"][o:o + c], single["params"][o:o + c], rtol=1e-4, atol=1e-6), (label, n)


@pytest.mark.parametrize("preset", ["unet_spectrogram", "unet_spectrogram_l1"])
def test_captured_graph_through_the_gather_callback(preset):
    L, Fi, B, T, k, lr = 3, 4, 2, 1024 + 768 * 7, 3, 1e-3
    cfg = model_config(preset, L, Fi, T)
    params, mix, targets = problem(L, Fi, B, T, seed=17)
    mix_d, tg_d = torch.from_numpy(mix).cuda(), torch.from_numpy(np.stack(targets)).cuda()

    def make():
        sep = UnetSpectrogramSeparator(cfg)
        sep.load_variables(params, device=torch.device("cuda", 0), num_frames=T)
        sep._ensure_training_state()
        return sep

    eager = make()
    for _ in range(k):
        eager.loss_and_gradients(mix_d, tg_d)
        eager.adam_step(lr)
    graphed = make()
    shard = OneRank(B)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        # allocates the workspace and the gathered buffer outside the capture; the state it touched is reloaded below
        graphed.loss_and_gradients(mix_d, tg_d, sync_batch_norm=shard)
    torch.cuda.current_stream().wait_stream(side)
    graphed.load_variables({n: params[n] for n in params})
    graphed._ensure_training_state()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.loss_and_gradients(mix_d, tg_d, sync_batch_norm=shard)
        graphed.adam_step(lr)
    for _ in range(k):
        g.replay()
    torch.cuda.synchronize()
    assert bits(eager._loss.cpu().numpy()).tobytes() == bits(graphed._loss.cpu().numpy()).tobytes()
    for a, b in ((eager.params, graphed.params), (eager.adam_m, graphed.adam_m), (eager.adam_v, graphed.adam_v),
                 (eager._dropout_step, graphed._dropout_step)):
        assert np.array_equal(bits(a.cpu().numpy()), bits(b.cpu().numpy()))
    assert graphed.global_step == k
