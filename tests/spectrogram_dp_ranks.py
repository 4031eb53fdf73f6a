"""One rank of the two-process data-parallel test of the spectrogram U-Net (tests/test_spectrogram_dp_gpu.py): both ranks run
on cuda:0 under the gloo backend.  The rank runs one synchronised step on its shard of a fixed batch, all-reduces the
gradients and writes what it holds, then trains three steps with Training.train(sync_batch_norm=True) and writes its state.
Kept out of the test module so that a spawned process imports only this."""
import os

import numpy as np
import torch

import Config
import Training
from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator
from oracle import spectrogram_oracle as S
from wun import parallel


def model_config(preset, L, Fi, T, **kw):
    return Config.build_config([preset], dict(num_layers=L, num_initial_filters=Fi, num_frames=T, **kw),
                               experiment_id=0)["model_config"]


def problem(L, Fi, B, T, seed):
    rng = np.random.default_rng(seed)
    params = S.random_params(L, Fi, seed=seed)
    t = np.arange(T) / 8192.0
    src = [np.stack([0.15 * np.sin(2 * np.pi * rng.uniform(80, 900) * t) + rng.uniform(-0.2, 0.2, T)
                     for _ in range(B)])[:, :, None].astype(np.float32) for _ in range(2)]
    return params, (src[0] + src[1]).astype(np.float32), src


def step_state(sep, cfg, B, T):
    """What one step left: loss, gradients, variables (moving statistics included), the last source's keep masks, batch
    statistics and activations, as numpy arrays keyed by name."""
    L = cfg["num_layers"]
    eng = sep.engine(num_frames=T)
    dev = sep.params.device
    out = {"loss": sep._loss.cpu().numpy().copy(), "grads": sep.grads.cpu().numpy().copy(),
           "params": sep.params.cpu().numpy().copy()}
    for d in range(L):
        out["level/%d" % d] = eng.debug_train_level(B, d, dev).cpu().numpy().copy()
        out["stats/down/%d" % d] = eng.debug_train_stats(B, d, False, dev).cpu().numpy().copy()
        if L - 4 <= d <= L - 2:
            out["keep/%d" % d] = eng.debug_train_keep(B, d, dev).cpu().numpy().copy()
    for i in range(L - 1):
        out["stats/up/%d" % i] = eng.debug_train_stats(B, i, True, dev).cpu().numpy().copy()
    return out


def one_step(cfg, params, mix, targets, shard=None):
    """One loss_and_gradients (of the shard of `shard`, then the gradient all-reduce) -> step_state."""
    T = mix.shape[1]
    sep = UnetSpectrogramSeparator(cfg)
    sep.load_variables(params, device=torch.device("cuda", 0), num_frames=T)
    mix_d, tg_d = torch.from_numpy(mix).cuda(), torch.from_numpy(np.stack(targets)).cuda()
    if shard is None:
        sep.loss_and_gradients(mix_d, tg_d)
        B = mix.shape[0]
    else:
        lo, B = shard.sample_offset, shard.local_batch
        sep.loss_and_gradients(mix_d[lo:lo + B].contiguous(), tg_d[:, lo:lo + B].contiguous(),
                               grad_scale=parallel.grad_scale_for(B, shard.global_batch), sync_batch_norm=shard)
        parallel.allreduce_gradients(sep.grads)
    torch.cuda.synchronize()
    return step_state(sep, cfg, B, T)


def train_three(cfg, params, T, tmp, world):
    """Training.train for 3 steps on SyntheticBatches (the same whole batches for every world size) -> final state."""
    cfg = dict(cfg, epoch_it=3, model_base_dir=os.path.join(tmp, "ck%d" % world), log_dir=os.path.join(tmp, "log"))
    sep = UnetSpectrogramSeparator(cfg)
    sep.load_variables(params, device=torch.device("cuda", 0), num_frames=T)
    in_shape, out_shape = sep.get_padding(np.array([cfg["batch_size"], T, 0]))
    src = Training.SyntheticBatches(cfg, in_shape, out_shape, seed=7)
    _, sep = Training.train(cfg, 0, batch_source=src, sep=sep, device=torch.device("cuda", 0), log_every=0,
                            sync_batch_norm=True)
    torch.cuda.synchronize()
    return {"params": sep.params.cpu().numpy(), "adam_m": sep.adam_m.cpu().numpy(), "adam_v": sep.adam_v.cpu().numpy(),
            "adam_state": sep._adam_state.cpu().numpy()}


def run_rank(rank, world, port, case, tmp):
    """Process entry: case = (preset, L, Fi, T, sizes, seed).  Writes tmp/rank<r>_step.npz and tmp/rank<r>_train.npz."""
    import torch.distributed as dist
    preset, L, Fi, T, sizes, seed = case
    B = sum(sizes)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        cfg = model_config(preset, L, Fi, T, batch_size=B)
        params, mix, targets = problem(L, Fi, B, T, seed)
        shard = parallel.BatchStatsGather(B)
        # the split under test, which may be one shard_range does not make (3 + 1)
        shard.sample_offset, shard.local_batch = sum(sizes[:rank]), sizes[rank]
        np.savez(os.path.join(tmp, "rank%d_step.npz" % rank), **one_step(cfg, params, mix, targets, shard))
        np.savez(os.path.join(tmp, "rank%d_train.npz" % rank), **train_three(cfg, params, T, tmp, world))
    finally:
        dist.destroy_process_group()
