"""Training entry point of the Wave-U-Net engine - stand-in for the reference's sacred experiment.

Keeps the reference's functions and command line (/root/reference/Training.py:24-166, README.md:84-92):

    python Training.py with cfg.baseline_stereo [cfg.model_config.batch_size=8 ...]
    torchrun --nproc-per-node 8 Training.py with cfg.full_multi_instrument        # data parallel

train()    one "epoch" of model_config["epoch_it"] steps (reference :103-109): every step is
           forward + MSE (:50-63) + backward + Adam(lr=init_sup_sep_lr) (:70-77), all inside libwun.so; with
           torch.distributed initialised the batch is sharded over the ranks and the flat gradient buffer is
           all-reduced once per step (NCCL).  Saves a TensorFlow-V2-format checkpoint (TFCheckpoint.py) of the
           "separator/..." variables, Adam slots and global_step, as the reference's Saver does (:98,113).
optimise() early stopping on a validation loss + fine-tuning stage with doubled batch and lr 1e-5 (:123-150).

The MUSDB/CCMixter TFRecord pipeline (Datasets.py) is out of scope; batches come from `batch_source`, by default the
synthetic generator of SURVEY 8(d) (uniform sources, random gains as Utils.random_amplify :26-36, centre-cropped
targets as Utils.crop_sample :38-42).
"""
import os
import sys
import time

import numpy as np

import Config
import TFCheckpoint
from Models.UnetAudioSeparator import UnetAudioSeparator
from wun import parallel


class SyntheticBatches(object):
    """Endless iterator of {"mix": [B,T_in,C], name: [B,T_out,C]} float32 numpy batches."""

    def __init__(self, model_config, input_shape, output_shape, seed=1337):
        self.cfg, self.in_shape, self.out_shape = model_config, input_shape, output_shape
        self.rng = np.random.default_rng(seed)

    def __iter__(self):
        return self

    def __next__(self):
        B, T_in, C = [int(v) for v in self.in_shape]
        T_out = int(self.out_shape[1])
        names = self.cfg["source_names"]
        crop = (T_in - T_out) // 2
        batch = {"mix": np.zeros((B, T_in, C), np.float32)}
        for name in names:
            s = self.rng.uniform(-1.0, 1.0, size=(B, T_in, C)).astype(np.float32) / np.float32(len(names))
            if self.cfg["augmentation"]:
                s *= self.rng.uniform(0.7, 1.0, size=(B, 1, 1)).astype(np.float32)     # Utils.py:33
            batch["mix"] += s
            batch[name] = np.ascontiguousarray(s[:, crop:T_in - crop] if crop > 0 else s)   # Utils.py:38-42
        return batch


def save_checkpoint(path, sep):
    """saver.save (reference :98,113).  `path` is a TF-V2 checkpoint prefix (<dir>/<experiment_id>-<global_step>, written as
    <prefix>.index + <prefix>.data-00000-of-00001 + the `checkpoint` state file); a path ending in .npz selects the
    round-1 numpy container instead.  Returns the path to hand to load_checkpoint / Predict.py."""
    return TFCheckpoint.save_separator(path, sep)


def load_checkpoint(path, sep, input_frames):
    """restorer.restore (reference :92-96): variables, Adam slots and global_step - from a checkpoint written here or by
    the reference's tf.train.Saver."""
    TFCheckpoint.restore_separator(path, sep, input_frames, with_optimizer=True)


def _to_device(batch, names, device):
    import torch
    mix = torch.from_numpy(batch["mix"]).to(device, non_blocking=True)
    tg = torch.stack([torch.from_numpy(batch[n]) for n in names]).to(device, non_blocking=True)
    return mix, tg


def _device_feeder(model_config, sep, eng, device, rank, world, local_batch):
    """The training data source when none is given: synthetic tracks resident in HBM + wun.feeder.DeviceFeeder (snippet
    sampling, random_amplify, centre crop in ONE kernel per batch: Datasets.py:196-214 / Utils.py:26-42 on the device).
    Built once per separator and input length, re-used by every later epoch; rank r draws its own shard of the batch."""
    from wun.feeder import DeviceFeeder, synthetic_tracks
    key = (eng.T_in, local_batch, str(device), bool(model_config["augmentation"]))
    if getattr(sep, "_feeder_key", None) != key:
        tracks = synthetic_tracks(model_config["source_names"], model_config["num_channels"], 8,
                                  (eng.T_in + 1 + eng.T_in // 4, 2 * eng.T_in), seed=4321)
        sep.last_feeder_tracks = tracks
        sep.last_feeder = DeviceFeeder(eng, tracks, model_config["source_names"], local_batch,
                                       augmentation=model_config["augmentation"], seed=1337 + 7919 * rank, device=device)
        sep._feeder_key = key
    return sep.last_feeder


def train(model_config, experiment_id, load_model=None, batch_source=None, sep=None, device=None, log_every=100, feeder=None):
    """One epoch (reference train(), :24-121).  Returns (checkpoint path, separator).
    Data: `batch_source` (an iterator of host numpy batches, e.g. SyntheticBatches) if given; otherwise, on a CUDA device,
    the device-side feeder (`feeder="device"`, the default there); `feeder="host"` forces the numpy generator."""
    import torch
    rank, world = parallel.world()
    if device is None:
        device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    if model_config["network"] != "unet":
        raise NotImplementedError                                   # reference :33 (unet_spectrogram is out of scope)
    if sep is None:
        sep = UnetAudioSeparator(model_config)
    disc_input_shape = [model_config["batch_size"], model_config["num_frames"], 0]
    in_shape, out_shape = sep.get_padding(np.array(disc_input_shape))                 # :35
    t_in = int(in_shape[1])
    eng = sep.engine(input_frames=t_in)
    if load_model is not None and sep.params is None:
        load_checkpoint(load_model, sep, t_in)
    sep._ensure_params(eng, device, create=True)
    sep._ensure_training_state()
    parallel.broadcast_parameters(sep.params)
    names = model_config["source_names"]
    lr = model_config["init_sup_sep_lr"]
    global_batch = int(in_shape[0])
    dev_feeder = None
    if batch_source is None and feeder != "host" and device.type == "cuda":
        lo, hi = parallel.shard_range(global_batch, rank, world)
        local_batch = hi - lo
        dev_feeder = _device_feeder(model_config, sep, eng, device, rank, world, local_batch)
    elif batch_source is None:
        batch_source = SyntheticBatches(model_config, in_shape, out_shape, seed=1337 + sep.global_step)
    running, t0 = 0.0, time.time()
    # N > 1: the gradient all-reduce runs bucketed on a communication stream while backward still computes
    overlap = parallel.BucketedAllReduce(eng, sep.grads) if (world > 1 and sep.grads.is_cuda) else None
    for it in range(model_config["epoch_it"]):                      # :103
        if dev_feeder is not None:
            mix_l, tg_l = dev_feeder.next_batch()                   # this rank's shard, built on the device
        else:
            mix, tg = _to_device(next(batch_source), names, device)
            mix_l = parallel.shard_batch(mix, rank, world).contiguous()
            tg_l = parallel.shard_batch(tg, rank, world, dim=1).contiguous()
        loss = sep.loss_and_gradients(mix_l, tg_l, grad_scale=parallel.grad_scale_for(mix_l.shape[0], global_batch))
        if overlap is not None:
            overlap.run()
        else:
            parallel.allreduce_gradients(sep.grads)
        sep.adam_step(lr)
        if log_every and (it + 1) % log_every == 0 and rank == 0:
            running = float(loss.item())
            print("step %d  sep_loss(local shard) %.6f  %.1f steps/s" % (sep.global_step, running,
                                                                         (it + 1) / (time.time() - t0)))
    path = None
    if rank == 0:
        path = save_checkpoint(os.path.join(model_config["model_base_dir"], str(experiment_id),
                                            "%s-%d" % (experiment_id, sep.global_step)), sep)
    return path, sep


def validation_loss(model_config, sep, batches=4, seed=99):
    """Running-mean MSE over a fixed synthetic validation set (reference Test.test, Test.py:57-71)."""
    import torch
    in_shape, out_shape = sep.get_padding(np.array([model_config["batch_size"], model_config["num_frames"], 0]))
    src = SyntheticBatches(model_config, in_shape, out_shape, seed=seed)
    names = model_config["source_names"]
    tot, n = 0.0, 0
    for _ in range(batches):
        b = next(src)
        mix = torch.from_numpy(b["mix"]).to(sep.params.device)
        out = sep.get_output(mix, training=False, reuse=True)
        loss = sum(float(torch.mean((torch.from_numpy(b[k]).to(mix.device) - out[k]) ** 2)) for k in names) / len(names)
        tot += loss; n += 1
    return tot / n


def optimise(model_config, experiment_id, max_epochs=None):
    """Early stopping + fine-tuning (reference optimise(), :123-150)."""
    epoch, best_loss, model_path, best_model_path, sep = 0, 10000, None, None, None
    for i in range(2):
        worse_epochs = 0
        if i == 1:
            print("Finished first round of training, now entering fine-tuning stage")
            model_config["batch_size"] *= 2
            model_config["init_sup_sep_lr"] = 1e-5
        while worse_epochs < model_config["worse_epochs"]:
            if max_epochs is not None and epoch >= max_epochs:
                break
            print("EPOCH: " + str(epoch))
            model_path, sep = train(model_config, experiment_id, load_model=model_path, sep=sep)
            curr_loss = validation_loss(model_config, sep)
            epoch += 1
            if curr_loss < best_loss:
                worse_epochs = 0
                print("Performance on validation set improved from " + str(best_loss) + " to " + str(curr_loss))
                best_model_path, best_loss = model_path, curr_loss
            else:
                worse_epochs += 1
                print("Performance on validation set worsened to " + str(curr_loss))
    return best_model_path, best_loss


def run(cfg, max_epochs=None):
    model_config = cfg["model_config"]
    print("SCRIPT START")
    for d in [model_config["model_base_dir"], model_config["log_dir"]]:
        os.makedirs(d, exist_ok=True)
    if "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    sup_model_path, sup_loss = optimise(model_config, cfg["experiment_id"], max_epochs=max_epochs)
    print("Supervised training finished! Saved model at " + str(sup_model_path) + ". Performance: " + str(sup_loss))
    return sup_model_path, sup_loss


if __name__ == "__main__":
    cfg, extras = Config.parse_command_line(sys.argv[1:])
    run(cfg, max_epochs=extras.get("max_epochs"))
