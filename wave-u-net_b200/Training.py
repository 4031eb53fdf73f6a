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

run(), and so the command line, writes the reference's TensorBoard summaries (Summaries.py) into
model_config["log_dir"]/<experiment_id>: a `sep_loss` scalar at every training step (:80-81,88,106) and a `test_loss` scalar
after every validation and the final test (Test.py:41,81-82).  train, optimise, validation_loss and Test.test take
summaries=False by default and write nothing.  The FileWriter's graph events are not written: there is no TensorFlow graph.

By default batches come from `batch_source`, by default the synthetic generator of SURVEY 8(d) (uniform sources, random
gains as Utils.random_amplify :26-36, centre-cropped targets as Utils.crop_sample :38-42).  Training on real music is
opt-in with a top-level extra:

    python Training.py with cfg.full model_config.musdb_path=/data/musdb18 dataset=musdb [ccmixter_xml=...] [valid_tracks=N]

which stages the MUSDB18 WAV dataset on the device (Datasets.py), validates with Test.test, returns the best checkpoint's
test loss and writes its estimates and BSS Eval JSONs (Evaluate.produce_musdb_source_estimates), as the reference does.

network="unet_spectrogram" (presets cfg.unet_spectrogram / U7 and cfg.unet_spectrogram_l1 / U7a) trains the spectrogram
U-Net the same way (Models/UnetSpectrogramSeparator.py).  Its batch norm normalises with the statistics of the whole batch,
so data parallelism is opt-in, as torch's SyncBatchNorm is:

    torchrun --nproc-per-node 8 Training.py with cfg.unet_spectrogram sync_batch_norm=1

gathers every batch-norm layer's per-channel sums from all ranks at every step, so that each step is the one-GPU step on the
whole batch up to the order of floating-point sums.  Without sync_batch_norm a data-parallel run of it is refused.
"""
import os
import sys
import time

import numpy as np

import Config
import Summaries
import TFCheckpoint
from Models.UnetAudioSeparator import UnetAudioSeparator
from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator
from wun import parallel


def separator_class(model_config):
    """The separator model_config["network"] names (reference Training.py:30-33)."""
    if model_config["network"] == "unet":
        return UnetAudioSeparator
    if model_config["network"] == "unet_spectrogram":
        return UnetSpectrogramSeparator
    raise NotImplementedError(model_config["network"])


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


def _device_feeder(model_config, sep, eng, device, rank, world, local_batch, dataset=None):
    """The training data source when none is given: synthetic tracks resident in HBM + wun.feeder.DeviceFeeder (snippet
    sampling, random_amplify, centre crop in ONE kernel per batch: Datasets.py:196-214 / Utils.py:26-42 on the device).
    Built once per separator and input length, re-used by every later epoch; rank r draws its own shard of the batch.
    With `dataset` (a Datasets.Dataset) the feeder draws from its staged train partition instead."""
    from wun.feeder import DeviceFeeder, synthetic_tracks
    key = (eng.T_in, local_batch, str(device), bool(model_config["augmentation"]))
    if dataset is not None:
        key += (id(dataset),)
        if getattr(sep, "_feeder_key", None) != key:
            sep.last_feeder_tracks = None
            sep.last_feeder = dataset.train_feeder(eng, local_batch, augmentation=model_config["augmentation"],
                                                   seed=1337 + 7919 * rank)
            sep._feeder_key = key
        return sep.last_feeder
    if getattr(sep, "_feeder_key", None) != key:
        tracks = synthetic_tracks(model_config["source_names"], model_config["num_channels"], 8,
                                  (eng.T_in + 1 + eng.T_in // 4, 2 * eng.T_in), seed=4321)
        sep.last_feeder_tracks = tracks
        sep.last_feeder = DeviceFeeder(eng, tracks, model_config["source_names"], local_batch,
                                       augmentation=model_config["augmentation"], seed=1337 + 7919 * rank, device=device)
        sep._feeder_key = key
    return sep.last_feeder


def train(model_config, experiment_id, load_model=None, batch_source=None, sep=None, device=None, log_every=100, feeder=None,
          dataset=None, summaries=False, sync_batch_norm=False):
    """One epoch (reference train(), :24-121).  Returns (checkpoint path, separator).
    Data: `batch_source` (an iterator of host numpy batches, e.g. SyntheticBatches) if given; otherwise, on a CUDA device,
    the device-side feeder (`feeder="device"`, the default there); `feeder="host"` forces the numpy generator.  With
    `dataset` (a Datasets.Dataset) the device-side feeder draws from its train partition.
    With `summaries`, rank 0 writes a new TensorBoard events file into log_dir/<experiment_id> (:80-81,88,106): one
    `sep_loss` scalar per step, the whole batch's loss of the forward pass before that step's update, at the global step
    before it.  The losses stay on the device until the epoch ends, so logging adds no host synchronisation per step.
    With `sync_batch_norm`, the spectrogram U-Net trains data parallel: every rank's batch norm uses the whole batch's
    statistics (wun.parallel.BatchStatsGather).  The Wave-U-Net has no batch norm and ignores it."""
    import torch
    rank, world = parallel.world()
    if device is None:
        device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    cls = separator_class(model_config)                             # reference :30-33
    spectrogram = cls is UnetSpectrogramSeparator
    if spectrogram and world > 1 and not sync_batch_norm:
        raise ValueError("the spectrogram U-Net trains on one GPU unless sync_batch_norm=True: with %d ranks every rank would "
                         "normalise with its own shard's batch statistics, which changes the model" % world)
    if sep is None:
        sep = cls(model_config)
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
    shard = parallel.BatchStatsGather(global_batch) if (spectrogram and world > 1) else None
    dev_feeder = None
    if batch_source is None and feeder != "host" and device.type == "cuda":
        lo, hi = parallel.shard_range(global_batch, rank, world)
        local_batch = hi - lo
        dev_feeder = _device_feeder(model_config, sep, eng, device, rank, world, local_batch, dataset)
    elif batch_source is None:
        if dataset is not None:
            raise ValueError("training on a dataset needs the device-side feeder on a CUDA device")
        batch_source = SyntheticBatches(model_config, in_shape, out_shape, seed=1337 + sep.global_step)
    history = done = None
    if summaries:
        # the engine writes each step's loss straight into its slot; an event after each step marks when it finished
        step0 = sep.global_step
        history = torch.empty(model_config["epoch_it"], dtype=sep._loss.dtype, device=sep.params.device)
        done = [torch.cuda.Event(enable_timing=True) for _ in range(model_config["epoch_it"])]
    running, t0 = 0.0, time.time()
    # N > 1: the gradient all-reduce runs bucketed on a communication stream while backward still computes
    # (the spectrogram engine reports no gradient buckets: its gradients are all-reduced after the call)
    overlap = parallel.BucketedAllReduce(eng, sep.grads) if (world > 1 and sep.grads.is_cuda and not spectrogram) else None
    for it in range(model_config["epoch_it"]):                      # :103
        if dev_feeder is not None:
            mix_l, tg_l = dev_feeder.next_batch()                   # this rank's shard, built on the device
        else:
            mix, tg = _to_device(next(batch_source), names, device)
            mix_l = parallel.shard_batch(mix, rank, world).contiguous()
            tg_l = parallel.shard_batch(tg, rank, world, dim=1).contiguous()
        sync = {} if shard is None else {"sync_batch_norm": shard}
        loss = sep.loss_and_gradients(mix_l, tg_l, grad_scale=parallel.grad_scale_for(mix_l.shape[0], global_batch),
                                      loss=None if history is None else history[it:it + 1], **sync)
        if overlap is not None:
            overlap.run()
        else:
            parallel.allreduce_gradients(sep.grads)
        sep.adam_step(lr)
        if done is not None:
            done[it].record(torch.cuda.current_stream(sep.params.device))
        if log_every and (it + 1) % log_every == 0 and rank == 0:
            running = float(loss.item())
            print("step %d  sep_loss(local shard) %.6f  %.1f steps/s" % (sep.global_step, running,
                                                                         (it + 1) / (time.time() - t0)))
    if done:
        lo, hi = parallel.shard_range(global_batch, rank, world)
        _write_sep_loss(os.path.join(model_config["log_dir"], str(experiment_id)), history, done, step0, hi - lo,
                        global_batch, rank)
    path = None
    if rank == 0:
        path = save_checkpoint(os.path.join(model_config["model_base_dir"], str(experiment_id),
                                            "%s-%d" % (experiment_id, sep.global_step)), sep)
    return path, sep


def _write_sep_loss(logdir, history, done, step0, local_batch, global_batch, rank):
    """The epoch's sep_loss summaries from the device-side loss history and the per-step CUDA events `done`: step i's
    wall time is the host time at the epoch's one wait for the device, less the device time from step i to the last."""
    done[-1].synchronize()
    t_last = time.time()
    walls = [t_last - ev.elapsed_time(done[-1]) / 1e3 for ev in done]
    losses = parallel.batch_loss_history(history, local_batch, global_batch).tolist()
    if rank == 0:
        with Summaries.EventFileWriter(logdir) as w:
            for i, (loss, wall) in enumerate(zip(losses, walls)):
                w.add_scalar("sep_loss", loss, step0 + i, wall)


def validation_loss(model_config, sep, batches=4, seed=99, summaries=False, model_folder=None):
    """Running-mean loss over a fixed synthetic validation set (reference Test.test, Test.py:57-71): MSE on audio, or for
    the spectrogram U-Net with raw_audio_loss=False the L1 loss on STFT magnitudes (Test.py:63-67).  With `summaries`,
    rank 0 writes it as Test.test does: a `test_loss` scalar at the separator's global step, in a new events file of
    log_dir/<model_folder>."""
    import torch
    in_shape, out_shape = sep.get_padding(np.array([model_config["batch_size"], model_config["num_frames"], 0]))
    src = SyntheticBatches(model_config, in_shape, out_shape, seed=seed)
    names = model_config["source_names"]
    l1 = model_config["network"] == "unet_spectrogram" and not model_config["raw_audio_loss"]
    tot, n = 0.0, 0
    for _ in range(batches):
        b = next(src)
        mix = torch.from_numpy(b["mix"]).to(sep.params.device)
        if l1:
            eng = sep.engine(num_frames=int(mix.shape[1]))
            est = eng.forward(sep.params, mix, False, return_spectrogram=True)
            tg = torch.stack([torch.from_numpy(b[k]) for k in names]).to(mix.device).contiguous()
            state = torch.zeros(2, dtype=torch.float64, device=mix.device)
            eng.l1_batch_loss(est, tg, state)
            tot += float(state[0].item()); n += 1
            continue
        out = sep.get_output(mix, training=False, reuse=True)
        loss = sum(float(torch.mean((torch.from_numpy(b[k]).to(mix.device) - out[k]) ** 2)) for k in names) / len(names)
        tot += loss; n += 1
    if summaries and parallel.world()[0] == 0:
        if model_folder is None:
            raise ValueError("validation_loss(summaries=True) needs the model_folder to write log_dir/<model_folder>")
        Summaries.write_scalar(os.path.join(model_config["log_dir"], str(model_folder)), "test_loss", tot / n,
                               sep.global_step)
    return tot / n


def optimise(model_config, experiment_id, max_epochs=None, dataset=None, summaries=False, sync_batch_norm=False):
    """Early stopping + fine-tuning (reference optimise(), :123-150).  Without `dataset`: synthetic batches, validated by
    validation_loss, returns (best checkpoint, its validation loss).  With `dataset` (a Datasets.Dataset): trained on its
    train partition, validated by Test.test on "valid" at the current batch size, and, as the reference does, returns
    (best checkpoint, Test.test of that checkpoint on "test").  `summaries` is passed to train and to the validation and
    test losses: sep_loss and test_loss TensorBoard scalars in log_dir/<experiment_id>.  `sync_batch_norm` is passed to
    train."""
    if dataset is not None:
        return _optimise_on_dataset(model_config, experiment_id, max_epochs, dataset, summaries, sync_batch_norm)
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
            model_path, sep = train(model_config, experiment_id, load_model=model_path, sep=sep, summaries=summaries,
                                    sync_batch_norm=sync_batch_norm)
            curr_loss = validation_loss(model_config, sep, summaries=summaries, model_folder=str(experiment_id))
            epoch += 1
            if curr_loss < best_loss:
                worse_epochs = 0
                print("Performance on validation set improved from " + str(best_loss) + " to " + str(curr_loss))
                best_model_path, best_loss = model_path, curr_loss
            else:
                worse_epochs += 1
                print("Performance on validation set worsened to " + str(curr_loss))
    return best_model_path, best_loss


def _optimise_on_dataset(model_config, experiment_id, max_epochs, dataset, summaries, sync_batch_norm):
    import Test
    rank, world = parallel.world()
    epoch, best_loss, model_path, best_model_path, best_step, sep = 0, 10000, None, None, None, None
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
            model_path, sep = train(model_config, experiment_id, load_model=model_path, sep=sep, dataset=dataset,
                                    summaries=summaries, sync_batch_norm=sync_batch_norm)
            # every rank evaluates the whole partition; the loss has the same bits on every rank, so they all take the
            # same early-stopping decision without a collective
            curr_loss = Test.test(model_config, "valid", str(experiment_id), model_path, dataset=dataset, separator=sep,
                                  summaries=summaries)
            epoch += 1
            if curr_loss < best_loss:
                worse_epochs = 0
                print("Performance on validation set improved from " + str(best_loss) + " to " + str(curr_loss))
                best_model_path, best_loss, best_step = model_path, curr_loss, sep.global_step
            else:
                worse_epochs += 1
                print("Performance on validation set worsened to " + str(curr_loss))
    if best_step is None:
        raise RuntimeError("no epoch was trained, so there is no checkpoint to test")
    # only rank 0 writes checkpoints (train()); every rank knows the best one's path from its global step
    best_model_path = os.path.join(model_config["model_base_dir"], str(experiment_id), "%s-%d" % (experiment_id, best_step))
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
    print("TRAINING FINISHED - TESTING WITH BEST MODEL " + best_model_path)
    test_loss = Test.test(model_config, "test", str(experiment_id), best_model_path, dataset=dataset, summaries=summaries)
    return best_model_path, test_loss


def dataset_options(extras):
    """The dataset extras of the command line: dataset=musdb [ccmixter_xml=<path>] [valid_tracks=N].  Returns the keyword
    arguments of run(); no dataset= gives {} (synthetic training, as without the extras)."""
    if "dataset" not in extras:
        unused = [k for k in ("ccmixter_xml", "valid_tracks") if k in extras]
        if unused:
            raise ValueError("%s need dataset=musdb" % ", ".join(unused))
        return {}
    if extras["dataset"] != "musdb":
        raise ValueError("dataset=%r: only dataset=musdb (the MUSDB18 WAV layout) is supported" % (extras["dataset"],))
    opts = {"dataset": "musdb", "valid_tracks": int(extras.get("valid_tracks", 25))}
    if extras.get("ccmixter_xml") is not None:
        opts["ccmixter_xml"] = str(extras["ccmixter_xml"])
    return opts


def run(cfg, max_epochs=None, dataset=None, ccmixter_xml=None, valid_tracks=25, sync_batch_norm=False):
    """The reference's run() (:152-166).  With dataset="musdb" the MUSDB18 WAV dataset at model_config["musdb_path"] (and
    CCMixter's tracks for the voice task, from `ccmixter_xml`) is staged on the device once, trained and validated on,
    and the best checkpoint's estimates and BSS Eval JSONs are written under model_config["estimates_path"].
    `sync_batch_norm` lets the spectrogram U-Net train data parallel (train)."""
    if dataset is not None:
        return _run_on_dataset(cfg, max_epochs, dataset, ccmixter_xml, valid_tracks, sync_batch_norm)
    model_config = cfg["model_config"]
    print("SCRIPT START")
    for d in [model_config["model_base_dir"], model_config["log_dir"]]:
        os.makedirs(d, exist_ok=True)
    if "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    sup_model_path, sup_loss = optimise(model_config, cfg["experiment_id"], max_epochs=max_epochs, summaries=True,
                                        sync_batch_norm=sync_batch_norm)
    print("Supervised training finished! Saved model at " + str(sup_model_path) + ". Performance: " + str(sup_loss))
    return sup_model_path, sup_loss


def _run_on_dataset(cfg, max_epochs, dataset, ccmixter_xml, valid_tracks, sync_batch_norm):
    import torch
    import Datasets
    import Evaluate
    if dataset != "musdb":
        raise ValueError("dataset=%r: only dataset=musdb is supported" % (dataset,))
    model_config = cfg["model_config"]
    print("SCRIPT START")
    for d in [model_config["model_base_dir"], model_config["log_dir"]]:
        os.makedirs(d, exist_ok=True)
    if "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    probe = separator_class(model_config)(model_config)
    in_shape, out_shape = probe.get_padding(np.array([model_config["batch_size"], model_config["num_frames"], 0]))
    ds = Datasets.load_musdb(model_config, int(in_shape[1]), int(out_shape[1]), model_config["musdb_path"], ccmixter_xml,
                             valid_tracks, device)
    sup_model_path, sup_loss = optimise(model_config, cfg["experiment_id"], max_epochs=max_epochs, dataset=ds,
                                        summaries=True, sync_batch_norm=sync_batch_norm)
    print("Supervised training finished! Saved model at " + str(sup_model_path) + ". Performance: " + str(sup_loss))
    Evaluate.produce_musdb_source_estimates(model_config, sup_model_path, model_config["musdb_path"],
                                            model_config["estimates_path"])
    return sup_model_path, sup_loss


def main(argv):
    """The command line: sacred-style `with cfg.<preset> ...` (Config.parse_command_line) and the top-level extras
    max_epochs=N, sync_batch_norm=1 and the dataset ones (dataset_options)."""
    cfg, extras = Config.parse_command_line(argv)
    return run(cfg, max_epochs=extras.get("max_epochs"), sync_batch_norm=bool(extras.get("sync_batch_norm", False)),
               **dataset_options(extras))


if __name__ == "__main__":
    main(sys.argv[1:])
