"""The reference's Test.test (Test.py:11-93): the mean MSE of a model over every snippet of a partition.

    loss = Test.test(model_config, "valid", model_folder, load_model, dataset=ds, separator=sep)

Snippets start every T_out frames (take_all_snippets, Datasets.py:21-25), the mix is the recorded mixture, the targets are
centre-cropped, batches of model_config["batch_size"] cross track boundaries and the last incomplete batch is dropped.  Per
batch, curr = sum_k mean((target_k - estimate_k)^2) / K with the forward in test mode (output clip on), and the result is
the running mean total += (1 / n) * (curr - total) (Test.py:57-79).  The spectrogram U-Net (network "unet_spectrogram") runs
the same way; with raw_audio_loss=False (preset unet_spectrogram_l1, U7a) curr is sum_k mean|STFTmag(target_k) -
estimate_k| / K over the magnitudes [B, n, 513] instead.

On the device: one CUDA graph of wun_snippet_batch -> wun_forward -> wun_eval_batch_loss, replayed once per batch; the
batch counter and the fp64 running mean live on the device, so the partition costs one host synchronisation, at the end,
and gives the same bits on every run.  With summaries=True the result is also written as the reference's `test_loss`
TensorBoard scalar (Test.py:41,81-82), in a new events file of log_dir/<model_folder> (Summaries.py).
"""
import os

import numpy as np


def test(model_config, partition, model_folder, load_model, dataset=None, separator=None, summaries=False):
    """Running-mean MSE (or, for U7a, L1 of magnitudes) over the full batches of `partition` ("valid" or "test") of `dataset` (a Datasets.Dataset; staged
    from model_config["musdb_path"] when None), with `separator` or else the variables of checkpoint `load_model`.
    Raises ValueError when the partition has fewer snippets than one batch.  With `summaries`, rank 0 writes the result,
    rounded to float32, as a `test_loss` scalar at the separator's global step (both partitions use that tag, as in the
    reference); every rank computes the same bits, so no collective is needed."""
    import torch
    import Datasets
    import Evaluate
    import Summaries
    import wun
    from wun import parallel
    if model_config["network"] not in ("unet", "unet_spectrogram"):
        raise NotImplementedError
    # the spectrogram U-Net's U7a preset scores magnitudes: mean |STFTmag(target) - estimate| (Test.py:63-67)
    magnitude_loss = model_config["network"] == "unet_spectrogram" and not model_config["raw_audio_loss"]
    if separator is None:
        separator = Evaluate.load_separator(model_config, load_model)
    B = int(model_config["batch_size"])
    in_shape, out_shape = separator.get_padding(np.array([B, model_config["num_frames"], 0]))
    t_in, t_out = int(in_shape[1]), int(out_shape[1])
    if dataset is None:
        dataset = Datasets.load_musdb(model_config, t_in, t_out)
    assert (dataset.t_in, dataset.t_out) == (t_in, t_out), "the dataset was staged for other input / output lengths"
    pool = dataset.partitions[partition].pool
    positions = dataset.positions(partition, B)
    n_batches = positions.numel() // B
    dev = pool.device
    eng = separator.engine(input_frames=t_in)
    separator._ensure_params(eng, dev, create=False)
    K, C = len(model_config["source_names"]), int(pool.shape[2])
    print("Testing...")

    counter = torch.zeros(1, dtype=torch.int64, device=dev)
    mix = torch.empty((B, t_in, C), dtype=torch.float32, device=dev)
    targets = torch.empty((K, B, t_out, C), dtype=torch.float32, device=dev)
    state = torch.zeros(2, dtype=torch.float64, device=dev)
    if magnitude_loss:
        outputs = torch.empty(eng.output_shape(B, return_spectrogram=True), dtype=torch.float32, device=dev)
    else:
        outputs = torch.empty_like(targets)
        slots = torch.empty(K * wun.EVAL_LOSS_CTAS, dtype=torch.float64, device=dev)

    def batch():
        wun.snippet_batch(pool, positions, B, counter, mix, targets)
        if magnitude_loss:
            eng.forward(separator.params, mix, False, out=outputs, return_spectrogram=True)
            eng.l1_batch_loss(outputs, targets, state)
        else:
            eng.forward(separator.params, mix, False, out=outputs)
            wun.eval_batch_loss(outputs, targets, state, slots)

    with torch.cuda.device(dev):
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)                # a graph is captured on a stream other than the default one
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            batch()                                  # batch 0 eagerly: the engine sets up its workspace outside the capture
            if n_batches > 1:
                graph = torch.cuda.CUDAGraph()
                graph.capture_begin()
                batch()
                graph.capture_end()
                for _ in range(n_batches - 1):
                    graph.replay()
        cur.wait_stream(side)
        total = float(state[0].item())
    if summaries and parallel.world()[0] == 0:
        Summaries.write_scalar(os.path.join(model_config["log_dir"], str(model_folder)), "test_loss", total, separator.global_step)
    print("Finished testing - Mean %s: %s" % ("L1" if magnitude_loss else "MSE", total))
    return total
