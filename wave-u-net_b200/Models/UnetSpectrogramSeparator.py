"""Drop-in for the reference's spectrogram U-Net separator (the Jansson et al. baselines U7 / U7a, presets unet_spectrogram
and unet_spectrogram_l1), backed by the CUDA kernels of libwun.so (include/wun.h wun_spec_*).

Same class name, constructor argument and method names as the reference's Models/UnetSpectrogramSeparator.py:

    sep = UnetSpectrogramSeparator(model_config)
    in_shape, out_shape = sep.get_padding(np.array([batch, num_frames, 0]))     # unchanged: [B, T, 1] both ways
    sources = sep.get_output(mix, training=False, return_spectrogram=False)

As with UnetAudioSeparator here, `mix` is a float32 CUDA tensor [B, T, 1] and the result an ordered dict source name ->
float32 CUDA tensor: audio [B, T, 1], or with return_spectrogram the magnitudes [B, n, 513].  The variables (kernels,
biases, batch-norm betas and moving statistics) live in one flat float32 CUDA buffer in TF creation order under
"separator".

Training is the training half of the graph Training.py builds (:47-77) and goes through loss_and_gradients() / adam_step(),
as with UnetAudioSeparator: training-mode batch norm (batch statistics, moving averages updated on every step), dropout on
the first three concatenations of the up path, the U7 (audio MSE) or U7a (L1 on magnitudes, raw_audio_loss=False) loss,
every trainable variable's gradient and tf.train.AdamOptimizer on kernels, biases and betas.  A standalone
get_output(training=True) graph does not exist and raises NotImplementedError.

Data-parallel training is opt-in, like torch's SyncBatchNorm: loss_and_gradients(..., sync_batch_norm=shard) with a
wun.parallel.BatchStatsGather runs this rank's shard with the whole batch's batch-norm statistics, dropout masks and 1/B
loss scaling, so that after the gradient all-reduce every rank holds the single-device step's gradients.
"""
from collections import OrderedDict
import math

import numpy as np

import wun


class UnetSpectrogramSeparator:
    def __init__(self, model_config):
        self.num_layers = model_config["num_layers"]
        self.num_initial_filters = model_config["num_initial_filters"]
        self.mono = model_config["mono_downmix"]
        self.source_names = list(model_config["source_names"])
        assert len(self.source_names) == 2      # acc / voice separation only, as in the reference
        assert self.mono                        # mono only
        self.frame_len = 1024
        self.hop = 768
        self._cfg = wun.spec_config_from_model_config(model_config)
        self.raw_audio_loss = bool(model_config.get("raw_audio_loss", True))
        self._engines = {}                      # T -> wun.SpecEngine
        self.params = None
        self.grads = None
        self.adam_m = None
        self.adam_v = None
        self._adam_state = None                 # device float32[3] {beta1_power, beta2_power, step}: TF's beta*_power
        self._betas = (0.9, 0.999)
        self._step0 = 0
        self._loss = None
        self._dropout_step = None               # device int64[1]: the dropout masks' step counter
        self.seed = 1337
        self.last_feeder = None
        self.last_feeder_tracks = None

    # global_step lives on the device next to Adam's beta-power accumulators, so that a CUDA-graph replay of a whole
    # training step advances it and uses the right bias correction every replay.
    @property
    def global_step(self):
        if self._adam_state is None:
            return self._step0
        return int(round(float(self._adam_state[2].item())))

    @global_step.setter
    def global_step(self, n):
        self._step0 = int(n)
        if self._adam_state is not None:
            self._write_adam_state()

    def _write_adam_state(self):
        import torch
        b1, b2 = self._betas
        n = self._step0
        vals = torch.tensor([b1 ** (n + 1), b2 ** (n + 1), float(n)], dtype=torch.float32)
        self._adam_state.copy_(vals.to(self._adam_state.device))

    def get_padding(self, shape):
        """The shape unchanged: input and output are [batch, frames, 1]."""
        return [shape[0], shape[1], 1], [shape[0], shape[1], 1]

    def get_output(self, input, training, return_spectrogram=False, reuse=True):
        """Audio estimates [B, T, 1] per source, or with return_spectrogram their magnitudes [B, n, 513]."""
        if training:
            raise NotImplementedError("the spectrogram U-Net trains through loss_and_gradients() / adam_step(); "
                                      "get_output runs with training=False")
        eng = self._engine_for(int(input.shape[1]))
        self._ensure_params(eng, input.device, create=not reuse)
        out = eng.forward(self.params, input.contiguous(), False, return_spectrogram=return_spectrogram)
        return OrderedDict((name, out[k]) for k, name in enumerate(self.source_names))

    def _engine_for(self, t):
        eng = self._engines.get(t)
        if eng is None:
            eng = wun.SpecEngine(self._cfg, num_frames=t)
            self._engines[t] = eng
        return eng

    def engine(self, num_frames=None, input_frames=None):
        return self._engine_for(int(input_frames if input_frames is not None else num_frames))

    def _ensure_params(self, eng, device, create):
        """TF's initial values when creating: glorot-uniform kernels, zero biases and betas, moving mean 0, variance 1."""
        import torch
        if self.params is not None:
            return
        if not create:
            raise ValueError("Variable separator/conv2d/kernel does not exist (get_output called with reuse=True "
                             "before the variables were created or loaded)")
        flat = np.zeros(eng.param_numel, np.float32)
        rng = np.random.default_rng(self.seed)
        for name, shape, off, numel in eng.param_table:
            if name.endswith("/kernel"):
                lim = math.sqrt(6.0 / (shape[0] * shape[1] * (shape[2] + shape[3])))
                flat[off:off + numel] = rng.uniform(-lim, lim, size=numel).astype(np.float32)
            elif name.endswith("/moving_variance"):
                flat[off:off + numel] = 1.0
        self.params = torch.from_numpy(flat).to(device)

    def param_table(self, num_frames=None, input_frames=None):
        eng = next(iter(self._engines.values())) if self._engines and num_frames is None and input_frames is None \
            else self.engine(num_frames, input_frames)
        return eng.param_table

    def variables(self):
        """Ordered dict TF-name -> view into the flat parameter buffer (what Saver would checkpoint)."""
        eng = next(iter(self._engines.values()))
        return OrderedDict((n, self.params[o:o + c].view(*s)) for n, s, o, c in eng.param_table)

    def load_variables(self, values, device=None, num_frames=None, input_frames=None):
        """values: mapping TF-name -> array; every variable of the table is required and shape-checked.  device: where the
        flat buffer goes - default: where the current variables live, else the current CUDA device (the host when there is
        none, so that checkpoints can be read and checked anywhere; forward needs the buffer on the GPU)."""
        import torch
        if device is None:
            if self.params is not None:
                device = self.params.device
            else:
                device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        eng = self.engine(num_frames, input_frames) if (num_frames or input_frames) else next(iter(self._engines.values()))
        flat = np.zeros(eng.param_numel, np.float32)
        for name, shape, off, numel in eng.param_table:
            a = np.asarray(values[name], dtype=np.float32)
            assert tuple(a.shape) == tuple(shape), (name, a.shape, shape)
            flat[off:off + numel] = a.reshape(-1)
        self.params = torch.from_numpy(flat).to(device)
        self.grads = self.adam_m = self.adam_v = None
        if self._adam_state is not None:
            self._step0 = self.global_step
            self._adam_state = None
            self._dropout_step = None

    def trainable_variable_names(self):
        """The variables AdamOptimizer trains and the checkpoint has slots for: kernels, biases, betas (not the moving
        statistics, which only the batch-norm update moves)."""
        eng = next(iter(self._engines.values()))
        return [n for n, _, _ in eng.trainable_ranges]

    def gradients(self):
        eng = next(iter(self._engines.values()))
        return OrderedDict((n, self.grads[o:o + c].view(*s)) for n, s, o, c in eng.param_table)

    # ------------------------------------------------------------------------------------------
    # the training half of the graph (Training.py:47-77)
    # ------------------------------------------------------------------------------------------
    def _ensure_training_state(self):
        import torch
        if self.grads is None:
            dev = self.params.device
            self.grads = torch.zeros_like(self.params)
            self.adam_m = torch.zeros_like(self.params)
            self.adam_v = torch.zeros_like(self.params)
            self._loss = torch.zeros(1, dtype=torch.float64, device=dev)
            self._adam_state = torch.zeros(3, dtype=torch.float32, device=dev)
            self._write_adam_state()
            # one dropout step per optimiser step: a resumed run continues the masks where the checkpoint left them
            self._dropout_step = torch.full((1,), self._step0, dtype=torch.int64, device=dev)

    def loss_and_gradients(self, mix, targets, reuse=True, grad_scale=1.0, loss=None, sync_batch_norm=None):
        """separator_loss (Training.py:50-63) of get_output(mix, training=True, not raw_audio_loss) and d loss / d variables;
        the batch-norm moving statistics in self.params take their update.  targets: [K, B, T, 1] tensor or dict.
        Returns the device float64 loss, written into `loss` (a float64 CUDA tensor, e.g. one slot of a per-step history)
        when given; the gradients land in self.grads (flat, 0 for the moving statistics).
        sync_batch_norm (a wun.parallel.BatchStatsGather): mix and targets are this rank's shard of the batch; batch norm
        uses the whole batch's statistics and the gradients are this shard's part of the whole batch's (grad_scale, if
        given, must be the shard's local_batch / global_batch), to be summed over the ranks.  The loss is the shard's mean."""
        import torch
        if sync_batch_norm is None and grad_scale != 1.0:
            raise ValueError("the spectrogram U-Net trains on one GPU unless sync_batch_norm is given: batch statistics of "
                             "a shard would change the model")
        if sync_batch_norm is not None:
            part = float(sync_batch_norm.local_batch) / float(sync_batch_norm.global_batch)
            if grad_scale != 1.0 and abs(grad_scale - part) > 1e-12:
                raise ValueError("grad_scale %r: a synchronised shard's gradients are scaled by local_batch / global_batch "
                                 "= %r" % (grad_scale, part))
            if int(mix.shape[0]) != sync_batch_norm.local_batch:
                raise ValueError("the shard holds %d examples, mix %d" % (sync_batch_norm.local_batch, int(mix.shape[0])))
        if isinstance(targets, dict):
            targets = torch.stack([targets[n] for n in self.source_names])
        eng = self._engine_for(int(mix.shape[1]))
        self._ensure_params(eng, mix.device, create=not reuse)
        self._ensure_training_state()
        loss = self._loss if loss is None else loss
        eng.forward_backward(self.params, mix.contiguous(), targets.contiguous(), self.grads, loss,
                             self.raw_audio_loss, self.seed, self._dropout_step, shard=sync_batch_norm)
        return loss

    def adam_step(self, learning_rate, beta1=0.9, beta2=0.999, epsilon=1e-8):
        """tf.train.AdamOptimizer(learning_rate).minimize step on the trainable separator variables (:77)."""
        eng = next(iter(self._engines.values()))
        if (beta1, beta2) != self._betas:
            self._step0 = self.global_step
            self._betas = (beta1, beta2)
            self._write_adam_state()
        eng.adam_step_device(self.params, self.grads, self.adam_m, self.adam_v, self._adam_state, learning_rate, beta1,
                             beta2, epsilon)
