"""Drop-in for the reference's Wave-U-Net separator class, backed by the H100 CUDA engine (libwun.so).

Same class name, constructor argument and method names/arguments as
/root/reference/Models/UnetAudioSeparator.py:9-144:

    sep = UnetAudioSeparator(model_config)
    in_shape, out_shape = sep.get_padding(np.array([batch, num_frames, 0]))
    sources = sep.get_output(mix, training, return_spectrogram=False, reuse=False)

Differences that follow from not being a TF graph builder:
  * `mix` is a float32 CUDA torch tensor [B, T_in, C] (channels-last like the reference, :88) and the
    result is an ordered dict  source name -> float32 CUDA tensor [B, T_out, C]  (same keys/order).
  * variables live in ONE flat float32 CUDA buffer owned by this object (`self.params`), laid out in
    TF creation order under scope "separator" (:92); `reuse=False` creates them (glorot-uniform kernels,
    zero biases - the tf.layers.conv1d defaults), `reuse=True` shares the existing ones.
  * the training half of the graph that TF derived for Training.py:50-77 (loss, gradients, Adam) is
    exposed as loss_and_gradients() / adam_step(); Training.py calls those.
There is no PyTorch / CPU implementation behind this class: every tensor op is a kernel in libwun.so.
"""
from collections import OrderedDict
import math

import numpy as np

import wun


class UnetAudioSeparator:
    def __init__(self, model_config):
        # the keys the reference constructor reads (:20-32)
        self.num_layers = model_config["num_layers"]
        self.num_initial_filters = model_config["num_initial_filters"]
        self.filter_size = model_config["filter_size"]
        self.merge_filter_size = model_config["merge_filter_size"]
        self.input_filter_size = model_config["input_filter_size"]
        self.output_filter_size = model_config["output_filter_size"]
        self.upsampling = model_config["upsampling"]
        self.output_type = model_config["output_type"]
        self.context = model_config["context"]
        self.padding = "valid" if model_config["context"] else "same"
        self.source_names = list(model_config["source_names"])
        self.num_channels = 1 if model_config["mono_downmix"] else 2
        self.output_activation = model_config["output_activation"]

        self._cfg = wun.config_from_model_config(model_config)
        self._engines = {}          # T_in -> wun.Engine
        self.params = None          # flat float32 CUDA tensor
        self.grads = None
        self.adam_m = None
        self.adam_v = None
        self._adam_state = None     # device float32[3] {beta1_power, beta2_power, step}: TF's beta*_power variables
        self._betas = (0.9, 0.999)
        self._step0 = 0
        self._loss = None
        self.seed = 1337            # Training.py:22
        self.last_feeder = None     # wun.feeder.DeviceFeeder Training.train built for this separator (device-side input pipeline)
        self.last_feeder_tracks = None

    # global_step lives on the device next to Adam's beta-power accumulators, so that a CUDA-graph replay of a whole
    # training step (bench.py, wun/prefetch.py) advances it and uses the right bias correction every replay.
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

    # ------------------------------------------------------------------------------------------
    # reference API
    # ------------------------------------------------------------------------------------------
    def get_padding(self, shape):
        """Input / output shapes for a desired output shape [batch, frames, _] (reference :34-83)."""
        if self.context:
            t_in, t_out = wun.get_padding(self._cfg, int(shape[1]))
            input_shape = np.concatenate([[shape[0]], [t_in], [self.num_channels]]).astype(np.int64)
            output_shape = np.concatenate([[shape[0]], [t_out], [self.num_channels]]).astype(np.int64)
            return input_shape, output_shape
        return [shape[0], shape[1], self.num_channels], [shape[0], shape[1], self.num_channels]

    def get_output(self, input, training, return_spectrogram=False, reuse=True):
        """Source estimates for a batch of mixtures (reference :85-144)."""
        if self.output_activation not in ("tanh", "linear"):
            raise NotImplementedError        # :136
        if self.output_type not in ("direct", "difference"):
            raise NotImplementedError        # :144
        eng = self._engine_for(int(input.shape[1]))
        self._ensure_params(eng, input.device, create=not reuse)
        out = eng.forward(self.params, input.contiguous(), bool(training))
        return OrderedDict((name, out[k]) for k, name in enumerate(self.source_names))

    # ------------------------------------------------------------------------------------------
    # variables ("separator/..." scope)
    # ------------------------------------------------------------------------------------------
    def _engine_for(self, t_in):
        eng = self._engines.get(t_in)
        if eng is None:
            eng = wun.Engine(self._cfg, input_frames=t_in)
            self._engines[t_in] = eng
        return eng

    def engine(self, num_frames=None, input_frames=None):
        if input_frames is None:
            input_frames = wun.get_padding(self._cfg, num_frames)[0]
        return self._engine_for(int(input_frames))

    def _ensure_params(self, eng, device, create):
        import torch
        if self.params is not None:
            return
        if not create:
            raise ValueError("Variable separator/conv1d/kernel does not exist (get_output called with reuse=True "
                             "before the variables were created or loaded)")
        flat = np.zeros(eng.param_numel, np.float32)
        rng = np.random.default_rng(self.seed)
        for name, shape, off, numel in eng.param_table:
            if name.endswith("/kernel"):
                k, cin, cout = shape
                lim = math.sqrt(6.0 / (k * cin + k * cout))
                flat[off:off + numel] = rng.uniform(-lim, lim, size=numel).astype(np.float32)
            elif not name.endswith("/bias"):        # interp_<level>
                lim = math.sqrt(6.0 / (2 * shape[0]))
                flat[off:off + numel] = rng.uniform(-lim, lim, size=numel).astype(np.float32)
        self.params = torch.from_numpy(flat).to(device)

    def param_table(self, num_frames=None, input_frames=None):
        eng = next(iter(self._engines.values())) if self._engines and num_frames is None and input_frames is None \
            else self.engine(num_frames, input_frames)
        return eng.param_table

    def variables(self):
        """Ordered dict TF-name -> view into the flat parameter buffer (what Saver would checkpoint)."""
        eng = next(iter(self._engines.values()))
        return OrderedDict((n, self.params[o:o + c].view(*s)) for n, s, o, c in eng.param_table)

    def gradients(self):
        eng = next(iter(self._engines.values()))
        return OrderedDict((n, self.grads[o:o + c].view(*s)) for n, s, o, c in eng.param_table)

    def load_variables(self, values, device=None, num_frames=None, input_frames=None):
        """values: mapping TF-name -> array (e.g. read from a checkpoint); all variables required.  device: where the
        flat buffer goes - default: where the current variables live, else the current CUDA device."""
        import torch
        if device is None:
            device = self.params.device if self.params is not None else torch.device("cuda", torch.cuda.current_device())
        eng = self.engine(num_frames, input_frames) if (num_frames or input_frames) else \
            next(iter(self._engines.values()))
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

    # ------------------------------------------------------------------------------------------
    # the training half of the graph (Training.py:50-77)
    # ------------------------------------------------------------------------------------------
    def _ensure_training_state(self):
        import torch
        if self.grads is None:
            self.grads = torch.zeros_like(self.params)
            self.adam_m = torch.zeros_like(self.params)
            self.adam_v = torch.zeros_like(self.params)
            self._loss = torch.zeros(1, dtype=torch.float32, device=self.params.device)
            self._adam_state = torch.zeros(3, dtype=torch.float32, device=self.params.device)
            self._write_adam_state()

    def stack_targets(self, batch):
        """dict name -> [B,T_out,C]  ->  [K,B,T_out,C] in source_names order."""
        import torch
        return torch.stack([batch[name] for name in self.source_names]).contiguous()

    def loss_and_gradients(self, mix, targets, reuse=True, grad_scale=1.0, outputs=None, loss=None):
        """separator_loss (Training.py:50-63) and d loss / d variables (the tf.gradients part of :77).
        targets: [K,B,T_out,C] tensor or dict.  Returns the device scalar loss, written into `loss` (a float32 CUDA
        tensor, e.g. one slot of a per-step history) when given; gradients land in self.grads (flat)."""
        if isinstance(targets, dict):
            targets = self.stack_targets(targets)
        eng = self._engine_for(int(mix.shape[1]))
        self._ensure_params(eng, mix.device, create=not reuse)
        self._ensure_training_state()
        loss = self._loss if loss is None else loss
        eng.forward_backward(self.params, mix.contiguous(), targets.contiguous(), self.grads, loss,
                             grad_scale=grad_scale, out=outputs)
        return loss

    def adam_step(self, learning_rate, beta1=0.9, beta2=0.999, epsilon=1e-8):
        """tf.train.AdamOptimizer(learning_rate).minimize step on the separator variables (:77)."""
        eng = next(iter(self._engines.values()))
        if (beta1, beta2) != self._betas:
            self._step0 = self.global_step
            self._betas = (beta1, beta2)
            self._write_adam_state()
        eng.adam_step_device(self.params, self.grads, self.adam_m, self.adam_v, self._adam_state, learning_rate, beta1,
                             beta2, epsilon)
