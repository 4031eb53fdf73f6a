"""Drop-in for the reference's spectrogram U-Net separator (the Jansson et al. baselines U7 / U7a, presets unet_spectrogram
and unet_spectrogram_l1), backed by the CUDA kernels of libwun.so (include/wun.h wun_spec_*).

Same class name, constructor argument and method names as the reference's Models/UnetSpectrogramSeparator.py:

    sep = UnetSpectrogramSeparator(model_config)
    in_shape, out_shape = sep.get_padding(np.array([batch, num_frames, 0]))     # unchanged: [B, T, 1] both ways
    sources = sep.get_output(mix, training=False, return_spectrogram=False)

As with UnetAudioSeparator here, `mix` is a float32 CUDA tensor [B, T, 1] and the result an ordered dict source name ->
float32 CUDA tensor: audio [B, T, 1], or with return_spectrogram the magnitudes [B, n, 513].  The variables (kernels,
biases, batch-norm betas and moving statistics) live in one flat float32 CUDA buffer in TF creation order under
"separator".  Only the inference graph exists: training=True raises NotImplementedError.
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
        self._engines = {}                      # T -> wun.SpecEngine
        self.params = None
        self.global_step = 0
        self.seed = 1337

    def get_padding(self, shape):
        """The shape unchanged: input and output are [batch, frames, 1]."""
        return [shape[0], shape[1], 1], [shape[0], shape[1], 1]

    def get_output(self, input, training, return_spectrogram=False, reuse=True):
        """Audio estimates [B, T, 1] per source, or with return_spectrogram their magnitudes [B, n, 513]."""
        if training:
            raise NotImplementedError("training the spectrogram U-Net is not supported; use training=False")
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
