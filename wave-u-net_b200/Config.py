"""Experiment configuration for the Wave-U-Net engine (sacred-free).

Mirrors the *data* the reference's sacred ingredient produces
(/root/reference/Config.py:6-161): one ``model_config`` dict plus an
``experiment_id``.  sacred is not available (and not wanted) here, so this module
re-creates the three sacred behaviours the callers rely on:

* named presets partially override the base dict          (Config.py:52-161)
* ``key=value`` command-line updates override both         (README.md:84-92)
* derived keys (``source_names``, ``num_sources``, ``num_channels``) are computed
  AFTER all overrides are applied                           (Config.py:43-50)

Command-line syntax accepted by :func:`parse_command_line` is the sacred one::

    python Training.py with cfg.baseline_stereo cfg.model_config.batch_size=8
"""
import ast
import copy
import random

# --- base dictionary (values: Config.py:9-39) --------------------------------------------
_BASE = dict(
    musdb_path="/mnt/windaten/Datasets/MUSDB18/",
    estimates_path="/mnt/windaten/Source_Estimates",
    data_path="data",
    model_base_dir="checkpoints",
    log_dir="logs",
    batch_size=16,
    init_sup_sep_lr=1e-4,
    epoch_it=2000,
    cache_size=4000,
    num_workers=4,
    num_snippets_per_track=100,
    num_layers=12,
    filter_size=15,
    merge_filter_size=5,
    input_filter_size=15,
    output_filter_size=1,
    num_initial_filters=24,
    num_frames=16384,
    expected_sr=22050,
    mono_downmix=True,
    output_type="direct",
    output_activation="tanh",
    context=False,
    network="unet",
    upsampling="linear",
    task="voice",
    augmentation=True,
    raw_audio_loss=True,
    worse_epochs=20,
)

_SPEC_FRAMES = 768 * 127 + 1024

# --- named presets: only the keys each preset changes (Config.py:52-161) ------------------
NAMED_CONFIGS = {
    "baseline": {},
    "baseline_diff": dict(output_type="difference"),
    "baseline_context": dict(output_type="difference", context=True),
    "baseline_stereo": dict(output_type="difference", context=True, mono_downmix=False),
    "full": dict(output_type="difference", context=True, upsampling="learned", mono_downmix=False),
    "full_44KHz": dict(output_type="difference", context=True, upsampling="learned",
                       mono_downmix=False, expected_sr=44100),
    "baseline_context_smallfilter_deep": dict(output_type="difference", context=True, num_layers=14,
                                              duration=7, filter_size=5, merge_filter_size=1),
    "full_multi_instrument": dict(output_type="difference", context=True, upsampling="linear",
                                  mono_downmix=False, task="multi_instrument"),
    "baseline_comparison": dict(batch_size=4, output_type="difference", context=True,
                                num_frames=_SPEC_FRAMES, duration=13, expected_sr=8192,
                                num_initial_filters=34),
    "unet_spectrogram": dict(batch_size=4, network="unet_spectrogram", num_layers=6, expected_sr=8192,
                             num_frames=_SPEC_FRAMES, duration=13, num_initial_filters=16),
    "unet_spectrogram_l1": dict(batch_size=4, network="unet_spectrogram", num_layers=6,
                                expected_sr=8192, num_frames=_SPEC_FRAMES, duration=13,
                                num_initial_filters=16, raw_audio_loss=False),
}

_TASK_SOURCES = {
    "multi_instrument": ["bass", "drums", "other", "vocals"],
    "voice": ["accompaniment", "vocals"],
}


def _derive(mc):
    """Keys the reference computes after overrides (Config.py:43-50)."""
    task = mc["task"]
    if task not in _TASK_SOURCES:
        raise NotImplementedError("unknown task %r" % (task,))
    mc["source_names"] = list(_TASK_SOURCES[task])
    mc["num_sources"] = len(mc["source_names"])
    mc["num_channels"] = 1 if mc["mono_downmix"] else 2
    return mc


def build_config(named=(), updates=None, experiment_id=None):
    """Return ``{"model_config": {...}, "experiment_id": int}``.

    ``named``   iterable of preset names (``"baseline_stereo"`` or ``"cfg.baseline_stereo"``),
                applied in order.
    ``updates`` dict of ``model_config`` key overrides applied last (highest priority).
    """
    mc = copy.deepcopy(_BASE)
    if isinstance(named, str):
        named = [named]
    for name in named:
        short = name[4:] if name.startswith("cfg.") else name
        if short not in NAMED_CONFIGS:
            raise KeyError("unknown named config %r" % (name,))
        mc.update(copy.deepcopy(NAMED_CONFIGS[short]))
    if updates:
        mc.update(copy.deepcopy(updates))
    _derive(mc)
    if experiment_id is None:
        experiment_id = random.randint(0, 999999)   # Config.py:40
    return {"model_config": mc, "experiment_id": int(experiment_id)}


def _literal(text):
    try:
        return ast.literal_eval(text)
    except (ValueError, SyntaxError):
        return text


def parse_command_line(argv):
    """Parse sacred-style ``[with] cfg.<preset> [cfg.]model_config.<key>=<value> <name>=<value>``.

    Returns ``(cfg, extras)`` where ``extras`` holds top-level non-``cfg`` assignments such as
    ``model_path=...`` / ``input_path=...`` used by Predict (Predict.py:8-12).
    """
    named, updates, extras = [], {}, {}
    experiment_id = None
    for tok in argv:
        if tok == "with":
            continue
        if "=" in tok:
            key, val = tok.split("=", 1)
            val = _literal(val)
            if key.startswith("cfg."):
                key = key[4:]
            if key.startswith("model_config."):
                updates[key[len("model_config."):]] = val
            elif key == "experiment_id":
                experiment_id = int(val)
            else:
                extras[key] = val
        else:
            named.append(tok)
    return build_config(named, updates, experiment_id), extras
