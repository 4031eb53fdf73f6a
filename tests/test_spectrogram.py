"""The spectrogram U-Net baselines (U7 / U7a) without a GPU: the float64 oracle against fixtures produced by the reference's
own UnetSpectrogramSeparator (tests/golden/make_spectrogram_golden.py), the engine's parameter table, shape checks and FLOP count, and
restoring a TF checkpoint into the facade."""
import glob
import json
import os

import numpy as np
import pytest

import Config
import Evaluate
import TFCheckpoint
import wun
from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator
from oracle import spectrogram_oracle as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spectrogram")
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz")))
PRESET_FRAMES = 768 * 127 + 1024


def load_case(name):
    """(npz, model_config, params float32, mix float32 [B, T, 1], {(kind, source): expected output})."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = json.loads(str(z["cfg_json"]))
    params = {k[len("param/"):]: z[k].astype(np.float32) for k in z.files if k.startswith("param/")}
    mix = z["mix_pcm16"].astype(np.float32) / np.float32(32768)
    outputs = {tuple(k.split("/")): z[k] for k in z.files if k.split("/")[0] in ("audio", "mag")}
    return z, cfg, params, mix, outputs


def mc(named, **kw):
    return Config.build_config([named], kw, experiment_id=0)["model_config"]


def test_fixtures_present():
    assert CASES == ["spec_l2", "spec_l3", "spec_l6"]
    assert OUTPUT_CASES == [("spec_l2", "audio"), ("spec_l2", "mag"), ("spec_l3", "audio"), ("spec_l3", "mag"),
                            ("spec_l6", "mag")]


# (fixture, output kind) pairs the fixtures record: both kinds for the small cases, magnitudes for the six-layer one
OUTPUT_CASES = [(n, kind) for n in CASES for kind in ("audio", "mag")
                if any(k.startswith(kind + "/") for k in np.load(os.path.join(GOLDEN, n + ".npz")).files)]


@pytest.mark.parametrize("name,kind", OUTPUT_CASES, ids=["%s-%s" % c for c in OUTPUT_CASES])
def test_oracle_matches_reference_fixture(name, kind):
    """The fixtures hold float64 results rounded to float32: agreement to a few float32 ulps of the largest value."""
    z, cfg, params, mix, outputs = load_case(name)
    wanted = {s: w for (k, s), w in outputs.items() if k == kind}
    out = S.forward(params, mix, cfg["num_layers"], cfg["source_names"], return_spectrogram=kind == "mag")
    for s, want in wanted.items():
        assert out[s].shape == want.shape
        scale = np.abs(want).max()
        assert np.abs(out[s] - want).max() <= 4e-7 * scale, (s, np.abs(out[s] - want).max(), scale)


@pytest.mark.parametrize("name", CASES)
def test_param_table_matches_reference_names_and_shapes(name):
    z, cfg, params, _, _ = load_case(name)
    eng = wun.SpecEngine(wun.spec_config_from_model_config(cfg), num_frames=int(z["T"]))
    assert [n for n, _, _, _ in eng.param_table] == list(z["param_names"])
    assert [tuple(s) for _, s, _, _ in eng.param_table] == [params[n].shape for n in z["param_names"]]
    offsets = [o for _, _, o, _ in eng.param_table]
    sizes = [c for _, _, _, c in eng.param_table]
    assert offsets == list(np.cumsum([0] + sizes[:-1])) and eng.param_numel == sum(sizes)
    assert [(n, tuple(s)) for n, s, _, _ in eng.param_table] == S.param_specs(cfg["num_layers"], cfg["num_initial_filters"])


@pytest.mark.parametrize("preset", ["unet_spectrogram", "unet_spectrogram_l1"])
def test_preset_shapes_params_and_flops(preset):
    cfg = mc(preset)
    sep = UnetSpectrogramSeparator(cfg)
    in_shape, out_shape = sep.get_padding(np.array([4, cfg["num_frames"], 0]))
    assert list(in_shape) == list(out_shape) == [4, PRESET_FRAMES, 1]
    eng = sep.engine(num_frames=PRESET_FRAMES)
    assert (eng.T_in, eng.T_out, eng.stft_frames) == (PRESET_FRAMES, PRESET_FRAMES, 128)
    assert eng.param_numel == 2 * 9824817
    names = [n for n, _, _, _ in eng.param_table]
    assert names.index("separator/conv2d_6/kernel") == len(names) // 2
    assert "separator/BatchNorm_11/beta" in names[len(names) // 2:len(names) // 2 + 5]
    # closed form: 2 FLOP per MAC over all 25 taps; down layers over their outputs, transposed convs over their inputs
    L, F, n, W = 6, 16, 128, 512
    macs = 0
    for i in range(L):
        macs += (n >> (i + 1)) * (W >> (i + 1)) * 25 * (1 if i == 0 else F << (i - 1)) * (F << i)
    cin = F << (L - 1)
    for i in range(L - 1):
        cout = F << (L - i - 2)
        macs += (n >> (L - i)) * (W >> (L - i)) * 25 * cin * cout
        cin = 2 * cout
    macs += (n >> 1) * (W >> 1) * 25 * cin
    assert eng.forward_flops(1) == pytest.approx(2 * 2 * macs, rel=1e-12)
    assert abs(eng.forward_flops(1) / 1e9 - 3.015) < 5e-4
    assert eng.forward_flops(4) == pytest.approx(4 * eng.forward_flops(1), rel=1e-12)
    assert eng.launches(False) == 1 + 2 * (2 * L + 2) and eng.launches(True) == 1 + 2 * 2 * L
    assert eng.workspace_bytes(4) > 0


def test_bad_shapes_are_rejected_like_the_reference():
    cfg = mc("unet_spectrogram")
    with pytest.raises(AssertionError):
        UnetSpectrogramSeparator(mc("unet_spectrogram", mono_downmix=False))
    with pytest.raises(AssertionError):
        UnetSpectrogramSeparator(mc("unet_spectrogram", task="multi_instrument"))
    c = wun.spec_config_from_model_config(cfg)
    for T in (PRESET_FRAMES + 1, PRESET_FRAMES - 768, 1023, 1024 + 768 * 64):     # hop misfit, 127 / 1 / 65 frames
        with pytest.raises(AssertionError):
            wun.SpecEngine(c, num_frames=T)
    stereo = wun.spec_config_from_model_config(mc("unet_spectrogram", mono_downmix=False))
    with pytest.raises(AssertionError):
        wun.SpecEngine(stereo, num_frames=PRESET_FRAMES)
    four = wun.spec_config_from_model_config(mc("unet_spectrogram", task="multi_instrument"))
    with pytest.raises(AssertionError):
        wun.SpecEngine(four, num_frames=PRESET_FRAMES)
    with pytest.raises(AssertionError):                           # 512 bins are not divisible by 2^10
        wun.SpecEngine(wun.spec_config_from_model_config(mc("unet_spectrogram", num_layers=10)), num_frames=PRESET_FRAMES)


def test_training_graph_is_not_available():
    sep = UnetSpectrogramSeparator(mc("unet_spectrogram"))
    with pytest.raises(NotImplementedError):
        sep.get_output(np.zeros((1, PRESET_FRAMES, 1), np.float32), True)


def _checkpoint_tensors(cfg, T, seed, drop=None):
    params = S.random_params(cfg["num_layers"], cfg["num_initial_filters"], seed)
    if drop is not None:
        params = {n: a for n, a in params.items() if not n.endswith(drop)}
    rng = np.random.default_rng(seed + 1)
    m = {n: rng.standard_normal(a.shape).astype(np.float32) for n, a in params.items()}
    v = {n: rng.uniform(0, 1, a.shape).astype(np.float32) for n, a in params.items()}
    return params, TFCheckpoint.separator_tensors(params, m, v, global_step=1234)


def test_checkpoint_round_trip_through_load_separator(tmp_path):
    cfg = mc("unet_spectrogram", num_layers=3, num_initial_filters=4, num_frames=1024 + 768 * 7)
    params, tensors = _checkpoint_tensors(cfg, cfg["num_frames"], seed=5)
    prefix = TFCheckpoint.write_checkpoint(str(tmp_path / "u7-1234"), tensors)
    sep = Evaluate.load_separator(cfg, prefix)
    assert isinstance(sep, UnetSpectrogramSeparator) and sep.global_step == 1234
    flat = sep.params.cpu().numpy()
    for name, shape, off, numel in sep.param_table():
        np.testing.assert_array_equal(flat[off:off + numel].reshape(shape), params[name])
    assert sep.params.numel() == sum(a.size for a in params.values())


def test_checkpoint_without_moving_variance_is_refused(tmp_path):
    cfg = mc("unet_spectrogram_l1", num_layers=2, num_initial_filters=2, num_frames=1024 + 768 * 3)
    _, tensors = _checkpoint_tensors(cfg, cfg["num_frames"], seed=9, drop="/moving_variance")
    prefix = TFCheckpoint.write_checkpoint(str(tmp_path / "u7a-1"), tensors)
    with pytest.raises(TFCheckpoint.CheckpointError):
        Evaluate.load_separator(cfg, prefix)


def test_load_separator_dispatches_on_network():
    from Models.UnetAudioSeparator import UnetAudioSeparator
    assert isinstance(Evaluate.load_separator(mc("baseline"), None), UnetAudioSeparator)
    assert isinstance(Evaluate.load_separator(mc("unet_spectrogram"), None), UnetSpectrogramSeparator)
    with pytest.raises(NotImplementedError):
        Evaluate.load_separator(mc("baseline", network="gan"), None)
