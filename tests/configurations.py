"""Configurations and oracle comparisons that several suites run: the forced pair-merge switches, the launch-replay
configurations, the A/B switch positions, the seeded random-configuration draws, the bars of two training steps against the
oracle, the plan audit of a preset and the parity helpers of the GPU tests against the oracle."""
import numpy as np

import Config
from oracle import wave_unet_oracle as O
from helpers import live_rows

FORCED = {"WUN_PAIR_MIN_CTAS": "1", "WUN_PAIR_DGRAD": "1"}     # the pair-merged conv variants, forced onto mid-size nets

# the launch replays of tests/test_kernels_gpu.py and test_step_kernels_gpu.py:
# (name, named presets, overrides, batch, num_frames (None: the preset's), environment)
REPLAYS = [("m4_like_L5", ["baseline_stereo"], dict(num_layers=5), 3, 200, {}),
           ("m5_like_L4", ["full"], dict(num_layers=4, num_initial_filters=16), 2, 123, {}),
           ("m6_like_L4", ["full_multi_instrument"], dict(num_layers=4), 2, 77, {}),
           ("m1_like_L5", ["baseline"], dict(num_layers=5), 3, 256, {}),
           ("same_learned_stereo", ["baseline_diff"], dict(num_layers=4, upsampling="learned", mono_downmix=False), 2, 128, {}),
           ("odd_filters", ["baseline_context"], dict(num_layers=3, filter_size=9, input_filter_size=9, merge_filter_size=3,
                                                       num_initial_filters=10, output_filter_size=3), 2, 50, {}),
           ("forced_m4_like_L5", ["baseline_stereo"], dict(num_layers=5), 3, 2000, FORCED),
           ("forced_m5_like_L4", ["full"], dict(num_layers=4, num_initial_filters=16), 2, 1500, FORCED),
           ("forced_m6_like_L4", ["full_multi_instrument"], dict(num_layers=4), 2, 1200, FORCED),
           ("forced_m1_like_L5", ["baseline"], dict(num_layers=5), 3, 4096, FORCED),
           ("forced_same_learned_stereo", ["baseline_diff"], dict(num_layers=4, upsampling="learned", mono_downmix=False), 2, 2048,
            FORCED),
           ("M1_full", ["baseline"], {}, 1, None, {}), ("M4_full", ["baseline_stereo"], {}, 1, None, {}),
           ("M5_full", ["full"], {}, 1, None, {}), ("M6_full", ["full_multi_instrument"], {}, 1, None, {}),
           ("M4_full_b16", ["baseline_stereo"], {}, 16, None, {})]

SWITCHES = [
    {"WUN_OUT_FUSE": "2"},                       # output-layer switch in its other positions (the output layer runs in its own
    {"WUN_OUT_FUSE": "0"},                       #   kernels either way: the step must not change)
    {"WUN_BULK_WGRAD": "0"},                     # converter-fed tensor-core wgrad, bias sums by colsum_kernel
    {"WUN_SPLIT_COLSUM": "0"},
    {"WUN_FIRST_LAYER": "0"},                    # first layer through the generic plane kernels
    {"WUN_DISABLE_UMMA": "1"},                   # the exact-fp32 CUDA-core path for everything
    {"WUN_UMMA_DGRAD": "0"},
    {"WUN_PAIR_FWD": "0", "WUN_PAIR_DGRAD": "0"},
    {"WUN_SIDE_STREAM": "0"},
]


def random_model_configs(n, seed):
    """n reproducible draws from the space of shapes the reference allows (Config.py:9-39 keys the separator reads)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        L = int(rng.integers(1, 5))
        context = bool(rng.integers(0, 2))
        # (even filter widths only with 'same' padding: with context they make T_in - T_out odd, which the reference's callers
        #  assert against - Test.py:25)
        fs = int(rng.choice([3, 5, 7, 9, 15] if context else [3, 5, 7, 9, 15, 4, 6]))
        ov = dict(num_layers=L, num_initial_filters=int(rng.choice([4, 8, 12, 16, 24, 40])), filter_size=fs, input_filter_size=fs,
                  merge_filter_size=int(rng.choice([1, 3, 5] if context else [1, 3, 5, 2])), output_filter_size=int(rng.choice([1, 1, 1, 3])), context=context,
                  upsampling=str(rng.choice(["linear", "learned"])), output_type=str(rng.choice(["direct", "difference"])),
                  output_activation=str(rng.choice(["tanh", "linear"])), mono_downmix=bool(rng.integers(0, 2)),
                  task=str(rng.choice(["voice", "multi_instrument"])))
        nf = int(rng.integers(40, 200)) if context else int((2 ** L) * rng.integers(4, 24))
        out.append(("draw%02d" % i, ["baseline"], ov, int(rng.integers(1, 4)), nf, None, 1.0))
    return out


def assert_steps_match_oracle(res, loss_tol=1e-5, grad_tol=1e-4, out_tol=1e-5):
    """The bars of two training steps with Adam and the inference calls (the result form of tests/hostsim/run_cpu_step.py).  The
    defaults are the CPU device's (tests/test_cpu_device.py); tests/test_configurations_gpu.py holds the GPU to the same checks
    with the wider loss / gradient / output bars of the fp32 tensor-core arithmetic."""
    for step in ("step1", "step2"):
        r = res[step]
        assert r["loss_rel"] < loss_tol, (step, r)
        ex = r.get("grad_explained")           # None, or the LeakyReLU-slope-flip proof for a gradient that is off (run_cpu_step.py)
        assert r["grad_worst_rel"] < grad_tol or (ex and ex["flips"] is not None and ex["worst_after"] < grad_tol), (step, r)
        assert r["outputs_rel"] < out_tol, (step, r)
        assert r["params_rel"] < 1e-5 and r["adam_slots_rel"] < 1e-4, (step, r)
    assert res["infer_outputs_rel"] < 1e-4, res["infer_outputs_rel"]
    assert res["train_mode_outputs_rel"] < 1e-4, res["train_mode_outputs_rel"]
    assert res["gather_exact"] and res["scatter_exact"]          # predict_track's window tiling (Evaluate.py:125-139)
    assert abs(res["adam_state"][0] - 0.9 ** 3) < 1e-6 and abs(res["adam_state"][1] - 0.999 ** 3) < 1e-6 and res["adam_state"][2] == 2.0


def plan_audit(preset, batch, overrides=None):
    """The engine's plan audit of a training step of `preset` at its full window and `batch` (host only)."""
    from Models.UnetAudioSeparator import UnetAudioSeparator
    mc = Config.build_config([preset], overrides or {}, experiment_id=0)["model_config"]
    sep = UnetAudioSeparator(mc)
    return sep.engine(num_frames=mc["num_frames"]).plan_audit(batch)


# The GPU against the oracle: separated sources within 1e-4 relative (rel-L2 and max-abs / max), gradients within 1e-3 rel-L2
# per tensor (tests/test_gpu_parity.py says why)
OUT_TOL = 1e-4
GRAD_TOL = 1e-3


def rel_l2(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def rel_max(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def engine_masks(sep, cfg, batch, t_in):
    """LeakyReLU slopes the ENGINE used in its last training step: sign of every saved (post-activation) tensor at the
    rows it keeps, as {LeakyReLU call index: [(rows, bool[B, len(rows), C])]} for O.forward_backward_with_masks."""
    eng = sep.engine(input_frames=t_in)
    masks = {}
    for idx, views in live_rows(cfg, t_in).items():
        masks[idx] = []
        for name, rows in views:
            m = eng.debug_tensor(name, batch, True).cpu().numpy() > 0
            assert m.shape[1] == len(rows), (name, m.shape, len(rows))
            masks[idx].append((rows, m))
    return masks


def make_sep(cfg, params, t_in):
    from Models.UnetAudioSeparator import UnetAudioSeparator
    sep = UnetAudioSeparator(cfg)
    sep.load_variables(params, input_frames=t_in)
    return sep


def check_outputs(got, want, names, tol=OUT_TOL):
    assert list(got.keys()) == list(names)
    for s in names:
        g = got[s].detach().cpu().numpy()
        assert g.shape == want[s].shape
        assert rel_l2(g, want[s]) <= tol, (s, rel_l2(g, want[s]))
        assert rel_max(g, want[s]) <= tol, (s, rel_max(g, want[s]))


def random_problem(cfg, batch, num_frames, seed):
    t_in, t_out = O.get_padding(cfg, num_frames)
    params = O.init_params(cfg, seed=seed)
    rng = np.random.default_rng(seed + 1)
    for k in params:
        if k.endswith("/bias"):
            params[k] = rng.uniform(-0.05, 0.05, size=params[k].shape).astype(np.float32)
    mix, targets = O.synthetic_batch(cfg, batch, t_in, t_out, seed=seed + 2)
    return t_in, t_out, params, mix, targets
