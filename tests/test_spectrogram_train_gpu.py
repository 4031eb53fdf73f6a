"""Training the spectrogram U-Net baselines (U7 / U7a) on the GPU (csrc/kernels_spec_train.cu, csrc/spec.cu): one step's
loss, gradients and moving statistics against the float64 oracle run with the engine's own dropout masks, Adam against
TF's formula, bit reproducibility, a captured CUDA graph of a whole step, Training.train's checkpoint and resume, and the
loss falling on a fixed batch.

Tolerance.  Every kernel accumulates in float32 in a fixed order (the channel statistics in float64): a convolution sums up
to 25 * 512 products, a weight gradient up to B * 64 * 256 of them; with unit round-off u = 6e-8 a sum of m terms is
typically off by ~sqrt(m) u relative to the sum of magnitudes.  The forward runs 2L layers, the backward 2L more, and batch
norm's backward subtracts two means from dy, so a gradient element carries a few 1e-6 of its tensor's scale.  Each trainable
tensor is checked against 1e-3 of its largest oracle value, far above that and far below a wiring mistake (a wrong tap,
channel half, mask or scale moves a tensor by O(1) of its scale).  The biases of the convolutions that feed batch norm have
a zero gradient in exact arithmetic; the engine, as TF, sums dz = rstd (dy - mean dy - xhat mean(dy xhat)), whose terms
cancel, so their bound is absolute: 64 u times the oracle's rstd * sum(|dy| + |mean dy| + |xhat mean(dy xhat)|) of the
channel, the magnitude the float32 roundings act on.  The worst errors seen are printed (-s)."""
import os

import numpy as np
import pytest
import torch

import Config
import TFCheckpoint
import Training
from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator
from oracle import spectrogram_oracle as S
from oracle import spectrogram_train_oracle as O

pytestmark = pytest.mark.gpu

TOL = 1e-3
U = 2.0 ** -24
PRESET_FRAMES = 768 * 127 + 1024


def mc(named="unet_spectrogram", **kw):
    return Config.build_config([named], kw, experiment_id=0)["model_config"]


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)


def signal(rng, B, T):
    t = np.arange(T) / 8192.0
    x = [0.3 * np.sin(2 * np.pi * rng.uniform(80, 900) * t) + rng.uniform(-0.4, 0.4, T) for _ in range(B)]
    return np.stack(x)[:, :, None].astype(np.float32)


def batch(seed, B, T):
    rng = np.random.default_rng(seed)
    src = [0.5 * signal(rng, B, T), 0.5 * signal(rng, B, T)]
    return (src[0] + src[1]).astype(np.float32), src


def separator(cfg, params, T):
    sep = UnetSpectrogramSeparator(cfg)
    sep.load_variables(params, device=torch.device("cuda"), num_frames=T)
    return sep


def engine_step(sep, mix, targets):
    """One forward_backward: (loss, grads dict, moving statistics dict, the dropout step it used)."""
    sep._ensure_training_state()
    step = int(sep._dropout_step.item())
    loss = sep.loss_and_gradients(torch.from_numpy(mix).cuda(), torch.from_numpy(np.stack(targets)).cuda())
    g = {n: t.cpu().numpy().copy() for n, t in sep.gradients().items()}
    p = {n: t.cpu().numpy().copy() for n, t in sep.variables().items()}
    moving = {n: v for n, v in p.items() if not O.trainable(n)}
    return float(loss.item()), g, moving, step


def gradient_errors(g, want_g, scale, names):
    """{name: error}: relative to the tensor's largest oracle value, or for a batch-norm-fed bias the ratio to its bound."""
    out = {}
    for name in names:
        got, want = g[name], want_g[name]
        if name in scale:
            out[name] = float(np.max(np.abs(got - want) / (64 * U * scale[name]))) * TOL
        else:
            out[name] = float(np.abs(got - want).max() / np.abs(want).max())
    return out


def engine_slopes(sep, cfg, B, T):
    """{batch-norm index: activation > 0} of the last source's U-Net, read from the engine's saved activations."""
    L, Fi = cfg["num_layers"], cfg["num_initial_filters"]
    eng = sep.engine(num_frames=T)
    base = 2 * L - 1                                  # batch norms per U-Net; the last source's come second
    pos = {}
    for d in range(L):
        lev = eng.debug_train_level(B, d, sep.params.device).cpu().numpy()
        c = Fi * 2 ** d
        pos[base + d] = lev[..., :c] > 0
        if d < L - 1:
            pos[base + L + (L - 2 - d)] = lev[..., c:] > 0
    return pos


def swapped(params, names):
    half = len(names) // 2
    out = dict(params)
    for a, b in zip(names[:half], names[half:]):
        out[a], out[b] = params[b], params[a]
    return out


def prove_slope_flips(cfg, params, mix, targets, label):
    """The engine's gradients are exact for the activation slopes it used: for the second U-Net, whose activations stay in
    the workspace, the oracle repeats the step with the engine's slopes; then every tensor must agree to TOL, and the
    slopes may differ from the oracle's own only at pre-activations within 1e-4 * rms of zero (forward rounding noise) and
    at fewer than 1e-5 of the elements.  A second step with the two U-Nets' variables and targets swapped covers the
    first U-Net's variables the same way."""
    L, Fi = cfg["num_layers"], cfg["num_initial_filters"]
    B, T = mix.shape[0], mix.shape[1]
    names = [n for n, _ in S.param_specs(L, Fi)]
    second = [n for n in names[len(names) // 2:] if O.trainable(n)]
    worst = 0.0
    for swap in (False, True):
        p = swapped(params, names) if swap else params
        t = targets[::-1] if swap else targets
        sep = separator(cfg, p, T)
        _, g, _, step = engine_step(sep, mix, t)
        report, scale = [], {}
        _, want_g, _ = O.forward_backward(p, mix, t, L, cfg["source_names"], cfg["raw_audio_loss"],
                                          O.engine_masks(sep.seed, step, B, S.stft_frames(T), L, Fi), bias_scale=scale,
                                          positive=engine_slopes(sep, cfg, B, T), report=report)
        err = gradient_errors(g, want_g, scale, second)
        assert max(err.values()) < TOL, ("not explained by activation slope flips", label, swap,
                                         sorted(err.items(), key=lambda kv: -kv[1])[:3])
        n_flip = sum(r[1] for r in report)
        n_elem = sum(int(np.prod(v.shape)) for v in engine_slopes(sep, cfg, B, T).values())
        assert all(r[2] <= 1e-4 for r in report), ("a slope differs away from zero", report)
        assert n_flip <= max(4, 1e-5 * n_elem), (n_flip, n_elem)
        worst = max(worst, max(err.values()))
        print("%s%s: exact for the engine's own slopes, %d of %d differ from the oracle's, all within %.1e * rms of 0; "
              "worst tensor %.2e" % (label, " (swapped)" if swap else "", n_flip, n_elem,
                                     max([r[2] for r in report] + [0.0]), max(err.values())))
    return worst


def check_step(cfg, params, mix, targets, label):
    L, Fi = cfg["num_layers"], cfg["num_initial_filters"]
    B, T = mix.shape[0], mix.shape[1]
    sep = separator(cfg, params, T)
    loss, g, moving, step = engine_step(sep, mix, targets)
    masks = O.engine_masks(sep.seed, step, B, S.stft_frames(T), L, Fi)
    scale = {}
    want_loss, want_g, want_moving = O.forward_backward(params, mix, targets, L, cfg["source_names"], cfg["raw_audio_loss"],
                                                        masks, bias_scale=scale)
    assert abs(loss - want_loss) <= 1e-5 * abs(want_loss), (label, loss, want_loss)
    for name, want in want_moving.items():
        e = float(np.abs(moving[name] - want).max() / max(np.abs(want).max(), 1e-30))
        assert e < 1e-5, (label, name, e)
    err = gradient_errors(g, want_g, scale, list(want_g))
    plain = {n: e for n, e in err.items() if n not in scale}
    biases = {n: e / TOL for n, e in err.items() if n in scale}
    print("%s: loss %.9g (oracle %.9g), worst gradient %.2e of its tensor's max (%s), BN-fed biases at %.2f of their bound"
          % (label, loss, want_loss, max(plain.values()), max(plain, key=plain.get), max(biases.values())))
    if max(err.values()) >= TOL:
        prove_slope_flips(cfg, params, mix, targets, label)


FIXTURES = ["train_l2_u7", "train_l3_u7a", "train_l5_u7"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spectrogram_train")


@pytest.mark.parametrize("name", FIXTURES)
def test_engine_matches_reference_training_fixtures(name):
    """The fixtures' dropout masks are the engine's hash at the recorded seed and dropout step, so the engine runs the very
    step the reference's graph was differentiated on."""
    import json
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = json.loads(str(z["cfg_json"]))
    params = {k[len("param/"):]: z[k].astype(np.float32) for k in z.files if k.startswith("param/")}
    mix = z["mix_pcm16"].astype(np.float32) / np.float32(32768)
    targets = [z["target_pcm16"][k].astype(np.float32) / np.float32(32768) for k in range(2)]
    L, Fi, B, T = cfg["num_layers"], cfg["num_initial_filters"], mix.shape[0], mix.shape[1]
    sep = separator(cfg, params, T)
    sep.seed = int(z["dropout_seed"])
    sep._ensure_training_state()
    sep._dropout_step.fill_(int(z["dropout_step"]))
    loss, g, moving, _ = engine_step(sep, mix, targets)
    assert abs(loss - float(z["loss"])) <= 1e-5 * abs(float(z["loss"])), (name, loss, float(z["loss"]))
    for n, v in moving.items():
        want = z["moving/" + n]
        assert float(np.abs(v - want).max() / np.abs(want).max()) < 1e-5, (name, n)
    scale = {}
    masks = O.engine_masks(sep.seed, int(z["dropout_step"]), B, S.stft_frames(T), L, Fi)
    O.forward_backward(params, mix, targets, L, cfg["source_names"], cfg["raw_audio_loss"], masks, bias_scale=scale)
    want_g = {k[len("grad/"):]: z[k].astype(np.float64) for k in z.files if k.startswith("grad/")}
    err = gradient_errors(g, want_g, scale, list(want_g))
    print("fixture %s: loss %.9g (reference %.9g), worst gradient %.2e (%s)"
          % (name, loss, float(z["loss"]), max(err.values()), max(err, key=err.get)))
    if max(err.values()) >= TOL:
        prove_slope_flips(cfg, params, mix, targets, name)


SMALL = [
    # (label, preset, layers, filters, STFT frames, batch)
    ("l2_u7", "unet_spectrogram", 2, 4, 4, 2),
    ("l3_u7a", "unet_spectrogram_l1", 3, 3, 8, 2),
    ("l5_u7", "unet_spectrogram", 5, 2, 32, 2),
    ("l5_u7a", "unet_spectrogram_l1", 5, 2, 32, 2),
]


@pytest.mark.parametrize("label,preset,L,Fi,n,B", SMALL, ids=[c[0] for c in SMALL])
def test_small_configurations_match_oracle(label, preset, L, Fi, n, B):
    T = 1024 + 768 * (n - 1)
    cfg = mc(preset, num_layers=L, num_initial_filters=Fi, num_frames=T)
    params = S.random_params(L, Fi, seed=100 + L)
    mix, targets = batch(L, B, T)
    check_step(cfg, params, mix, targets, label)


@pytest.mark.parametrize("preset", ["unet_spectrogram", "unet_spectrogram_l1"])
def test_presets_at_full_size_match_oracle(preset):
    cfg = mc(preset)
    params = S.random_params(cfg["num_layers"], cfg["num_initial_filters"], seed=21)
    mix, targets = batch(5, 4, PRESET_FRAMES)
    check_step(cfg, params, mix, targets, preset)


def test_adam_step_matches_tf_formula_and_keeps_moving_statistics():
    T = 1024 + 768 * 7
    cfg = mc("unet_spectrogram_l1", num_layers=3, num_initial_filters=3, num_frames=T)
    sep = separator(cfg, S.random_params(3, 3, seed=8), T)
    mix, targets = batch(9, 2, T)
    _, g, moving, _ = engine_step(sep, mix, targets)
    before = {n: t.cpu().numpy().copy() for n, t in sep.variables().items()}
    lr = 1e-3
    sep.adam_step(lr)
    after = {n: t.cpu().numpy() for n, t in sep.variables().items()}
    zero = {n: np.zeros_like(a) for n, a in g.items()}
    is_mask = lambda n: "transpose" in n and g[n.replace("/bias", "/kernel")].shape[2] == 1
    bn_fed = {n for n in g if n.endswith("/bias") and not is_mask(n)}
    want, _, _ = O.adam(before, {n: a for n, a in g.items() if O.trainable(n)}, zero, zero, 1, lr)
    worst = 0.0
    for n in before:
        if not O.trainable(n):
            assert np.array_equal(bits(after[n]), bits(before[n])), n
            continue
        d_got, d_want = after[n].astype(np.float64) - before[n], want[n] - before[n]
        if n in bn_fed:
            # rounding-noise gradients (~1e-20 and below, squares in float32's subnormal range): Adam's step is bounded
            # by lr * |m| / sqrt(v) = lr * sqrt(1 - b2) / (1 - b1) ~ 3.2 lr at the first step
            assert np.abs(d_got).max() <= 3.2 * lr * (1 + 1e-3), n
            continue
        e = float(np.abs(d_got - d_want).max() / np.abs(d_want).max())
        worst = max(worst, e)
        assert e < 1e-3, (n, e)
    assert sep.global_step == 1
    print("Adam: worst update error %.2e of the tensor's largest update" % worst)


def run_steps(cfg, params, T, k, lr=1e-3):
    sep = separator(cfg, params, T)
    losses = []
    for i in range(k):
        mix, targets = batch(40 + i, 2, T)
        losses.append(engine_step(sep, mix, targets)[0])
        sep.adam_step(lr)
    return sep, losses


def state_bits(sep):
    return [bits(t.cpu().numpy()) for t in (sep.params, sep.adam_m, sep.adam_v, sep._adam_state, sep._dropout_step)]


def test_three_steps_repeat_bit_for_bit():
    T = 1024 + 768 * 15
    cfg = mc("unet_spectrogram", num_layers=4, num_initial_filters=3, num_frames=T)
    params = S.random_params(4, 3, seed=13)
    a, la = run_steps(cfg, params, T, 3)
    b, lb = run_steps(cfg, params, T, 3)
    assert bits(np.array(la)).tobytes() == bits(np.array(lb)).tobytes()
    for x, y in zip(state_bits(a), state_bits(b)):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("preset", ["unet_spectrogram", "unet_spectrogram_l1"])
def test_captured_graph_replays_equal_eager_steps(preset):
    from wun.feeder import DeviceFeeder, synthetic_tracks
    T = 1024 + 768 * 7
    cfg = mc(preset, num_layers=3, num_initial_filters=4, num_frames=T)
    params = S.random_params(3, 4, seed=17)
    tracks = synthetic_tracks(cfg["source_names"], 1, 4, (T + 100, 2 * T), seed=3)
    k, lr = 3, 1e-3

    def make():
        sep = separator(cfg, params, T)
        eng = sep.engine(num_frames=T)
        feeder = DeviceFeeder(eng, tracks, cfg["source_names"], 2, augmentation=True, seed=5, device="cuda")
        sep._ensure_training_state()
        return sep, feeder

    eager, fe = make()
    for _ in range(k):
        mix, tg = fe.next_batch()
        eager.loss_and_gradients(mix, tg)
        eager.adam_step(lr)
    graphed, fg = make()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eng = graphed.engine(num_frames=T)
        # allocates the training workspace outside the capture; the state it touched is reloaded below
        eng.forward_backward(graphed.params, torch.zeros_like(fg.mix), torch.zeros_like(fg.targets), graphed.grads,
                             graphed._loss, graphed.raw_audio_loss, graphed.seed,
                             torch.zeros(1, dtype=torch.int64, device="cuda"))
    torch.cuda.current_stream().wait_stream(side)
    graphed.load_variables({n: params[n] for n in params})
    graphed._ensure_training_state()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        mix, tg = fg.next_batch()
        graphed.loss_and_gradients(mix, tg)
        graphed.adam_step(lr)
    for _ in range(k):
        g.replay()
    torch.cuda.synchronize()
    assert bits(eager._loss.cpu().numpy()).tobytes() == bits(graphed._loss.cpu().numpy()).tobytes()
    for x, y in zip(state_bits(eager), state_bits(graphed)):
        assert np.array_equal(x, y)
    assert graphed.global_step == k


def test_training_train_checkpoints_restores_and_resumes(tmp_path):
    T = 1024 + 768 * 7
    cfg = mc("unet_spectrogram_l1", num_layers=2, num_initial_filters=4, num_frames=T, batch_size=2, epoch_it=3,
             model_base_dir=str(tmp_path / "ck"), log_dir=str(tmp_path / "log"))
    path, sep = Training.train(dict(cfg), 7, log_every=0)
    assert sep.global_step == 3 and os.path.exists(path + ".index")
    names = [v[0] for v in TFCheckpoint.list_variables(path)]
    fresh = UnetSpectrogramSeparator(cfg)
    TFCheckpoint.restore_separator(path, fresh, T)
    assert fresh.global_step == 3
    assert np.array_equal(bits(fresh.params.cpu().numpy()), bits(sep.params.cpu().numpy()))
    trainable = np.zeros(sep.params.numel(), bool)
    for _, o, c in sep.engine(num_frames=T).trainable_ranges:
        trainable[o:o + c] = True
    for a, b in ((fresh.adam_m, sep.adam_m), (fresh.adam_v, sep.adam_v)):
        assert np.array_equal(bits(a.cpu().numpy()[trainable]), bits(b.cpu().numpy()[trainable]))
    slots = [n for n in names if n.endswith(("/Adam", "/Adam_1"))]
    assert len(slots) == 2 * len(sep.trainable_variable_names())
    assert not any("moving_" in n for n in slots)
    path2, sep2 = Training.train(dict(cfg), 7, load_model=path, log_every=0)
    assert sep2.global_step == 6 and path2.endswith("7-6")
    loss = Training.validation_loss(dict(cfg), sep2)
    assert np.isfinite(loss) and loss > 0


@pytest.mark.parametrize("preset", ["unet_spectrogram", "unet_spectrogram_l1"])
def test_loss_falls_on_a_fixed_batch(preset):
    T = 1024 + 768 * 15
    cfg = mc(preset, num_layers=3, num_initial_filters=8, num_frames=T)
    sep = separator(cfg, S.random_params(3, 8, seed=2), T)
    mix, targets = batch(77, 4, T)
    mix_d, tg_d = torch.from_numpy(mix).cuda(), torch.from_numpy(np.stack(targets)).cuda()
    losses = []
    for _ in range(50):
        losses.append(float(sep.loss_and_gradients(mix_d, tg_d).item()))
        sep.adam_step(2e-3)
    first, last = np.mean(losses[:5]), np.mean(losses[-5:])
    print("%s: loss %.5g over the first 5 steps, %.5g over the last 5" % (preset, first, last))
    assert np.isfinite(losses).all() and last < 0.9 * first
