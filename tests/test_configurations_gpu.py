"""The configurations the GPU actually runs, checked on the GPU: the benchmarked batch sizes, the two reference presets no other test
builds (baseline_context_smallfilter_deep, baseline_comparison), the seeded random-configuration sweep and every A/B switch.

The planner's choices depend on the model and on the batch (output-channel splits, pair merging, batch-folded wgrad chunks, CUDA-core
fallback for channel counts that are not multiples of 8, the dedicated first layer or not), so the launch sets these configurations
emit are not the ones the smaller replay and parity tests reach.  Four checks:
  A  every conv / dgrad / wgrad / first / output / upsample / Adam launch of each configuration, alone, against the float64
     interpreter, with the bounds, sentinels and "outside the views" checks of tests/test_kernels_gpu.py and
     tests/test_step_kernels_gpu.py (the replays of tests/conv_launches.py and tests/step_launches.py);
  B  whole training steps against the oracle with the bars of tests/test_gpu_parity.py (outputs 1e-4, gradients 1e-3 or proven
     LeakyReLU slope flips), grads(B) == sum of per-example grads, and windowed prediction over two forward batch sizes;
  C  the random sweep of tests/test_cpu_device.py (same draws) on the device: two training steps with Adam plus inference against
     the oracle with that file's bars, and the launch replays of A;
  D  every switch of SWITCHES (tests/configurations.py) against the oracle and against the default path's gradients.
A host-only test (E) asserts from the dry runs that the configurations still reach the paths A-D are meant to cover.

Run with -s for the per-configuration table: launches replayed per kernel family, worst err / ref_abs against its bound, the
peak device memory and the time per configuration.
"""
import time
from collections import OrderedDict, defaultdict

import numpy as np
import pytest
import torch

import Config
import wun
from configurations import (FORCED, GRAD_TOL, OUT_TOL, SWITCHES, assert_steps_match_oracle, check_outputs, engine_masks, make_sep,
                            random_model_configs, random_problem, rel_l2, rel_max)
from conv_launches import replay_conv_and_wgrad
from launch_checks import engine, gpu_lib, lib_or_skip, print_report, set_env
from oracle import wave_unet_oracle as O
from step_launches import replay_step_launches

START = time.time()
REPORT = OrderedDict()               # configuration -> (peak device GB, seconds)

# (name, named presets, overrides, batch, num_frames (None: the preset's), environment)
CONFIGS = [
    ("M5_full_b16", ["full"], {}, 16, None, {}),
    ("M6_full_b4", ["full_multi_instrument"], {}, 4, None, {}),
    ("M6_full_b32", ["full_multi_instrument"], {}, 32, None, {}),
    ("M1_full_b16", ["baseline"], {}, 16, None, {}),
    ("smallfilter_deep_b2", ["baseline_context_smallfilter_deep"], {}, 2, None, {}),
    ("comparison_b4", ["baseline_comparison"], {}, 4, None, {}),
    ("forced_smallfilter_deep_b2", ["baseline_context_smallfilter_deep"], {}, 2, None, FORCED),
    ("forced_comparison_b4", ["baseline_comparison"], {}, 4, None, FORCED),
]
DRAWS = random_model_configs(16, seed=2026)
# The bars of assert_steps_match_oracle for the GPU.  The CPU device's reference routines accumulate in double; the GPU's forward
# is ~5e-6 from the oracle (three bf16 MMAs per fp32 product), and the loss, a mean of squared residuals, magnifies that as the
# residual shrinks: after one Adam step of the L=5 switch net the loss sits 1.1e-5 from float64 (1.0e-6 before it), and one
# learned-upsampling draw's interp gradient 1.3e-4.  These are the bars of tests/test_gpu_parity.py for outputs and gradients.
GPU_BARS = dict(loss_tol=1e-4, grad_tol=1e-3, out_tol=1e-4)


def model_config(named, ov):
    return Config.build_config(named, ov, experiment_id=0)["model_config"]


def tensor_core_expected(D):
    """A conv launch of these configurations runs on tensor cores exactly when every input plane's channel count is a multiple of
    8 (umma_plan_from_conv; any N >= 16 is padded to the tile)."""
    return D["launch"]["N"] >= 16 and all(P["C"] % 8 == 0 for P in D["planes"])


# ------------------------------------------------------------------------------------------------
# E: host only - the dry runs still reach what the GPU tests rely on
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,named,ov,batch,nf,env", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_configurations_reach_the_paths_their_gpu_tests_cover(name, named, ov, batch, nf, env, monkeypatch):
    """Host only: a planner change cannot quietly drop a path from the GPU tests of this file."""
    lib = lib_or_skip()
    set_env(monkeypatch, env)
    cfg, _, eng, descs = engine(named, ov, batch, nf)
    audit = eng.plan_audit(batch)
    wgmma = {(d["layer"], d["pass"]) for d in audit if d["op"] == "conv"}
    kinds = [k for k, _ in eng.step_launches]
    for D in descs:                                  # tensor cores exactly on the multiple-of-8 launches
        assert ((D["launch"]["layer"], D["launch"]["pass"]) in wgmma) == tensor_core_expected(D), (name, D["launch"])
    if "comparison" in name:
        simt = [D for D in descs if not tensor_core_expected(D)]
        assert len(simt) >= len(descs) // 2 and len(wgmma) > 0, (len(simt), len(descs), len(wgmma))
        assert max(sum(P["C"] for P in D["planes"]) for D in simt) > 512   # merge convs of ~850 input channels on CUDA cores
        assert "first" not in kinds and not lib.wkh_first_supported(cfg["num_channels"], cfg["num_initial_filters"],
                                                                      cfg["input_filter_size"])
        assert any(eng.layer_kernel(L, 2) == "simt" for L in range(2 * cfg["num_layers"] + 2))
    else:
        assert kinds.count("first") == 1
    if "smallfilter_deep" in name:
        classes = [q for D in descs for q in D["cls"]]
        assert any(q["term_end"] - q["term_begin"] == 1 for q in classes)          # merge_filter_size 1: single-tap classes
        assert any(0 < q["m_hi"] - q["m_lo"] < 16 for q in classes)                # the deepest levels: a few rows
    if name in ("M5_full_b16", "M6_full_b32"):
        assert sum(1 for d in audit if d["op"] == "conv" and d.get("nsplit", 1) > 1) >= 4
    if env and "smallfilter_deep" in name:
        assert any(d.get("pair") for d in audit if d["op"] == "conv")
    ups = [d for k, d in eng.step_launches if k == "upsample"]
    assert len(ups) == cfg["num_layers"]
    if cfg["upsampling"] == "learned":
        assert all(d["mid_mode"] != 1 for d in ups)                                # learned upsampling never uses MID_CLAMP
        assert all(P["mid_mode"] != 1 for D in descs for P in D["planes"] if P["kind"] == 1)


def test_random_draws_and_switch_nets_reach_their_paths_host_only(monkeypatch):
    """Host only: the random sweep keeps drawing CUDA-core launches and learned upsampling (never with MID_CLAMP), and every switch
    of SWITCHES changes the launch set it is meant to change."""
    lib_or_skip()
    set_env(monkeypatch, {})
    seen = defaultdict(int)
    for label, named, ov, batch, nf, _, _ in DRAWS:
        cfg = model_config(named, ov)
        try:
            t_in, _ = O.get_padding(cfg, nf)
            eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
        except AssertionError:
            continue
        descs = eng.launch_descriptions(batch)
        seen["feasible"] += 1
        seen["simt"] += sum(1 for D in descs if not tensor_core_expected(D))
        seen["wgmma"] += sum(1 for D in descs if tensor_core_expected(D))
        if cfg["upsampling"] == "learned":
            seen["learned"] += 1
            assert all(d["mid_mode"] != 1 for k, d in eng.step_launches if k == "upsample"), label
    assert seen["feasible"] >= 10 and seen["simt"] > 0 and seen["wgmma"] > 0 and seen["learned"] > 0, dict(seen)
    _, named, ov, batch, nf, _ = _switch_nets()[0]
    set_env(monkeypatch, FORCED)
    audit0 = engine(named, ov, batch, nf)[2].plan_audit(batch)
    for sw in SWITCHES:
        set_env(monkeypatch, dict(FORCED, **sw))
        eng = engine(named, ov, batch, nf)[2]
        audit = eng.plan_audit(batch)
        if sw.get("WUN_DISABLE_UMMA") == "1":
            assert not any(d["op"] == "conv" for d in audit)
        if sw.get("WUN_FIRST_LAYER") == "0":
            assert "first" not in [k for k, _ in eng.step_launches]
        if sw.get("WUN_PAIR_FWD") == "0":
            assert not any(d.get("pair") for d in audit if d["op"] == "conv")
            assert any(d.get("pair") for d in audit0 if d["op"] == "conv")
        if sw.get("WUN_UMMA_DGRAD") == "0":
            assert not any(d["op"] == "conv" and d["pass"] == 1 for d in audit)


# ------------------------------------------------------------------------------------------------
# A: launch-by-launch replays
# ------------------------------------------------------------------------------------------------
def replay_all(name, named, ov, batch, nf):
    gpu_lib()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    prefix = name + ": "
    n_conv = replay_conv_and_wgrad(name, named, ov, batch, nf, prefix=prefix)
    steps = replay_step_launches(name, named, ov, batch, nf, adam=True, prefix=prefix)
    REPORT[name] = (torch.cuda.max_memory_allocated() / 1e9, time.time() - t0)
    print_report(prefix + " kernel family", prefix)
    print("%s: %d conv / wgrad and %d step launches replayed, peak %.1f GB, %.0f s" % (name, n_conv, len(steps), REPORT[name][0],
                                                                                       REPORT[name][1]))
    return n_conv, steps


@pytest.mark.gpu
@pytest.mark.parametrize("name,named,ov,batch,nf,env", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_replayed_launches_of_the_configuration_match_float64(name, named, ov, batch, nf, env, monkeypatch):
    set_env(monkeypatch, env)
    replay_all(name, named, ov, batch, nf)


# ------------------------------------------------------------------------------------------------
# B: training steps against the oracle
# ------------------------------------------------------------------------------------------------
def step_vs_oracle(cfg, B, seed, per_example=True, oracle=True):
    """Estimates (test and train mode), loss and every gradient of one training step at batch B against the oracle, and with
    `per_example` grads(B) == the sum of the B per-example gradients at grad_scale = 1/B.  Returns the separator."""
    t_in, t_out, params, mix, targets = random_problem(cfg, B, cfg["num_frames"], seed)
    names = cfg["source_names"]
    sep = make_sep(cfg, params, t_in)
    mix_d = torch.from_numpy(mix).cuda()
    t_oracle = 0.0
    if oracle:
        for training in (False, True):
            t = time.time()
            want = O.forward_np(cfg, params, mix, training)
            t_oracle += time.time() - t
            check_outputs(sep.get_output(mix_d, training, False, reuse=True), want, names)
    tg = sep.stack_targets({k: torch.from_numpy(v).cuda() for k, v in targets.items()})
    outs = torch.empty((len(names), B, t_out, O.num_channels(cfg)), device="cuda")
    loss_b = float(sep.loss_and_gradients(mix_d, tg, outputs=outs).item())
    g_b = sep.grads.clone()
    named_b = {n: g.cpu().numpy().copy() for n, g in sep.gradients().items()}
    outs = outs.cpu().numpy()
    masks = engine_masks(sep, cfg, B, t_in)
    tab = sep.engine(input_frames=t_in).param_table
    per = {}
    if per_example:
        acc = torch.zeros_like(g_b)
        losses = []
        for b in range(B):
            losses.append(float(sep.loss_and_gradients(mix_d[b:b + 1].contiguous(), tg[:, b:b + 1].contiguous(),
                                                       grad_scale=1.0 / B).item()))
            acc += sep.grads
        assert abs(np.mean(losses) - loss_b) <= 1e-5 * loss_b, (np.mean(losses), loss_b)
        per = {n: rel_l2(g_b[o:o + c].cpu().numpy(), acc[o:o + c].cpu().numpy()) for n, _, o, c in tab}
        print("B=%d vs the sum of B=1 gradients: worst tensor %.2e" % (B, max(per.values())))
    per_o = {}
    if oracle:
        t = time.time()
        loss_o, outs_o, grads_o = O.forward_backward(cfg, params, mix, targets)
        t_oracle += time.time() - t
        assert abs(loss_b - loss_o) <= 1e-5 * abs(loss_o), (loss_b, loss_o)
        for k, s in enumerate(names):
            assert rel_l2(outs[k], outs_o[s]) <= OUT_TOL and rel_max(outs[k], outs_o[s]) <= OUT_TOL, s
        per_o = {n: rel_l2(named_b[n], grads_o[n]) for n in params}
        print("B=%d vs oracle: worst tensor %.2e (oracle CPU time %.0f s)" % (B, max(per_o.values()), t_oracle))
    if max(list(per_o.values()) + [0.0]) > GRAD_TOL or max(list(per.values()) + [0.0]) > 1e-4:
        # LeakyReLU slope flips (test_gpu_parity.check_grads): the oracle with the engine's own slopes of the batch-B step
        _, _, grads_m, report = O.forward_backward_with_masks(cfg, params, mix, targets, masks)
        per_m = {n: rel_l2(named_b[n], grads_m[n]) for n in params}
        assert max(per_m.values()) <= GRAD_TOL, sorted(per_m.items(), key=lambda kv: -kv[1])[:3]
        assert max(r[2] for r in report) <= 1e-4, report
        assert max(list(per.values()) + [0.0]) <= GRAD_TOL, max(per.values())
    return sep, t_in


@pytest.mark.gpu
@pytest.mark.parametrize("preset,B", [("full", 16), ("full_multi_instrument", 4)])
def test_benchmarked_batches_match_the_oracle(preset, B, monkeypatch):
    """M5 `full` at batch 16 (bench.py's M5 workload) and M6 at 4 per GPU (its 8-GPU split): the planner really takes output-channel
    splits here, and estimates, loss and every gradient match the oracle and the per-example sum."""
    set_env(monkeypatch, {})
    cfg = model_config([preset], {})
    sep, t_in = step_vs_oracle(cfg, B, 4243)
    audit = sep.engine(input_frames=t_in).plan_audit(B)
    assert sum(1 for d in audit if d["op"] == "conv" and d.get("nsplit", 1) > 1) >= 4


@pytest.mark.gpu
def test_m6_batch32_matches_the_per_example_sum_and_the_oracle(monkeypatch):
    """bench.py's one-GPU M6 workload (batch 32): grads(32) == the sum of the 32 per-example gradients, and the oracle."""
    set_env(monkeypatch, {})
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    step_vs_oracle(model_config(["full_multi_instrument"], {}), 32, 4244)
    REPORT["M6_full_b32 parity"] = (torch.cuda.max_memory_allocated() / 1e9, time.time() - t)


@pytest.mark.gpu
@pytest.mark.parametrize("preset,B", [("baseline_context_smallfilter_deep", 2), ("baseline_comparison", 4)])
def test_unrun_presets_match_the_oracle(preset, B, monkeypatch):
    """The two reference presets no other test builds, at their full window: 14 levels of single-tap merge convs down to a few
    rows, and 34 * k channels, mostly on the CUDA-core kernels with the first layer through the generic plane kernels."""
    set_env(monkeypatch, {})
    cfg = model_config([preset], {})
    sep, t_in = step_vs_oracle(cfg, B, 4245, per_example=False)
    eng = sep.engine(input_frames=t_in)
    descs = eng.launch_descriptions(B)
    wgmma = {(d["layer"], d["pass"]) for d in eng.plan_audit(B) if d["op"] == "conv"}
    for D in descs:
        assert ((D["launch"]["layer"], D["launch"]["pass"]) in wgmma) == tensor_core_expected(D), D["launch"]
    if preset == "baseline_comparison":
        assert any(not tensor_core_expected(D) for D in descs) and wgmma
        assert "first" not in [k for k, _ in eng.step_launches]
    else:
        assert any(q["term_end"] - q["term_begin"] == 1 for D in descs for q in D["cls"])
        assert any(0 < q["m_hi"] - q["m_lo"] < 16 for D in descs for q in D["cls"])


@pytest.mark.gpu
def test_predict_track_at_two_forward_batch_sizes_matches_the_oracle(monkeypatch):
    """Evaluate.predict_track with full_44KHz on a stereo track of 18 windows, 16 windows per forward: one handle runs a batch of
    16 and a batch of 2, against the oracle's window-by-window loop."""
    import Evaluate
    set_env(monkeypatch, {})
    cfg = model_config(["full_44KHz"], {})
    t_in, t_out, params, _, _ = random_problem(cfg, 1, cfg["num_frames"], 4246)
    n = 17 * t_out + t_out // 3
    assert len(Evaluate.window_starts(n, t_out)) == 18
    audio = (np.random.default_rng(4247).uniform(-1.0, 1.0, size=(n, 2)) * 0.5).astype(np.float32)
    sep = make_sep(cfg, params, t_in)
    got = Evaluate.predict_track(cfg, sep, audio, batch_windows=16)
    want = O.predict_track(cfg, params, audio, t_in, t_out)
    for s in cfg["source_names"]:
        assert got[s].shape == want[s].shape
        assert rel_l2(got[s], want[s]) <= OUT_TOL and rel_max(got[s], want[s]) <= OUT_TOL, (s, rel_l2(got[s], want[s]))


# ------------------------------------------------------------------------------------------------
# C / D: two training steps with Adam and inference on the device (the problem of tests/hostsim/run_cpu_step.py)
# ------------------------------------------------------------------------------------------------
def device_steps(cfg, batch, nf, grad_scale=1.0):
    """Two training steps with TF-form Adam and the inference calls on the GPU, each against the oracle at the parameters the
    engine holds, in the result form of tests/hostsim/run_cpu_step.py; plus "grads1" (the first step's flat gradient) and
    "repro1" (the first step run twice from the same state gives the same bits)."""
    from Models.UnetAudioSeparator import UnetAudioSeparator
    t_in, t_out = O.get_padding(cfg, nf)
    params = O.init_params(cfg, seed=11)
    rng = np.random.default_rng(12)
    for k in params:
        if k.endswith("/bias") or "interp" in k:
            params[k] = rng.uniform(-0.3, 0.3, size=params[k].shape).astype(np.float32)
    mix, targets = O.synthetic_batch(cfg, batch, t_in, t_out, seed=13)
    names = list(cfg["source_names"])
    Kn, C = len(names), O.num_channels(cfg)
    sep = UnetAudioSeparator(cfg)
    sep.load_variables(params, input_frames=t_in)
    mix_d = torch.from_numpy(mix).cuda()
    tg = sep.stack_targets({k: torch.from_numpy(v).cuda() for k, v in targets.items()})
    out = torch.empty((Kn, batch, t_out, C), device="cuda")
    res = {}
    for step in (1, 2):
        o_par = OrderedDict((n, v.cpu().numpy().copy()) for n, v in sep.variables().items())
        loss = float(sep.loss_and_gradients(mix_d, tg, grad_scale=grad_scale, outputs=out).item())
        g = sep.grads.clone()
        if step == 1:
            res["grads1"] = g.cpu().numpy().copy()
            sep.loss_and_gradients(mix_d, tg, grad_scale=grad_scale)
            res["repro1"] = bool(torch.equal(sep.grads.view(torch.int32), g.view(torch.int32))) and \
                float(sep._loss.item()) == loss
            sep.grads.copy_(g)
        loss_o, outs_o, _ = O.forward_backward(cfg, o_par, mix, targets)
        tp = O._as_torch(o_par, torch.float64, True)
        outs64 = O.forward(cfg, tp, torch.as_tensor(mix).to(torch.float64), True)
        l64 = O.mse_loss(cfg, outs64, {k: torch.as_tensor(v).to(torch.float64) for k, v in targets.items()})
        grads_o = {k: gg.numpy() for k, gg in zip(tp, torch.autograd.grad(l64, list(tp.values())))}
        got = {n: v.cpu().numpy().copy() / np.float32(grad_scale) for n, v in sep.gradients().items()}
        per = {n: rel_l2(got[n], grads_o[n]) for n in got}
        which = max(per, key=per.get)
        explained = None
        if per[which] >= GPU_BARS["grad_tol"]:
            flips, w_after = O.explain_gradient_mismatch(cfg, o_par, mix, targets, got, tol=GPU_BARS["grad_tol"])
            explained = {"flips": None if flips is None else len(flips), "worst_after": float(w_after)}
        o = out.cpu().numpy()
        res["step%d" % step] = {"loss_rel": abs(loss - loss_o) / abs(loss_o), "grad_worst_rel": per[which], "grad_worst_tensor": which,
                                "grad_explained": explained, "outputs_rel": max(rel_l2(o[k], outs_o[s]) for k, s in enumerate(names))}
        p_prev, g_now = sep.params.cpu().numpy().copy(), sep.grads.cpu().numpy().copy()
        m_prev, v_prev = sep.adam_m.cpu().numpy().copy(), sep.adam_v.cpu().numpy().copy()
        sep.adam_step(1e-3)
        p_want, m_want, v_want = O.adam_update(p_prev, g_now, m_prev, v_prev, step, 1e-3)
        res["step%d" % step]["params_rel"] = rel_l2(sep.params.cpu().numpy(), p_want)
        res["step%d" % step]["adam_slots_rel"] = max(rel_l2(sep.adam_m.cpu().numpy(), m_want), rel_l2(sep.adam_v.cpu().numpy(), v_want))
    res["adam_state"] = [float(x) for x in sep._adam_state.cpu()]
    o_par = OrderedDict((n, v.cpu().numpy().copy()) for n, v in sep.variables().items())
    for training, key in ((False, "infer_outputs_rel"), (True, "train_mode_outputs_rel")):
        got_o = sep.get_output(mix_d, training, False, reuse=True)
        want = O.forward_np(cfg, o_par, mix, training)
        res[key] = max(rel_l2(got_o[s].cpu().numpy(), want[s]) for s in names)
    # the window gather / scatter of predict_track (the last window shifted back, plain overwrite)
    eng = sep.engine(input_frames=t_in)
    n_frames = 3 * t_out - 7
    starts = [n_frames - t_out if pos + t_out > n_frames else pos for pos in range(0, n_frames, t_out)]
    padded = torch.from_numpy(rng.standard_normal((n_frames + (t_in - t_out), C)).astype(np.float32)).cuda()
    st = torch.tensor(starts, dtype=torch.int64, device="cuda")
    win = torch.empty((len(starts), t_in, C), device="cuda")
    eng.gather_windows(padded, st, win)
    res["gather_exact"] = bool(torch.equal(win, torch.stack([padded[s0:s0 + t_in] for s0 in starts])))
    outs = torch.randn((Kn, len(starts), t_out, C), device="cuda")
    preds = torch.empty((Kn, n_frames, C), device="cuda")
    eng.scatter_windows(outs, st, preds)
    want_p = torch.zeros_like(preds)
    for w, s0 in enumerate(starts):
        want_p[:, s0:s0 + t_out] = outs[:, w]
    res["scatter_exact"] = bool(torch.equal(preds, want_p))
    torch.cuda.synchronize()
    return res


def feasibility(cfg, nf):
    """None for a feasible draw, else the outcome the CPU test demands of it: infeasible shapes are refused by oracle and engine
    with AssertionError; where get_padding's formula and the graph disagree (a reference quirk) the engine follows the graph."""
    try:
        t_in, t_out = O.get_padding(cfg, nf)
        probe = O.forward_np(cfg, O.init_params(cfg, seed=1), np.zeros((1, t_in, O.num_channels(cfg)), np.float32), False)
    except AssertionError:
        wcfg = wun.config_from_model_config(cfg)
        with pytest.raises(AssertionError):
            e_in, _ = wun.get_padding(wcfg, nf)
            wun.Engine(wcfg, input_frames=e_in)
        return "infeasible"
    real_out = int(next(iter(probe.values())).shape[1])
    if real_out != t_out:
        eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
        assert eng.T_out == real_out != t_out, (eng.T_out, real_out, t_out)
        return "formula quirk"
    return None


@pytest.mark.gpu
@pytest.mark.parametrize("label,named,ov,batch,nf,env,grad_scale", DRAWS, ids=[d[0] for d in DRAWS])
def test_random_configuration_on_the_device(label, named, ov, batch, nf, env, grad_scale, monkeypatch):
    """The seeded sweep of tests/test_cpu_device.py (the same 16 draws) on the GPU: two training steps with Adam and inference
    against the oracle, and every launch of the draw replayed against float64."""
    set_env(monkeypatch, {})
    cfg = model_config(named, ov)
    outcome = feasibility(cfg, nf)
    if outcome is not None:
        print("%s: %s, handled as the CPU test handles it" % (label, outcome))
        return
    res = device_steps(cfg, batch, nf, grad_scale)
    try:
        assert_steps_match_oracle(res, **GPU_BARS)
    except AssertionError as ex:
        raise AssertionError("%s %r batch %d frames %d: %s" % (label, ov, batch, nf, ex))
    replay_all(label, named, ov, batch, nf)


def _switch_nets():
    return [("m6_L3_learned_forced", ["full_multi_instrument"], dict(num_layers=3, upsampling="learned"), 2, 200, FORCED),
            ("m4_like_L5", ["baseline_stereo"], dict(num_layers=5), 3, 200, {})]


# switch positions that run the default path's kernels in the default order: the step must be the default's bit for bit
SAME_KERNELS = ({"WUN_OUT_FUSE": "2"}, {"WUN_OUT_FUSE": "0"}, {"WUN_SIDE_STREAM": "0"})
# switch positions that add across CTAs with float atomics (DESIGN.md section 8 item 4): not bit-reproducible
ATOMIC = ({"WUN_BULK_WGRAD": "0"}, {"WUN_SPLIT_COLSUM": "0"}, {"WUN_FIRST_LAYER": "0"}, {"WUN_DISABLE_UMMA": "1"})
_DEFAULT = {}


@pytest.mark.gpu
@pytest.mark.parametrize("net", [n[0] for n in _switch_nets()])
@pytest.mark.parametrize("sw", SWITCHES, ids=["+".join("%s=%s" % kv for kv in s.items()) for s in SWITCHES])
def test_every_switch_position_gives_the_same_step_on_the_device(net, sw, monkeypatch):
    """Each A/B switch position (DESIGN.md section 9) computes the step the default path computes: against the oracle with the bars
    of tests/test_cpu_device.py, against the default path's gradients to 1e-4 rel-L2, bit for bit where the same kernels run,
    and reproducible bit for bit wherever the path is free of float atomics."""
    _, named, ov, batch, nf, env = next(n for n in _switch_nets() if n[0] == net)
    if net not in _DEFAULT:
        set_env(monkeypatch, env)
        _DEFAULT[net] = device_steps(model_config(named, ov), batch, nf)
        assert_steps_match_oracle(_DEFAULT[net], **GPU_BARS)
        assert _DEFAULT[net]["repro1"], "two identical steps of the default path differ"
    set_env(monkeypatch, dict(env, **sw))
    res = device_steps(model_config(named, ov), batch, nf)
    assert_steps_match_oracle(res, **GPU_BARS)
    g, g0 = res["grads1"], _DEFAULT[net]["grads1"]
    assert rel_l2(g, g0) <= 1e-4, rel_l2(g, g0)
    if sw in SAME_KERNELS:
        assert np.array_equal(g.view(np.uint32), g0.view(np.uint32))
    if sw not in ATOMIC:
        assert res["repro1"], "two identical steps differ on an atomics-free path"


@pytest.mark.gpu
def test_zz_configuration_report():
    """Prints the peak device memory and time of each replayed configuration and the file's wall time so far."""
    print("\n%-34s %10s %8s" % ("configuration", "peak GB", "s"))
    for name, (gb, sec) in REPORT.items():
        print("%-34s %10.1f %8.0f" % (name, gb, sec))
    print("wall time of the file so far: %.0f s" % (time.time() - START))
    assert REPORT
