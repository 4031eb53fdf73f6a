"""The engine's REAL host code executed end to end on the CPU (no GPU): two training steps + an inference call, vs the oracle.

tests/hostsim/ builds the engine's sources a second time with `nvcc --cudart none` against a stand-in CUDA runtime.  In execute
mode that runtime carries every launch out on host memory with the reference routines of tests/hostsim/cpu_kernels.cpp - an
independent statement, in plain double-precision loops, of what each kernel must compute from its by-value parameter block.
What runs unmodified is everything the HOST does: the planner, the plane / class / group / term tables and packed-weight jobs
built for the tensor-core kernels (incl. pair-merged halves and output-channel splits), the
split-pass jobs that carry the bias sums, the first-layer / upsampling-backward / output-layer blocks, gradient scales,
accumulate ranges, memsets and the device-side Adam state.  Loss, every gradient, the source estimates and the parameters after
two TF-form Adam steps must agree with the oracle to rounding (1e-5 / 1e-4: the reference routines accumulate in double).

This is NOT a CPU path of the product (libwun.so has none and fails loudly without a GPU); it is test infrastructure that lets
the host half of the engine be checked for configurations and batch sizes no GPU test has run (e.g. the per-GPU batches of the
8-GPU M6 split).  The device half - the kernels' own arithmetic - is what `-m gpu` tests."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
import schedule  # noqa: E402


_SIM = None


@pytest.fixture(scope="module", autouse=True)
def _build_once():
    """Built when the first test of this module RUNS, not at collection (a `-m gpu` run collects this file but runs none of it)."""
    global _SIM
    try:
        _SIM = schedule.build()
    except Exception:                                        # noqa: BLE001 (tests/test_stream_schedule.py reports build failures)
        _SIM = None
    yield


@pytest.fixture(autouse=True)
def _need_simulation(_build_once):
    if _SIM is None:
        pytest.skip("host simulation of the engine not built (needs nvcc and g++)")


FORCED = {"WUN_PAIR_MIN_CTAS": "1", "WUN_PAIR_DGRAD": "1"}


def run_steps(named, overrides, batch, nf, env=None, grad_scale=1.0):
    e = dict(os.environ)
    for k in [k for k in e if k.startswith("WUN_")]:
        del e[k]
    e.update(env or {})
    e["WUN_LIB"] = _SIM
    e["OMP_NUM_THREADS"] = e["MKL_NUM_THREADS"] = "1"       # small nets; several of these run side by side
    out = subprocess.run([sys.executable, os.path.join(HERE, "hostsim", "run_cpu_step.py"), str(batch), str(nf), repr(float(grad_scale)),
                          json.dumps(overrides)] + list(named), env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert out.returncode == 0, out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def assert_matches_oracle(res):
    assert res["unknown"] == []
    assert res["footprint_miss"] == [], res["footprint_miss"][:3]     # (only populated under HOSTSIM_POISON=1, see below)
    for step in ("step1", "step2"):
        r = res[step]
        assert r["loss_rel"] < 1e-5, (step, r)
        ex = r.get("grad_explained")           # None, or the LeakyReLU-slope-flip proof for a gradient that is off (run_cpu_step.py)
        assert r["grad_worst_rel"] < 1e-4 or (ex and ex["flips"] is not None and ex["worst_after"] < 1e-4), (step, r)
        assert r["outputs_rel"] < 1e-5, (step, r)
        assert r["params_rel"] < 1e-5 and r["adam_slots_rel"] < 1e-4, (step, r)
    assert res["infer_outputs_rel"] < 1e-4, res["infer_outputs_rel"]
    assert res["train_mode_outputs_rel"] < 1e-4, res["train_mode_outputs_rel"]
    assert res["gather_exact"] and res["scatter_exact"]          # predict_track's window tiling (Evaluate.py:125-139)
    assert abs(res["adam_state"][0] - 0.9 ** 3) < 1e-6 and abs(res["adam_state"][1] - 0.999 ** 3) < 1e-6 and res["adam_state"][2] == 2.0


FAMILIES = [
    ("m4_like", ["baseline_stereo"], dict(num_layers=3), 2, 300),
    ("m5_like_learned", ["full"], dict(num_layers=3, num_initial_filters=16), 2, 260),
    ("m6_like_multi_instrument", ["full_multi_instrument"], dict(num_layers=3), 2, 200),
    ("m1_like_same_padding_mono", ["baseline"], dict(num_layers=3), 2, 256),
    ("same_learned_stereo_difference", ["baseline_diff"], dict(num_layers=3, upsampling="learned", mono_downmix=False), 2, 128),
]


def run_many(cases):
    """cases: [(label, named, overrides, batch, nf, env, grad_scale)] -> {label: result}; the subprocesses run side by side."""
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=min(6, os.cpu_count() or 2)) as pool:
        futs = {c[0]: pool.submit(run_steps, c[1], c[2], c[3], c[4], c[5], c[6]) for c in cases}
        return {k: f.result() for k, f in futs.items()}


@pytest.mark.parametrize("variant", ["planner_default", "gpu_filling_variants_forced"])
def test_two_training_steps_and_inference_on_the_cpu_device_match_the_oracle(variant):
    forced = variant.startswith("gpu")
    # HOSTSIM_POISON=1: the footprint "poison test" (tests/hostsim/fake_cudart.cpp) - before every launch all words outside its
    # DECODED footprint are overwritten with NaNs and restored afterwards; the step still has to match the oracle and no launch may
    # touch a word outside the footprint the racecheck (tests/test_stream_schedule.py) attributes to it
    env = dict(FORCED if forced else {}, HOSTSIM_POISON="1")
    results = run_many([(name, named, ov, batch, nf, env, 0.5 if forced else 1.0) for name, named, ov, batch, nf in FAMILIES])
    assert sorted(results) == sorted(c[0] for c in FAMILIES)
    for name, res in results.items():
        try:
            assert_matches_oracle(res)
            ks = res["kernels"]
            assert any(k.startswith("plane_conv_umma_kernel<") and k.endswith("false>") for k in ks), sorted(ks)   # forward
            assert any(k.startswith("plane_conv_umma_kernel<") and k.endswith("true>") for k in ks), sorted(ks)    # dgrad
            assert any(k.startswith("wgrad_umma_bulk_kernel<") for k in ks) and "umma_pack_kernel" in ks, sorted(ks)
            assert "output_fwd_kernel" in ks, sorted(ks)
        except AssertionError as ex:
            raise AssertionError("%s: %s" % (name, ex))


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


def test_every_structural_switch_gives_the_same_step():
    cases = []
    for sw in SWITCHES:
        env = dict(FORCED, HOSTSIM_POISON="1")
        env.update(sw)
        cases.append(("+".join("%s=%s" % kv for kv in sw.items()), ["full_multi_instrument"], dict(num_layers=3, upsampling="learned"), 2, 200, env, 1.0))
    for label, res in run_many(cases).items():
        try:
            assert_matches_oracle(res)
        except AssertionError as ex:
            raise AssertionError("%s: %s" % (label, ex))


def test_batch_sizes_of_the_data_parallel_splits():
    """The planner's choices depend on the batch (pair merging, splits, folded tiles): the per-GPU batches the scaling runs use."""
    cases = [("batch %d" % b, ["full_multi_instrument"], dict(num_layers=4), b, 260, None, 1.0 / 8) for b in (1, 3, 4, 8)]
    for label, res in run_many(cases).items():
        try:
            assert_matches_oracle(res)
        except AssertionError as ex:
            raise AssertionError("%s: %s" % (label, ex))


def test_wider_output_filter_and_other_filter_sizes():
    """output_filter_size > 1 (no fused epilogue: the separate output kernels with 'same' / 'valid' taps), other filter widths."""
    cases = [("same padding, ofs 3", ["baseline"], dict(num_layers=3, output_filter_size=3, filter_size=9, merge_filter_size=3), 2, 256, FORCED, 1.0),
             ("context, ofs 5", ["baseline_stereo"], dict(num_layers=2, output_filter_size=5, filter_size=7, input_filter_size=7), 1, 300, None, 1.0)]
    for label, res in run_many(cases).items():
        try:
            assert_matches_oracle(res)
        except AssertionError as ex:
            raise AssertionError("%s: %s" % (label, ex))


def test_arithmetic_model_of_the_three_mma_scheme_meets_the_parity_bar_and_a_single_bf16_pass_does_not():
    """DESIGN.md 4.1: every fp32 operand is split into two bf16 (hi, lo) and a product is three bf16 MMAs (hi*hi + hi*lo + lo*hi,
    fp32 accumulation).  With the reference routines of the tensor-core launches switched to that arithmetic
    (FAKECUDA_MMA_MODEL=3) the step stays two orders of magnitude inside the 1e-4 parity bar of BASELINE.json - the same ~5e-6 the
    GPU measures - while a single bf16 pass (=1) misses it by a factor of 40: why the kernels issue three MMAs per product."""
    case = (["baseline_stereo"], dict(num_layers=4), 2, 600)
    res = run_many([("exact", *case, FORCED, 1.0), ("three_mma", *case, dict(FORCED, FAKECUDA_MMA_MODEL="3"), 1.0),
                    ("one_mma", *case, dict(FORCED, FAKECUDA_MMA_MODEL="1"), 1.0)])
    exact, three, one = (res[k]["step1"] for k in ("exact", "three_mma", "one_mma"))
    assert exact["outputs_rel"] < 1e-6 and exact["grad_worst_rel"] < 1e-5
    assert 1e-6 < three["outputs_rel"] < 3e-5 and three["grad_worst_rel"] < 1e-4 and three["loss_rel"] < 1e-5
    assert one["outputs_rel"] > 1e-3 and one["grad_worst_rel"] > 1e-3


def test_sharded_gradients_sum_to_the_single_device_gradient(tmp_path):
    """The data-parallel invariant (SURVEY section 4 item 6, Training.py:62: the loss is a mean over the batch) at the level of the
    engine's real host code: two ranks with half the batch each and grad_scale = local / global produce gradients whose SUM (what
    the all-reduce computes) is the gradient one device computes for the whole batch."""
    import numpy as np
    case = (["full_multi_instrument"], dict(num_layers=3, upsampling="learned"), 4, 260)
    files = {k: str(tmp_path / (k + ".npy")) for k in ("all", "r0", "r1")}
    res = run_many([("all", *case, dict(FORCED, HOSTSIM_DUMP_GRADS=files["all"]), 1.0),
                    ("r0", *case, dict(FORCED, HOSTSIM_DUMP_GRADS=files["r0"], HOSTSIM_SHARD="0:2"), 0.5),
                    ("r1", *case, dict(FORCED, HOSTSIM_DUMP_GRADS=files["r1"], HOSTSIM_SHARD="2:4"), 0.5)])
    for r in res.values():
        assert r["step1"]["grad_worst_rel"] < 1e-4 and r["unknown"] == []
    g = {k: np.load(f).astype(np.float64) for k, f in files.items()}
    err = np.linalg.norm(g["r0"] + g["r1"] - g["all"]) / np.linalg.norm(g["all"])
    assert err < 1e-6, err
    assert np.linalg.norm(g["r0"] - g["r1"]) / np.linalg.norm(g["all"]) > 1e-2          # the shards do differ


def test_predict_track_pipeline_through_the_c_abi_matches_the_oracle():
    """Evaluate.py:82-145 end to end on the CPU device: context padding, window gather (the last window shifted back), ONE batched
    test-time forward over all windows, scatter with overwrite - vs the oracle's window-by-window loop; stereo context model and
    mono 'same'-padding model."""
    res = run_many([("context_stereo", ["baseline_stereo"], dict(num_layers=3), 1, 300, dict(FORCED, HOSTSIM_PREDICT="1"), 1.0),
                    ("same_mono_learned", ["baseline"], dict(num_layers=3, upsampling="learned"), 1, 256, dict(HOSTSIM_PREDICT="1"), 1.0)])
    for label, r in res.items():
        assert r["predict_windows"] == 3 and r["predict_rel"] < 1e-4, (label, r["predict_rel"])


def random_model_configs(n, seed):
    """n reproducible draws from the space of shapes the reference allows (Config.py:9-39 keys the separator reads)."""
    import numpy as np
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


def test_random_model_configurations_on_the_cpu_device():
    """A seeded sweep over the configuration space (layers, filter widths incl. even ones, channel counts that are not multiples
    of 8, both paddings, both upsamplers, both output types / activations, mono / stereo, 2 / 4 sources, batch 1-3): whatever
    mix of tensor-core and CUDA-core launches the planner picks, the step must match the oracle; shapes the reference's asserts
    reject (UnetAudioSeparator.py:55, :121, Utils.py:114-117) must be rejected by the engine with the same exception type."""
    cases = random_model_configs(16, seed=2026)
    results = run_many(cases)
    feasible = 0
    for label, named, ov, batch, nf, _, _ in cases:
        res = results[label]
        if res.get("infeasible"):
            assert res["engine_error"] is not None and res["engine_error"].startswith("AssertionError"), (label, ov, nf, res)
            continue
        if res.get("formula_quirk"):          # get_padding's formula vs the graph (reference quirk): the plan follows the graph
            assert res["engine_t_out"] == res["graph_t_out"] != res["formula_t_out"], (label, ov, nf, res)
            continue
        feasible += 1
        try:
            assert_matches_oracle(res)
        except AssertionError as ex:
            raise AssertionError("%s %r batch %d frames %d: %s" % (label, ov, batch, nf, ex))
    assert feasible >= 10, feasible


def test_shapes_the_reference_asserts_against_are_refused_with_the_same_exception():
    """'same' padding with a length that does not halve cleanly through every level (UnetAudioSeparator.py:121 asserts the skip and
    the upsampled tensor have equal length): the oracle raises AssertionError, and so must the engine's planner (WUN_E_SHAPE)."""
    res = run_many([("odd_length", ["baseline"], dict(num_layers=3), 1, 65, None, 1.0),
                    ("not_divisible", ["baseline_diff"], dict(num_layers=4, upsampling="learned"), 2, 72, None, 1.0)])
    for label, r in res.items():
        assert r.get("infeasible") and (r["engine_error"] or "").startswith("AssertionError"), (label, r)


def test_one_handle_at_two_batch_sizes():
    """After two steps at batch b: a step at b - 1 on its own workspace and one at b again - loss and gradients vs float64
    autograd through the oracle (the planner's batch-dependent choices must not leak between calls)."""
    res = run_many([("forced", ["full_multi_instrument"], dict(num_layers=3, upsampling="learned"), 3, 200, dict(FORCED, HOSTSIM_OTHER_BATCH="1"), 1.0),
                    ("default", ["baseline_stereo"], dict(num_layers=4), 2, 400, dict(HOSTSIM_OTHER_BATCH="1"), 1.0)])
    for label, r in res.items():
        assert_matches_oracle(r)
        assert r["other_batch_worst_rel"] < 1e-4, (label, r["other_batch_worst_rel"])
