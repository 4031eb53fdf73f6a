"""Racecheck of the engine's multi-stream schedule on the host (no GPU).

The engine's REAL host code (csrc/engine.cu: launch sequencing, the weight-pack / weight-gradient / split-pass / helper streams,
every event fork and join, the gradient-bucket events of the data-parallel overlap) is built a second time with
`nvcc --cudart none` against a recording stand-in for the CUDA runtime (tests/hostsim/fake_cudart.cpp) and run for two
consecutive training steps with made-up device addresses.  Every launch is decoded from its by-value parameter block into the
exact words it reads, writes or atomically accumulates into; tests/hostsim/schedule.py replays the trace with vector clocks over
streams and events and a shadow memory at 4-byte granularity.  Any pair of conflicting accesses that the events do not order is
a race the GPU parity tests could only catch by luck.

Covered: the planner's default choices and the GPU-filling kernel variants forced onto mid-size nets (pair-merged classes) for
the five model families, every A/B switch of the stream structure in its other
position, inference, the bucketed all-reduce on a communication stream (wun/parallel.py) followed by Adam and the NEXT step's
weight packs - and the checker itself: dropping any single necessary stream wait from a trace must be reported."""
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
import schedule  # noqa: E402



_SIM, _WHY = None, "not built yet"


@pytest.fixture(scope="module", autouse=True)
def _build_once():
    """Built when the first test of this module RUNS, not at collection (a `-m gpu` run collects this file but runs none of it)."""
    global _SIM, _WHY
    try:
        _SIM, _WHY = schedule.build(), ""
    except Exception as ex:                                  # noqa: BLE001 - a broken tool chain must not take the suite down
        _SIM, _WHY = None, "%s: %s" % (type(ex).__name__, str(ex)[:200])
    yield


@pytest.fixture(autouse=True)
def _need_simulation(request, _build_once):
    if _SIM is None and "simulation_library_builds" not in request.node.name:
        pytest.skip("host simulation of the engine not built (needs nvcc and g++) " + _WHY)


def test_the_simulation_library_builds_where_the_tool_chain_exists():
    """(Not skipped with the rest: with nvcc and g++ present a build failure is a failure, not a reason to skip the racecheck.)"""
    if not (os.path.exists(schedule.NVCC) and __import__("shutil").which("g++")):
        pytest.skip("no nvcc / g++ here")
    assert _SIM is not None and os.path.exists(_SIM), _WHY


FORCED = {"WUN_PAIR_MIN_CTAS": "1", "WUN_PAIR_DGRAD": "1"}      # as tests/test_gpu_parity.py
FAMILIES = [
    ("m4_like_L5", ["baseline_stereo"], dict(num_layers=5), 3, 2000),
    ("m5_like_L4", ["full"], dict(num_layers=4, num_initial_filters=16), 2, 1500),
    ("m6_like_L4", ["full_multi_instrument"], dict(num_layers=4), 2, 1200),
    ("m1_like_L5", ["baseline"], dict(num_layers=5), 3, 4096),
    ("same_learned_stereo", ["baseline_diff"], dict(num_layers=4, upsampling="learned", mono_downmix=False), 2, 2048),
]


def kernels(ops):
    return {o[2].split("(")[0].replace("void_", "").replace("wun::", "") for o in ops if o[0] == "L"}


def assert_race_free(meta, ops):
    violations, stats = schedule.check(meta, ops)
    assert not violations, "\n".join("%(name)s [%(mode)s %(region)s, %(words)d words] is not ordered after %(other_name)s" % v
                                     for v in violations)
    return stats


@pytest.mark.parametrize("name,named,ov,batch,nf", FAMILIES, ids=[c[0] for c in FAMILIES])
def test_forced_gpu_filling_variants_are_race_free_incl_bucketed_allreduce(name, named, ov, batch, nf):
    meta, ops = schedule.trace("train_dp", named, ov, batch, nf, FORCED)
    stats = assert_race_free(meta, ops)
    ks = kernels(ops)
    assert any(k.startswith("plane_conv_umma_kernel<") and k.endswith("true>") for k in ks), sorted(ks)
    assert any(k.startswith("wgrad_umma_bulk_kernel<") for k in ks), sorted(ks)
    assert {"split_views_kernel", "umma_pack_kernel", "upsample_bwd_kernel", "output_fwd_kernel"} <= ks
    assert len(stats["per_stream"]) == 5 and min(stats["per_stream"]) > 0      # caller, packs + wgrad, split passes, helper, comm
    assert stats["joined_into_caller"]          # every forked stream is joined back: the step is capturable as one CUDA graph
    # the launch count the library reports (bench.py's gpu_launches) is what was launched: 2 steps of (step + 2 memsets + 2 Adam)
    lib_launches = sum(1 for o in ops if o[0] == "L" and not o[2].startswith("nccl"))
    assert lib_launches == 2 * (meta["launches_reported"] + 4)


@pytest.mark.parametrize("name,named,ov,batch,nf", FAMILIES[:3], ids=[c[0] for c in FAMILIES[:3]])
def test_default_planner_choices_are_race_free(name, named, ov, batch, nf):
    meta, ops = schedule.trace("train_dp", named, ov, batch, nf)
    assert_race_free(meta, ops)
    assert any(k.startswith("plane_conv_umma_kernel<") for k in kernels(ops))


SWITCHES = ["WUN_SPLIT_AHEAD=0", "WUN_SIDE_STREAM=0", "WUN_DGRAD_PAR=0", "WUN_FIRST_TAIL=0", "WUN_BULK_WGRAD=0", "WUN_PACK_EVENTS=0",
            "WUN_OUT_FUSE=0", "WUN_OUT_FUSE=2", "WUN_FIRST_LAYER=0", "WUN_SPLIT_COLSUM=0", "WUN_DISABLE_UMMA=1", "WUN_UMMA_WGRAD=0"]


@pytest.mark.parametrize("switch", SWITCHES)
def test_every_switch_of_the_stream_structure_in_its_other_position(switch):
    env = dict(FORCED)
    k, v = switch.split("=")
    env[k] = v
    meta, ops = schedule.trace("train", ["baseline_stereo"], dict(num_layers=4), 2, 1500, env)
    assert_race_free(meta, ops)


def test_inference_and_training_with_estimates_share_a_handle_without_races():
    for scenario in ("infer", "train_out"):
        meta, ops = schedule.trace(scenario, ["full"], dict(num_layers=4, num_initial_filters=16), 2, 1500, FORCED)
        assert assert_race_free(meta, ops)["joined_into_caller"]


def test_training_alternating_with_validation_at_another_batch_size():
    """Training.optimise (Training.py:123-150) on one handle: the workspaces differ, the internal streams and events do not."""
    meta, ops = schedule.trace("train_validate", ["baseline_stereo"], dict(num_layers=4), 2, 1500, FORCED)
    assert assert_race_free(meta, ops)["joined_into_caller"]
    meta, ops = schedule.trace("train_validate", ["full"], dict(num_layers=3, num_initial_filters=16), 3, 500)
    assert assert_race_free(meta, ops)["joined_into_caller"]


def test_training_steps_at_two_batch_sizes_on_one_handle():
    """The last batch of an epoch has another size: other planner choices, other arena layouts, the same streams and events."""
    for named, ov, batch, nf, env in ((["baseline_stereo"], dict(num_layers=4), 2, 1500, FORCED), (["full_multi_instrument"], dict(num_layers=3), 3, 300, None)):
        meta, ops = schedule.trace("train_two_batches", named, ov, batch, nf, env)
        assert assert_race_free(meta, ops)["joined_into_caller"]


def test_an_unjoined_stream_is_noticed():
    """Drop the last wait of the caller's stream (the join of the weight-gradient stream): the trace no longer ends joined."""
    meta, ops = schedule.trace("train", ["baseline_stereo"], dict(num_layers=3), 1, 300, FORCED)
    assert schedule.check(meta, ops)[1]["joined_into_caller"]
    last_adam = max(i for i, o in enumerate(ops) if o[0] == "L" and "adam_kernel" in o[2])
    main_waits = [i for i, o in enumerate(ops) if o[0] == "S" and o[1] == meta["main"] and i < last_adam]
    cut = [o for i, o in enumerate(ops) if i < last_adam and i not in main_waits[-3:]]
    assert not schedule.check(meta, cut, init_regions=())[1]["joined_into_caller"]


def test_the_checker_reports_every_necessary_wait_when_it_is_dropped():
    """Teeth: remove one cudaStreamWaitEvent at a time from a race-free trace.  Most waits are the only ordering between two
    conflicting launches - the checker must name that pair; the rest are implied by other event chains.  The named pairs must
    include each kind of cross-stream dependency the engine has."""
    meta, ops = schedule.trace("train_dp", ["baseline_stereo"], dict(num_layers=3), 1, 300, FORCED)
    assert_race_free(meta, ops)
    waits = [i for i, o in enumerate(ops) if o[0] == "S"]
    pairs = set()
    necessary = 0
    for i in waits:
        v, _ = schedule.check(meta, ops[:i] + ops[i + 1:], max_reports=1)
        if v:
            necessary += 1
            short = lambda n: str(n).split("(")[0].replace("void_", "").replace("wun::", "").split("<")[0]      # noqa: E731
            pairs.add((short(v[0]["name"]), short(v[0]["other_name"])))
    assert necessary >= 0.6 * len(waits), (necessary, len(waits))
    expected = {
        ("wgrad_umma_bulk_kernel", "split_views_kernel"),          # a wgrad kernel reads the split arrays of its layer
        ("split_views_kernel", "wgrad_umma_bulk_kernel"),          # the arena half is rewritten two layers later
        ("umma_pack_kernel", "adam_kernel"),                       # the next step's packs read the updated parameters
        ("adam_kernel", "nccl_all_reduce_bucket3"),                # Adam after the last bucket's all-reduce
    }
    assert expected <= pairs, sorted(pairs)
    assert any(a.startswith("plane_conv_umma") and b == "umma_pack_kernel" for a, b in pairs)          # a conv waits for its own pack
    assert any(a.startswith("nccl_all_reduce") and b in ("wgrad_umma_bulk_kernel", "split_views_kernel", "first_wgrad_kernel",
                                                         "output_wgrad_kernel", "upsample_bwd_kernel", "memset") for a, b in pairs)
    assert any(a == "split_views_kernel" and (b.startswith("plane_conv_umma") or b == "upsample_bwd_kernel") for a, b in pairs)


def test_steady_state_steps_create_no_streams_or_events():
    """include/wun.h: "no hidden synchronisation, allocation or host<->device copy inside forward / backward / adam".  The
    internal streams and events are created by the first call (before a CUDA graph of the step would be captured); the second
    step of a trace must consist of launches, event records and stream waits only - and issue exactly what the first one did."""
    meta, ops = schedule.trace("train", ["baseline_stereo"], dict(num_layers=4), 2, 1500, FORCED)
    adam = [i for i, o in enumerate(ops) if o[0] == "L" and "adam_advance_kernel" in o[2]]
    assert len(adam) == 2
    first, second = ops[:adam[0] + 1], ops[adam[0] + 1:]
    assert any(o[0] == "C" for o in first) and any(o[0] == "N" for o in first)
    assert not any(o[0] in ("C", "N") for o in second)
    shape = lambda part: [(o[0], o[2].split("(")[0]) if o[0] == "L" else (o[0],) for o in part if o[0] in ("L", "E", "S")]      # noqa: E731
    assert shape(first) == shape(second)


BENCHMARK_SIZES = [("baseline_stereo", 16, "train"), ("full", 16, "train"), ("full_multi_instrument", 32, "train"),
                   ("full_multi_instrument", 4, "train"), ("baseline", 16, "train"), ("full_44KHz", 16, "infer")]


@pytest.mark.parametrize("preset,batch,scenario", BENCHMARK_SIZES, ids=["%s_b%d" % (p, b) for p, b, _ in BENCHMARK_SIZES])
def test_launch_geometry_at_the_benchmark_sizes_respects_the_hardware_limits(preset, batch, scenario):
    """The grid, block, dynamic shared memory and cluster width the engine REALLY passes to the runtime for every launch of the
    configurations bench.py times (full windows; trace only, no shadow memory): within the sm_90 limits, and every launch above
    the 48 KB default opted in to its shared memory with cudaFuncSetAttribute first."""
    import Config
    cfg = Config.build_config([preset], experiment_id=0)["model_config"]
    meta, ops = schedule.trace(scenario, [preset], {}, batch, cfg["num_frames"])
    assert schedule.launch_limit_violations(ops) == []
    geos = [o[4] for o in ops if o[0] == "L" and o[4] is not None]
    convs = [o[4] for o in ops if o[0] == "L" and "plane_conv_umma_kernel" in o[2]]
    assert convs and all(g[3] == 256 and 2 * (g[6] + 1024) <= 228 * 1024 for g in convs), convs[:3]   # two CTAs per SM
    if scenario == "train":                                          # the wgrad stages use most of the 227 KB
        assert max(o[4][6] for o in ops if o[0] == "L" and "wgrad_umma_bulk_kernel" in o[2]) > 100 * 1024


def test_the_limit_check_notices_an_oversized_launch():
    meta, ops = schedule.trace("infer", ["baseline_stereo"], dict(num_layers=3), 1, 300)
    i = next(k for k, o in enumerate(ops) if o[0] == "L" and o[4] is not None and o[4][6] > 49152)
    g = list(ops[i][4])
    broken = list(ops)
    g[7] = 49152                                                     # as if the cudaFuncSetAttribute call had been forgotten
    broken[i] = ops[i][:4] + (tuple(g),)
    assert len(schedule.launch_limit_violations(broken)) == 1 and schedule.launch_limit_violations(ops) == []


def test_random_model_configurations_are_race_free_and_within_the_launch_limits():
    """A seeded sweep over the configuration space (the draws of tests/test_cpu_device.py: layer counts, filter widths, channel
    counts that fall back to the CUDA-core kernels, both paddings / upsamplers / output types, batch 1-3) with the bucketed
    all-reduce: whatever mix of launches and streams the planner produces, no race, no out-of-bounds or uninitialised access,
    every stream joined, every launch within the hardware limits.  (One-off campaigns: 96 draws, none bad.)"""
    from test_cpu_device import random_model_configs
    for i, (label, named, ov, batch, nf, _, _) in enumerate(random_model_configs(6, seed=77)):
        meta, ops = schedule.trace("train_dp", named, ov, batch, nf, FORCED if i % 2 else None)
        stats = assert_race_free(meta, ops)
        assert stats["joined_into_caller"] and schedule.launch_limit_violations(ops) == [], (label, ov)
