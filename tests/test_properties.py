"""Property tests (hypothesis) of the host-side pieces: shape algebra of the C planner vs the oracle for arbitrary
hyper-parameters, plan invariants, and the checkpoint container for arbitrary tensor sets.  CPU only."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import Config
import TFCheckpoint as tfc
import wun
from oracle import wave_unet_oracle as O

odd = lambda lo, hi: st.integers(lo // 2, hi // 2).map(lambda v: 2 * v + 1)


@settings(max_examples=120, deadline=None, suppress_health_check=[HealthCheck.too_slow])
@given(L=st.integers(1, 9), fs=odd(3, 15), mfs=odd(1, 7), ifs=odd(3, 15), ofs=odd(1, 5), nf=st.integers(1, 40000))
def test_get_padding_equals_oracle_for_any_hyperparameters(L, fs, mfs, ifs, ofs, nf):
    mc = Config.build_config(["baseline_stereo"], dict(num_layers=L, filter_size=fs, merge_filter_size=mfs,
                                                       input_filter_size=ifs, output_filter_size=ofs), experiment_id=0)["model_config"]
    try:
        want = O.get_padding(mc, nf)
    except AssertionError:
        with pytest.raises(AssertionError):                   # infeasible shapes fail on both sides as the reference does (assert, :55)
            wun.get_padding(wun.config_from_model_config(mc), nf)
        return
    assert wun.get_padding(wun.config_from_model_config(mc), nf) == want
    t_in, t_out = want
    # (input_filter_size only exists in the reference's get_padding, :69-73 - get_output convolves every down block with
    #  filter_size, :98 - so the formula and the graph agree only for ifs == fs, which holds in every preset)
    if ifs == fs:
        if t_out <= 0:                                          # the reference's formula has no guard here (:76); building fails loudly
            with pytest.raises(AssertionError):
                wun.Engine(wun.config_from_model_config(mc), num_frames=nf)
            return
        eng = wun.Engine(wun.config_from_model_config(mc), num_frames=nf)
        assert (eng.T_in, eng.T_out) == (t_in, t_out)           # the planner's walk over the graph lands on the same lengths
    if t_out <= 0:
        return
    assert t_in > t_out
    if ofs == 1:
        assert t_out >= nf                                      # rounded UP to the next feasible length (the reference's
                                                                # formula can come out shorter when output_filter_size > 1)


@settings(max_examples=25, deadline=None, suppress_health_check=[HealthCheck.too_slow])
@given(L=st.integers(1, 6), f0=st.sampled_from([8, 16, 24, 40]), nf=st.integers(16, 3000), learned=st.booleans(),
       context=st.booleans(), batch=st.sampled_from([1, 3, 16]))
def test_plan_invariants_for_arbitrary_small_networks(L, f0, nf, learned, context, batch):
    ov = dict(num_layers=L, num_initial_filters=f0, upsampling="learned" if learned else "linear", context=context)
    if not context:
        nf = max(1, nf >> L) << L                               # same-padding nets need lengths divisible by 2^L
    mc = Config.build_config(["baseline_stereo"], ov, experiment_id=0)["model_config"]
    cfg = wun.config_from_model_config(mc)
    try:
        t_in, t_out = O.get_padding(mc, nf)
    except AssertionError:
        return
    eng = wun.Engine(cfg, num_frames=nf)
    assert (eng.T_in, eng.T_out) == (t_in, t_out)
    table = O.param_table(mc)
    assert [(n, tuple(s)) for n, s, _, _ in eng.param_table] == [(n, tuple(s)) for n, s in table]
    offs = [o for _, _, o, _ in eng.param_table]
    assert offs == sorted(offs) and eng.param_numel == sum(c for _, _, _, c in eng.param_table)
    assert eng.workspace_bytes(batch, True) >= eng.workspace_bytes(batch, False) > 0
    assert eng.forward_backward_flops(batch) <= 3.0 * eng.forward_flops(batch) + 1
    for d in eng.plan_audit(batch):                             # whatever runs on tensor cores respects the hardware limits
        assert d["smem"] <= 200 * 1024


names = st.text(alphabet=st.characters(min_codepoint=33, max_codepoint=126), min_size=1, max_size=40)
dtypes = st.sampled_from([np.float32, np.float64, np.int32, np.int64, np.uint8, np.float16, np.bool_])
shapes = st.lists(st.integers(0, 7), min_size=0, max_size=4)


@settings(max_examples=40, deadline=None, suppress_health_check=[HealthCheck.too_slow, HealthCheck.function_scoped_fixture])
@given(spec=st.dictionaries(names, st.tuples(dtypes, shapes), min_size=1, max_size=40), block=st.sampled_from([48, 200, 4096, tfc.BLOCK_SIZE]),
       seed=st.integers(0, 2 ** 31 - 1))
def test_checkpoint_round_trip_for_arbitrary_tensor_sets(tmp_path_factory, spec, block, seed):
    rng = np.random.default_rng(seed)
    tensors = {}
    for n, (dt, shp) in spec.items():
        a = rng.integers(0, 2, size=shp) if dt is np.bool_ else rng.integers(-100, 100, size=shp)
        tensors[n] = np.asarray(a).astype(dt)
    prefix = str(tmp_path_factory.mktemp("ck") / "model-1")
    tfc.write_checkpoint(prefix, tensors, block_size=block)
    got = tfc.read_checkpoint(prefix)
    assert list(got) == sorted(tensors, key=lambda s: s.encode("utf-8"))
    for n, a in tensors.items():
        assert got[n].dtype == a.dtype and got[n].shape == a.shape and np.array_equal(got[n], a)
    assert [(n, s) for n, _, s in tfc.list_variables(prefix)] == [(n, tensors[n].shape) for n in got]
