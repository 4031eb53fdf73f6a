"""CPU tests of the host side: Config shim, C-ABI symbols, shape solver, parameter table, plan FLOPs.
No compute entry point is exercised (no GPU needed); they must fail loudly without one."""
import ctypes
import json
import os
import re

import numpy as np
import pytest

import Config
import wun
from Models.UnetAudioSeparator import UnetAudioSeparator
from oracle import wave_unet_oracle as O

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")


def mc(named=(), **kw):
    return Config.build_config(list(named), kw, experiment_id=0)["model_config"]


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(REPO, "include", "wun.h")).read()
    declared = set(re.findall(r"\b(wun_[a-z0-9_]+)\s*\(", header))
    assert declared == set(wun.SYMBOLS), declared ^ set(wun.SYMBOLS)
    lib = ctypes.CDLL(wun.LIB_PATH)
    for s in declared:
        assert hasattr(lib, s), s
    assert b"sm_90a" in wun.lib.wun_version()


def test_config_presets_and_cli():
    c = mc(["baseline_stereo"])
    assert (c["output_type"], c["context"], c["mono_downmix"], c["num_channels"]) == ("difference", True, False, 2)
    assert c["source_names"] == ["accompaniment", "vocals"] and c["num_sources"] == 2
    c = mc(["full_multi_instrument"])
    assert c["source_names"] == ["bass", "drums", "other", "vocals"] and c["num_sources"] == 4
    cfg, extras = Config.parse_command_line(
        ["with", "cfg.full_44KHz", "cfg.model_config.batch_size=8", "input_path=a.mp3", "model_config.task=voice"])
    assert cfg["model_config"]["expected_sr"] == 44100 and cfg["model_config"]["batch_size"] == 8
    assert cfg["model_config"]["upsampling"] == "learned" and extras == {"input_path": "a.mp3"}
    with pytest.raises(NotImplementedError):
        mc([], task="speech")
    with pytest.raises(KeyError):
        mc(["nonexistent"])
    # defaults == reference base dict values (Config.py:9-39)
    d = mc([])
    assert (d["num_layers"], d["filter_size"], d["merge_filter_size"], d["num_initial_filters"],
            d["num_frames"], d["batch_size"], d["init_sup_sep_lr"]) == (12, 15, 5, 24, 16384, 16, 1e-4)


def test_get_padding_facade_matches_reference_rows():
    rows = json.load(open(os.path.join(GOLDEN, "padding.json")))
    for r in rows:
        cfg = mc([r["preset"]]) if "preset" in r else mc(["baseline_context"], **r["overrides"])
        if cfg["network"] != "unet":
            continue
        sep = UnetAudioSeparator(cfg)
        shape = np.array([cfg["batch_size"] if "preset" in r else 3, r["num_frames"], 0])
        if "error" in r:
            with pytest.raises(AssertionError):
                sep.get_padding(shape)
            continue
        i, o = sep.get_padding(shape)
        assert [int(v) for v in i] == r["in_shape"], r
        assert [int(v) for v in o] == r["out_shape"], r
        if cfg["context"]:
            assert isinstance(i, np.ndarray) and i.dtype == np.int64
        else:
            assert isinstance(i, list)


@pytest.mark.parametrize("preset", ["baseline", "baseline_stereo", "full", "full_multi_instrument",
                                    "baseline_context", "baseline_diff"])
def test_param_table_matches_oracle(preset):
    cfg = mc([preset])
    sep = UnetAudioSeparator(cfg)
    eng = sep.engine(num_frames=cfg["num_frames"])
    want = O.param_table(cfg)
    assert [(n, tuple(s)) for n, s, _, _ in eng.param_table] == [(n, tuple(s)) for n, s in want]
    off = 0
    for n, s, o, c in eng.param_table:
        assert o == off and c == int(np.prod(s))
        off += c
    assert off == eng.param_numel
    assert (eng.T_in, eng.T_out) == O.get_padding(cfg, cfg["num_frames"])


def test_live_flops_match_survey():
    """SURVEY 8(d): live forward GFLOP at B=16: M4 222.65, M6(B=32) 445.41, M1 78.20; fwd+bwd 666.1."""
    e = UnetAudioSeparator(mc(["baseline_stereo"])).engine(num_frames=16384)
    assert abs(e.forward_flops(16) * 1e-9 - 222.65) < 0.05
    assert abs(e.forward_backward_flops(16) * 1e-9 - 666.1) < 0.2
    e = UnetAudioSeparator(mc(["full_multi_instrument"])).engine(num_frames=16384)
    assert abs(e.forward_flops(32) * 1e-9 - 445.41) < 0.1
    e = UnetAudioSeparator(mc(["baseline"])).engine(num_frames=16384)
    assert abs(e.forward_flops(16) * 1e-9 - 78.20) < 0.05


def test_errors_mirror_reference():
    with pytest.raises(NotImplementedError):
        wun.Engine(wun.config_from_model_config(dict(mc(["baseline"]), output_type="foo")), num_frames=64)
    with pytest.raises(NotImplementedError):
        wun.Engine(wun.config_from_model_config(dict(mc(["baseline"]), output_activation="relu")), num_frames=64)
    with pytest.raises(AssertionError):      # :121 - lengths must match without context
        wun.Engine(wun.config_from_model_config(mc(["baseline"])), num_frames=1000)
    with pytest.raises(AssertionError):      # :55
        wun.Engine(wun.config_from_model_config(mc(["baseline_context"], num_layers=1, filter_size=3,
                                                   merge_filter_size=3, input_filter_size=3)), num_frames=-10)


def test_workspace_and_describe():
    e = UnetAudioSeparator(mc(["baseline_stereo"])).engine(num_frames=16384)
    inf, tr = e.workspace_bytes(16, False), e.workspace_bytes(16, True)
    assert 0 < inf < tr < 4e9          # ~0.6 GB saved activations + gradients at B=16
    d = e.describe()
    assert "down0" in d and "up11" in d and "T_in=147443" in d
    assert e.launches(False) > 20 and e.launches(True) > e.launches(False)


def test_compute_entry_points_fail_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("has GPU")
    e = UnetAudioSeparator(mc(["baseline"], num_layers=2)).engine(num_frames=64)
    buf = (ctypes.c_float * 16)()
    rc = wun.lib.wun_forward(e._h, ctypes.addressof(buf), ctypes.addressof(buf), 1, 0, ctypes.addressof(buf),
                             ctypes.addressof(buf), 1 << 40, None)
    assert rc == wun.WUN_E_NOGPU
    assert b"no CPU fallback" in wun.lib.wun_last_error()


# ------------------------------------------------------------------------------------------------
# plan audit: every tensor-core launch the planner would issue, against the hardware limits (no GPU needed)
# ------------------------------------------------------------------------------------------------
SMEM_LIMIT = 200 * 1024      # cudaFuncSetAttribute value of the conv and wgrad instantiations in kernels_umma.cu
SMEM_PER_SM = 228 * 1024     # H100: shared memory of one SM (1 KB of it reserved per resident CTA)


def _audit(preset, batch, overrides=None):
    from Models.UnetAudioSeparator import UnetAudioSeparator
    mc = Config.build_config([preset], overrides or {}, experiment_id=0)["model_config"]
    sep = UnetAudioSeparator(mc)
    return sep.engine(num_frames=mc["num_frames"]).plan_audit(batch)


@pytest.mark.parametrize("preset", ["baseline", "baseline_context", "baseline_stereo", "full", "full_multi_instrument", "full_44KHz"])
@pytest.mark.parametrize("batch", [1, 2, 4, 8, 16, 32])
def test_planned_tcgen05_launches_respect_hardware_limits(preset, batch):
    """Every tensor-core (wgmma) launch the planner would issue, against the H100 limits."""
    lines = _audit(preset, batch)
    convs = [d for d in lines if d["op"] == "conv"]
    wgs = [d for d in lines if d["op"] == "wgrad"]
    assert convs and wgs
    for d in convs:
        assert d["kernel"] == "wgmma", d
        # accumulators: 64 rows x NPAD fp32 registers per warpgroup
        assert d["NPAD"] % 16 == 0 and 16 <= d["NPAD"] <= 128 and d["NPAD"] * d["nsplit"] >= d["N"] and d["nsplit"] <= 4, d
        assert d["MT"] == 1 and d["rows_alloc"] % 8 == 0 and d["rows_alloc"] >= 128 + d["span"], d
        assert 1 <= d["TB"] <= 4 and 2 <= d["nbs"] <= 6, d
        assert d["smem"] <= SMEM_LIMIT and 2 * (d["smem"] + 1024) <= SMEM_PER_SM, d      # two CTAs per SM
        assert d["tiles"] >= 1 and d["span"] <= 24, d
        if d["pair"]:                                      # pair-merged class: two halves of `pair` columns
            assert d["N"] == 2 * d["pair"] and d["pair"] % 4 == 0, d
        assert not d["outfuse"], d                         # the output layer runs in its own kernels
    for d in wgs:
        assert d["NT"] % 16 == 0 and 16 <= d["NT"] <= 128 and d["NT"] * d["ntiles"] >= min(d["Cp"], d["Cg"]), d
        assert d["mtiles"] * 128 >= max(d["Cp"], d["Cg"]), d
        assert d["taps_per_cta"] * d["tapsets"] >= d["ntaps"] and 1 <= d["taps_per_cta"] <= 8, d
        assert d["taps_per_cta"] * d["NT"] <= 256, d       # register accumulators: 128 fp32 per thread
        assert d["nstages"] in (2, 3) and d["smem"] <= SMEM_LIMIT, d
        gx, gy, gz = [int(v) for v in d["grid"].split("x")]
        assert gx >= 1 and 1 <= gy <= 65535 and 1 <= gz <= 65535 and d["chunks_per_cta"] >= 1 and d["n_ctas_x"] <= gx, d


def test_plan_audit_matches_the_measured_configuration():
    """The tiling of the benchmark (M4, batch 16): every conv but the first layer's on the tensor cores, the wide layers split
    over output channels, one wgrad launch per layer."""
    lines = _audit("baseline_stereo", 16)
    fwd = {d["layer"]: d for d in lines if d["op"] == "conv" and d["pass"] == 0}
    assert all(d["kernel"] == "wgmma" for d in fwd.values())
    assert fwd[3]["NPAD"] == 96 and fwd[3]["nsplit"] == 1
    assert fwd[12]["nsplit"] >= 3 and fwd[12]["NPAD"] <= 128                  # bottleneck: 312 output channels
    assert 0 not in fwd                                                       # the first layer (C_in = 2) is a CUDA-core kernel
    assert len([d for d in lines if d["op"] == "conv"]) == 60                # 13 forward + 13 dgrad + 34 (split classes)
    assert len({d["layer"] for d in lines if d["op"] == "wgrad"}) == 24


def test_round2_planner_decisions_for_the_benchmark():
    """What bench.py times at M4 batch 16 (DESIGN.md 2 / 4.1): pair-merged forward classes for the up blocks that still fill the GPU,
    the pair-merged dgrad only where the merged width stays narrow (down1) - and no forward merge at batch 1, where those
    launches do not fill the GPU."""
    lines = [d for d in _audit("baseline_stereo", 16) if d["op"] == "conv"]
    fwd = {d["layer"]: d for d in lines if d["pass"] == 0}
    dg = [d for d in lines if d["pass"] == 1]
    assert sorted(l for l, d in fwd.items() if d["pair"]) == [20, 21, 22, 23, 24]        # up7 .. up11
    assert all(fwd[l]["N"] == 2 * fwd[l]["pair"] for l in (20, 21, 22, 23, 24))
    assert [(d["layer"], d["N"]) for d in dg if d["pair"]] == [(1, 48)]                    # down1: 2 x 24 columns
    small = [d for d in _audit("baseline_stereo", 1) if d["op"] == "conv"]
    assert not any(d["pair"] and d["pass"] == 0 for d in small)


def test_long_window_mode_plans_and_amortises_the_context():
    """SURVEY 8f N3: any num_frames builds a plan (engines are cached per input length); the 131054-frame context of M4 is
    paid once per window, so live FLOPs per OUTPUT frame fall as the window grows."""
    from oracle import wave_unet_oracle as O
    mc = Config.build_config(["baseline_stereo"], experiment_id=0)["model_config"]
    per_frame = []
    for nf in (16384, 65536, 262144):
        t_in, t_out = wun.get_padding(wun.config_from_model_config(mc), nf)
        assert (t_in, t_out) == O.get_padding(mc, nf)
        assert t_in - t_out == 147443 - 16389                 # the context is independent of the window length
        eng = wun.Engine(wun.config_from_model_config(mc), num_frames=nf)
        assert eng.T_in == t_in and eng.T_out == t_out
        per_frame.append(eng.forward_flops(1) / t_out)
        audit = eng.plan_audit(2)
        assert all(d["smem"] <= 220 * 1024 for d in audit)
    assert per_frame[0] > 1.5 * per_frame[1] > 1.5 * per_frame[2] * 1.0
    assert abs(per_frame[0] - 849e3) / 849e3 < 0.01           # SURVEY 8d: 849 kFLOP per output frame at the default window


def test_device_prefetcher_slot_protocol(monkeypatch):
    """wun.prefetch.DevicePrefetcher on fake streams / events: slots alternate, a slot is refilled only behind the `free`
    event of the copy that drained it, is consumed only behind its `ready` event, and over-issuing is refused."""
    import torch
    from wun import prefetch
    log = []

    class FakeEvent(object):
        n = 0
        def __init__(self):
            FakeEvent.n += 1; self.id = FakeEvent.n
        def record(self, stream):
            log.append(("record", self.id, stream.name))

    class FakeStream(object):
        def __init__(self, device=None, name="copy"):
            self.name = name
        def wait_event(self, ev):
            log.append(("wait", ev.id, self.name))

    class Ctx(object):
        def __init__(self, s): self.s = s
        def __enter__(self): log.append(("enter", self.s.name))
        def __exit__(self, *a): log.append(("exit", self.s.name))

    compute = FakeStream(name="compute")
    monkeypatch.setattr(torch.cuda, "Stream", FakeStream)
    monkeypatch.setattr(torch.cuda, "Event", FakeEvent)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: Ctx(s))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: compute)
    a, b = torch.zeros(4), torch.zeros(2, 3)
    pf = prefetch.DevicePrefetcher([a, b])
    ready, free = [e.id for e in pf.ready], [e.id for e in pf.free]
    h = [[torch.full((4,), float(i)), torch.full((2, 3), 10.0 + i)] for i in range(3)]
    with pytest.raises(RuntimeError):
        pf.consume()
    pf.issue(h[0]); pf.issue(h[1])
    with pytest.raises(RuntimeError):
        pf.issue(h[2])                                     # both staging slots in flight
    pf.consume()
    assert float(a[0]) == 0.0 and float(b[0, 0]) == 10.0
    pf.issue(h[2])                                          # refills slot 0 ...
    pf.consume(); assert float(a[0]) == 1.0
    pf.consume(); assert float(a[0]) == 2.0 and float(b[1, 2]) == 12.0
    ev = [x for x in log if x[0] in ("wait", "record")]
    assert ev == [("wait", free[0], "copy"), ("record", ready[0], "copy"), ("wait", free[1], "copy"), ("record", ready[1], "copy"),
                  ("wait", ready[0], "compute"), ("record", free[0], "compute"),
                  ("wait", free[0], "copy"), ("record", ready[0], "copy"),      # ... only behind the copy that drained it
                  ("wait", ready[1], "compute"), ("record", free[1], "compute"),
                  ("wait", ready[0], "compute"), ("record", free[0], "compute")]


def test_predict_track_host_logic_with_a_stub_engine():
    """Evaluate.predict_track's own work (Evaluate.py:82-145: mono mix / channel tiling, extension of short inputs, context
    padding - zero-filled on the device -, window starts with the shifted last window, batching, scatter, removal of the
    extension) with a stand-in engine on CPU tensors whose "network" returns (k + 1) x the centre crop of every window: the
    separation of source k must then be exactly (k + 1) x the (down-mixed / tiled) input, frame for frame."""
    import numpy as np
    import torch
    import Evaluate

    class StubEngine(object):
        def __init__(self, t_in, t_out, K):
            self.t_in, self.t_out, self.K = t_in, t_out, K

        def gather_windows(self, padded, starts, out):
            for i, s0 in enumerate(starts.tolist()):
                out[i] = padded[s0:s0 + self.t_in]

        def forward(self, params, batch, training=False):
            assert training is False and batch.shape[1] == self.t_in
            crop = (self.t_in - self.t_out) // 2
            core = batch[:, crop:crop + self.t_out, :]
            return torch.stack([core * float(k + 1) for k in range(self.K)])

        def scatter_windows(self, outs, starts, preds):
            for w, s0 in enumerate(starts.tolist()):
                preds[:, s0:s0 + self.t_out] = outs[:, w]

    class StubSeparator(object):
        params = None

        def __init__(self, t_in, t_out, K, C):
            self.t_in, self.t_out, self.K, self.C = t_in, t_out, K, C

        def get_padding(self, shape):
            return np.array([shape[0], self.t_in, self.C]), np.array([shape[0], self.t_out, self.C])

        def engine(self, input_frames=None):
            assert input_frames == self.t_in
            return StubEngine(self.t_in, self.t_out, self.K)

        def _ensure_params(self, eng, device, create=False):
            pass

    rng = np.random.default_rng(3)
    for mono_downmix, in_ch, n_frames in ((False, 2, 1000), (False, 2, 333), (False, 1, 700), (True, 2, 650), (False, 2, 40), (False, 2, 297)):
        cfg = {"mono_downmix": mono_downmix, "num_frames": 99, "source_names": ["a", "b", "c"]}
        C = 1 if mono_downmix else 2
        sep = StubSeparator(t_in=139, t_out=99, K=3, C=C)
        audio = rng.standard_normal((n_frames, in_ch)).astype(np.float32)
        got = Evaluate.predict_track(cfg, sep, audio, batch_windows=4, device="cpu")
        want = np.mean(audio, axis=1, keepdims=True) if mono_downmix else (np.tile(audio, [1, 2]) if in_ch == 1 else audio)
        assert list(got) == ["a", "b", "c"]
        for k, name in enumerate(got):
            assert got[name].shape == (n_frames, C) and got[name].dtype == np.float32
            np.testing.assert_array_equal(got[name], want * np.float32(k + 1), err_msg="%s %s" % (name, (mono_downmix, in_ch, n_frames)))
