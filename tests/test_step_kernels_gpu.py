"""The rest of a training step, launch by launch, against float64: the first-layer forward and weight gradient (kernels_first.cu),
the output layer's forward (estimates, difference output, clip, loss, dL/dpre), dgrad and weight gradient, the upsampling backward
with the interp gradient, sigmoid, Adam and the window gather / scatter of prediction (kernels_simt.cu).

Each launch runs alone through tests/kernels/harness.cu (the product's own launchers) on buffers framed by GUARD sentinel words;
words the launch contract says are never read (gaps of wide batch strides, partial-sum arenas before they are written) hold NaN.
Every word outside a launch's outputs must keep its bits, gradients are pre-filled (the contract is +=), the partial-sum arenas
are exactly as long as the product's size functions say and followed by a guard, and every reduction runs twice with the same
bits.  The regimes and the report are those of tests/test_kernels_gpu.py:
  exact - activations k/4 in [-4, 4], weights integers in [-3, 3], blend weights in {1/4, 1/2, 3/4}, power-of-two scales and
          inv_count: every sum is exact in fp32 (checked per case), so the result must equal float64 bit for bit, with the fp32
          epilogues applied in the kernels' order.
  float - random data over a wide dynamic range: |got - ref| <= TAU * ref_abs (+ a stated ulp allowance for tanhf / expf /
          sqrtf and division), ref_abs the same computation on |x| and |w|.  A power check per family shows TAU flags one
          dropped item of the kind that family can lose.
Replays run every first / output / upsample / adam launch the engine emits for the configurations of
tests/configurations.py REPLAYS and M5 at batch 16, on random buffers of the exported geometry.  The launch runners are in
tests/step_launches.py, the bounds and checks in tests/launch_checks.py.
"""
import pytest
import torch

import configurations
from launch_checks import COUNTS, GUARD, SENTINEL, U32, H, Mem, check, engine, gpu_lib, lib_or_skip, print_report, set_env, stream
from step_launches import (replay_step_launches, run_adam, run_first_fwd, run_first_wgrad, run_output_dgrad, run_output_fwd,
                           run_output_wgrad, run_upsample)


# ------------------------------------------------------------------------------------------------
# first layer
# ------------------------------------------------------------------------------------------------
def first_case(C, N, k, pad, T, batch, stride_pad=0, name=None):
    Td = (T + 1) // 2 + 2                                   # the last rows read x past T (zero)
    mo_lo, mo_hi = 3, Td - 5 - (k % 3)                      # a shorter odd class: its CTAs exit early on the last row tile
    return dict(C=C, N=N, k=k, pad_left=pad, batch=batch, T=T, x_bstride=T * C + stride_pad * C, Td=Td, dec_bstride=Td * N + stride_pad * N,
                mo_lo=mo_lo, mo_hi=mo_hi, odd_bstride=(mo_hi - mo_lo) * N + stride_pad * N, name=name or "C%dN%dk%dp%dT%db%d" % (C, N, k, pad, T, batch))


def first_cases():
    cs = []
    lib = H.load()
    for C, N in ((1, 16), (1, 24), (2, 16), (2, 24)):
        kmax = max(k for k in range(1, 17) if lib.wkh_first_supported(C, N, k))
        for k in range(1, kmax + 1):
            for pad in sorted({0, (k - 1) // 2}):
                cs.append(first_case(C, N, k, pad, 601 + 37 * k, 1 + (k % 3), stride_pad=(k % 2) * 5))
    return cs


# ------------------------------------------------------------------------------------------------
# output layer
# ------------------------------------------------------------------------------------------------
def out_case(*, batch, Tf, C, F, K_, ofs, output_type, activation, training, pad=None, name=""):
    nconv = K_ - 1 if output_type == 1 else K_
    pad = (ofs - 1) // 2 if pad is None else pad
    T_out = Tf - (ofs - 1) + 2 * pad                       # 'valid' conv of the feature rows, with pad rows of zeros on the left
    crop_feat, crop_out = 7, 7 + 3
    T_in = max(crop_feat + Tf, crop_out + T_out) + 5
    G = dict(batch=batch, T_in=T_in, Tf=Tf, T_out=T_out, C=C, F=F, nconv=nconv, K=K_, ofs=ofs, pad_left=pad, crop_feat=crop_feat,
             crop_out=crop_out, output_type=output_type, activation=activation, training=training, name=name)
    off = 16                                                # the output convs' weights and biases, NaN between them
    for s in range(8):
        if s < nconv:
            G["w_off%d" % s] = off
            off += ofs * (C + F) * C + 9
            G["b_off%d" % s] = off
            off += C + 5
        else:
            G["w_off%d" % s] = G["b_off%d" % s] = -1
    G["n_params"] = off + 16
    return G


def output_cases():
    cs = []
    for ot in (0, 1):
        for act in (0, 1):
            for tr in (0, 1):
                # B * T_out * C * K a power of two (inv_count exact); ofs 1 and 3 with both paddings
                cs.append(out_case(batch=2, Tf=256 + 0, C=2, F=24, K_=2, ofs=1, output_type=ot, activation=act, training=tr,
                                   name="ot%d_act%d_tr%d_ofs1" % (ot, act, tr)))
                cs.append(out_case(batch=4, Tf=128, C=1, F=31, K_=4, ofs=3, pad=1, output_type=ot, activation=act, training=tr,
                                   name="ot%d_act%d_tr%d_ofs3_same" % (ot, act, tr)))
                cs.append(out_case(batch=1, Tf=258, C=2, F=8, K_=2, ofs=3, pad=0, output_type=ot, activation=act, training=tr,
                                   name="ot%d_act%d_tr%d_ofs3_valid" % (ot, act, tr)))
    # nconv * C = WUN_MAX_OUT_COLS (8 sources, stereo, direct); F = 33 (Cin + 1 = 36 > 32: the second cbase pass)
    cs.append(out_case(batch=2, Tf=64, C=2, F=33, K_=8, ofs=1, output_type=0, activation=1, training=1, name="cols16_F33"))
    cs.append(out_case(batch=2, Tf=66, C=2, F=12, K_=8, ofs=3, pad=0, output_type=1, activation=0, training=1, name="diff8_ofs3"))
    return cs


# ------------------------------------------------------------------------------------------------
# upsampling backward
# ------------------------------------------------------------------------------------------------
def up_cases():
    cs = []
    for mode in (0, 1, 2):
        for B, N, C in ((1, 40, 24), (3, 300, 50), (16, 2000, 72), (2, 9000, 17)):
            nmid = N - 1 if mode == 0 else N
            cs.append(dict(batch=B, N=N, nmid=nmid, C=C, mid_mode=mode, name="mode%d_B%d_N%d_C%d" % (mode, B, N, C)))
    return cs


# ------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "float"])
def test_first_layer_matches_float64(regime):
    gpu_lib()
    for i, G in enumerate(first_cases()):
        run_first_fwd(G, regime, 100 + i)
        run_first_wgrad(G, regime, 300 + i, scale=0.5 if i % 2 else 2.0, null_db=(i % 7 == 3))
    if regime == "float":
        # a batch large enough that rows_per_cta grows past 128 (several 128-row blocks per CTA), wide batch strides, batch 1
        for C, N in ((1, 16), (1, 24), (2, 16), (2, 24)):
            G = first_case(C, N, 5, 2, 8001, 20, stride_pad=3, name="big_C%dN%d" % (C, N))
            run_first_fwd(G, regime, 11)
            run_first_wgrad(G, regime, 12)
        G = first_case(2, 24, 15, 7, 300001, 1, name="long_b1")
        run_first_fwd(G, regime, 13)
        run_first_wgrad(G, regime, 14)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "float"])
def test_output_layer_matches_float64(regime):
    gpu_lib()
    for i, G in enumerate(output_cases()):
        if regime == "exact" and G["activation"] == 0:
            continue                                          # tanhf: float regime only
        run_output_fwd(G, regime, 500 + i)
        run_output_fwd(G, regime, 600 + i, targets=(i % 2 == 0), outputs=(i % 2 == 1))
        run_output_dgrad(G, regime, 700 + i)
        run_output_wgrad(G, regime, 800 + i)
    # B * Tf * F above 132 * 16 * 256: output_dgrad_kernel's grid-stride loop runs; many row chunks in the wgrad
    G = out_case(batch=16, Tf=8192, C=2, F=24, K_=2, ofs=1, output_type=1, activation=1, training=1, name="b16_long")
    run_output_dgrad(G, regime, 900)
    run_output_fwd(G, regime, 901)
    if regime == "float":
        run_output_wgrad(G, regime, 902)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "float"])
def test_upsample_backward_matches_float64(regime):
    gpu_lib()
    for i, G in enumerate(up_cases()):
        for learned in (False, True):
            if learned and G["mid_mode"] == 1:
                continue                                      # the plan never pairs learned upsampling with MID_CLAMP (host test)
            if regime == "exact" and G["batch"] * G["N"] > 20000 and learned:
                continue                                      # dvar sums leave the exact range
            run_upsample(G, regime, 1000 + i, learned)


@pytest.mark.gpu
def test_adam_matches_float64():
    gpu_lib()
    for n in (0, 1, 2, 3, 4, 5, 4097, 132 * 8 * 256 * 4 + 13):
        for dev in (False, True):
            if n == 0:
                z = torch.zeros(8, device="cuda")
                H.call("adam", z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), 0, 1e-3, 0.9, 0.999, 1e-8, 0, stream())
                torch.cuda.synchronize()
                assert not bool(z.any())
                continue
            run_adam(n, 40 + n % 97, dev, steps=3 if dev else 1)


@pytest.mark.gpu
def test_sigmoid_extreme_inputs():
    gpu_lib()
    xs = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 1.0, -1.0, 15.0, -15.0, 87.0, -87.0, 88.5, -88.5, 89.0, -89.0, 100.0, -100.0,
                       1e30, -1e30, float("inf"), float("-inf"), float("nan")], device="cuda")
    xs = torch.cat([xs, torch.randn(1000, device="cuda") * 30])
    mem = Mem()
    mem.add("x", xs)
    mem.add("y", torch.full_like(xs, float(SENTINEL)))
    before = mem.snapshot()
    H.call("sigmoid", mem.ptr("x"), mem.ptr("y"), xs.numel(), stream())
    torch.cuda.synchronize()
    mem.check_rest(before, {"y": torch.ones(xs.numel(), dtype=torch.bool, device="cuda")}, "sigmoid")
    y, x = mem.d("y"), xs.double()
    ref = 1.0 / (1.0 + torch.exp(-x))
    fin = ~torch.isnan(x)
    assert bool(torch.isnan(y[~fin]).all())
    # expf <= 2 ulp, the add and the division <= 0.5 ulp each; below 2^-126 the result is subnormal (absolute floor)
    check("sigmoid", y[fin], ref[fin], 4 * U32 * ref[fin].abs() + 2.0 ** -126, "sigmoid")
    assert bool((y[fin] >= 0).all() & (y[fin] <= 1).all())
    COUNTS["sigmoid"] += 1


@pytest.mark.gpu
def test_gather_scatter_windows_bit_exact():
    gpu_lib()
    for C, T_in, T_out, n_frames, K_ in ((2, 300, 100, 1234, 3), (1, 64, 16, 50, 2), (2, 1000, 400, 100000, 4)):
        step = T_out
        starts = list(range(0, n_frames - T_out + 1, step))
        if not starts or starts[-1] + T_out < n_frames:
            starts.append(n_frames - T_out)                   # the shifted last window overlaps its predecessor
        nw = len(starts)
        n_padded = n_frames + (T_in - T_out) // 2 + 3          # windows near the end read past n_padded (zeros)
        st = torch.tensor(starts, dtype=torch.int64, device="cuda")
        padded = torch.randn(n_padded * C + 8, device="cuda")
        padded[n_padded * C:] = float("nan")                   # never read
        out = torch.full((nw * T_in * C + GUARD,), float(SENTINEL), device="cuda")
        H.call("gather_windows", padded.data_ptr(), n_padded, st.data_ptr(), nw, T_in, C, out.data_ptr(), stream())
        torch.cuda.synchronize()
        src = (st[:, None] * C + torch.arange(T_in * C, device="cuda")[None, :]).reshape(-1)
        want = torch.where(src < n_padded * C, padded[src.clamp(max=n_padded * C - 1)], torch.zeros((), device="cuda"))
        assert torch.equal(out[:nw * T_in * C].view(torch.int32), want.view(torch.int32))
        assert bool((out[nw * T_in * C:] == SENTINEL).all())
        assert starts[-1] + T_in > n_padded                    # the case reaches the zero fill
        outs = torch.randn(K_ * nw * T_out * C, device="cuda")
        preds = torch.full((K_ * n_frames * C + GUARD,), float(SENTINEL), device="cuda")
        H.call("scatter_windows", outs.data_ptr(), st.data_ptr(), nw, K_, T_out, C, preds.data_ptr(), n_frames, stream())
        torch.cuda.synchronize()
        ref = torch.full((K_, n_frames, C), float(SENTINEL), device="cuda")
        o = outs.view(K_, nw, T_out, C)
        for w in range(nw):                                    # in order: the last window wins where it overlaps
            a, b = starts[w], min(starts[w] + T_out, n_frames)
            ref[:, a:b] = o[:, w, :b - a]
        assert torch.equal(preds[:K_ * n_frames * C].view(torch.int32), ref.reshape(-1).view(torch.int32))
        assert bool((preds[K_ * n_frames * C:] == SENTINEL).all())
    COUNTS["gather/scatter"] += 1


# ------------------------------------------------------------------------------------------------
# replays: the step launches the engine emits
# ------------------------------------------------------------------------------------------------
REPLAYS = configurations.REPLAYS + [("M5_full_b16", ["full"], {}, 16, None, {})]


@pytest.mark.gpu
@pytest.mark.parametrize("name,named,ov,batch,nf,env", REPLAYS, ids=[r[0] for r in REPLAYS])
def test_replayed_step_launches_match_float64(name, named, ov, batch, nf, env, monkeypatch):
    gpu_lib()
    set_env(monkeypatch, env)
    replay_step_launches(name, named, ov, batch, nf, adam=batch == 1 and name.startswith("M"))


# ------------------------------------------------------------------------------------------------
# host tests (no GPU)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,named,ov,batch,nf,env", REPLAYS, ids=[r[0] for r in REPLAYS])
def test_exported_step_launches_parse_and_learned_upsampling_never_clamps(name, named, ov, batch, nf, env, monkeypatch):
    """Host only: every configuration exports one output and one adam line, one upsample line per level (with an interp gradient
    exactly for learned upsampling) and a first line exactly when the dedicated first layer runs.  The kernel's interp gradient
    at row N-1 is only right for MID_ZERO and MID_VALID: the plan never builds learned upsampling with MID_CLAMP."""
    lib = lib_or_skip()
    set_env(monkeypatch, env)
    cfg, _, eng, _ = engine(named, ov, batch, nf)
    kinds = [k for k, _ in eng.step_launches]
    assert kinds.count("output") == 1 and kinds.count("adam") == 1
    ups = [d for k, d in eng.step_launches if k == "upsample"]
    assert sorted(d["level"] for d in ups) == list(range(cfg["num_layers"]))
    learned = cfg["upsampling"] == "learned"
    for d in ups:
        assert (d["dvar"] >= 0) == learned and (d["blend"] >= 0) == learned
        assert not (d["dvar"] >= 0 and d["mid_mode"] == 1)
        assert d["batch"] == batch and d["nmid"] in (d["N"], d["N"] - 1)
    dedicated = bool(lib.wkh_first_supported(cfg["num_channels"], cfg["num_initial_filters"], cfg["input_filter_size"]))
    assert kinds.count("first") == (1 if dedicated else 0), (kinds.count("first"), dedicated)
    for d in (d for k, d in eng.step_launches if k == "first"):
        assert d["batch"] == batch and d["k"] == cfg["input_filter_size"] and d["N"] == cfg["num_initial_filters"]
    assert dict(eng.step_launches)["adam"]["n"] == eng.param_numel
    monkeypatch.setenv("WUN_FIRST_LAYER", "0")
    eng0 = engine(named, ov, batch, nf)[2]
    assert "first" not in [k for k, _ in eng0.step_launches]


@pytest.mark.gpu
def test_zz_step_report():
    """Prints the case count per kernel family, the exact-regime matches and the worst err / ref_abs of the float regime."""
    print_report("kernel family", required=("first fwd", "first wgrad", "output fwd", "output dgrad", "output wgrad", "upsample bwd",
                                            "adam", "sigmoid", "gather/scatter"))
