"""Host-only check of the planner's launch algebra (no GPU): the engine exports the full description of every plane-convolution
launch of a training step (wun_debug_launches: planes, classes, terms - csrc/launch.h), and a numpy interpreter executes those
descriptions (tests/launch_interp.py) on a random workspace.  A pair-merged launch (launch.h OutView::pairC: two classes of equal width issued as one class
of 2C columns, round 2) must write exactly what the two-class form of the same launch writes - forward (bias + LeakyReLU with the
bias repeated per half) and dgrad (slope from the saved activation, skip-window accumulate ranges, per-half row ranges), for
context ('valid'), 'same'-padding and learned-upsampling nets.  The interpreter follows plane_conv_kernel (csrc/kernels_simt.cu),
the exact-fp32 reference form of a ConvLaunch."""
import numpy as np
import pytest

import Config
import wun
from launch_interp import decode, plane_rows, run_launch, run_wgrad_group
from oracle import wave_unet_oracle as O

CASES = [
    ("context_stereo", ["baseline_stereo"], dict(num_layers=4), 2, 700),
    ("same_padding_mono", ["baseline"], dict(num_layers=4), 2, 512),
    ("learned_upsampling", ["full"], dict(num_layers=3, num_initial_filters=16), 2, 500),
    ("same_learned_stereo", ["baseline_diff"], dict(num_layers=3, upsampling="learned", mono_downmix=False), 3, 256),
]


@pytest.mark.parametrize("name,named,ov,batch,nf", CASES, ids=[c[0] for c in CASES])
def test_pair_merged_launches_compute_what_the_two_class_launches_do(name, named, ov, batch, nf, monkeypatch):
    cfg = Config.build_config(named, ov, experiment_id=0)["model_config"]
    t_in, _ = O.get_padding(cfg, nf)
    wcfg = wun.config_from_model_config(cfg)
    for k, v in (("WUN_FOLD", "0"), ("WUN_PAIR_FWD", "0"), ("WUN_PAIR_DGRAD", "0")):
        monkeypatch.setenv(k, v)
    plain = wun.Engine(wcfg, input_frames=t_in)
    LA = plain.launch_descriptions(batch)
    for k, v in (("WUN_PAIR_FWD", "1"), ("WUN_PAIR_DGRAD", "1"), ("WUN_PAIR_MIN_CTAS", "1")):
        monkeypatch.setenv(k, v)
    merged = wun.Engine(wcfg, input_frames=t_in)
    LB = merged.launch_descriptions(batch)
    assert [(d["launch"]["layer"], d["launch"]["pass"]) for d in LA] == [(d["launch"]["layer"], d["launch"]["pass"]) for d in LB]
    n_pair_fwd = sum(1 for d in LB if d["launch"]["pairC"] and d["launch"]["pass"] == 0)
    n_pair_dg = sum(1 for d in LB if d["launch"]["pairC"] and d["launch"]["pass"] == 1)
    assert n_pair_fwd >= 2 and n_pair_dg >= 2, (n_pair_fwd, n_pair_dg)
    assert not any(d["launch"]["pairC"] for d in LA)

    rng = np.random.default_rng(5)
    n_ws = plain.workspace_bytes(batch, True) // 4
    margin = 1 << 14                                     # views may start a few rows before their tensor: keep indices in range
    mem0 = {"ws": rng.standard_normal(n_ws + 2 * margin), "par": rng.standard_normal(plain.param_numel + 64) * 0.1,
            "mix": rng.standard_normal(batch * t_in * wcfg.num_channels + 64)}
    # sigmoid(interp) blend vectors live in the workspace: keep them in (0, 1) like the engine does - any value tests the algebra
    checked = 0
    for a, b in zip(LA, LB):
        if not b["launch"]["pairC"]:
            continue
        ma = {k: v.copy() for k, v in mem0.items()}
        mb = {k: v.copy() for k, v in mem0.items()}
        for m in (ma, mb):                               # shift the workspace so that small negative offsets stay valid
            m["ws"] = m["ws"][margin:]
        run_launch(ma, a)
        run_launch(mb, b)
        changed = np.flatnonzero(ma["ws"] != mem0["ws"][margin:])
        assert changed.size > 0, a["launch"]
        np.testing.assert_allclose(mb["ws"], ma["ws"], rtol=1e-9, atol=1e-9, err_msg=str(a["launch"]))
        checked += 1
    assert checked == n_pair_fwd + n_pair_dg


def test_exported_launches_cover_the_step():
    """One forward + one dgrad description per tensor-core conv layer (the first layer has its own kernels), in execution order."""
    cfg = Config.build_config(["baseline_stereo"], dict(num_layers=3), experiment_id=0)["model_config"]
    t_in, _ = O.get_padding(cfg, 300)
    eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
    L = eng.launch_descriptions(2)
    fwd = [d["launch"]["layer"] for d in L if d["launch"]["pass"] == 0]
    assert fwd == list(range(1, 2 * 3 + 1))
    dg_layers = sorted({d["launch"]["layer"] for d in L if d["launch"]["pass"] == 1})
    assert dg_layers == list(range(1, 2 * 3 + 1))        # no input gradient for the first layer
    for d in L:
        assert len(d["planes"]) == d["launch"]["nplanes"] and len(d["cls"]) == d["launch"]["ncls"]
        assert all(0 <= t["plane"] < d["launch"]["nplanes"] for t in d["terms"])
    # the step's other launches: the dedicated first layer, the output layer, one upsampling backward per level, Adam
    kinds = [k for k, _ in eng.step_launches]
    assert kinds.count("first") == 1 and kinds.count("output") == 1 and kinds.count("adam") == 1
    ups = [d for k, d in eng.step_launches if k == "upsample"]
    assert len(ups) == 3 and all(d["dvar"] == -1 for d in ups)                  # linear upsampling: no interp gradient
    cfg = Config.build_config(["full"], dict(num_layers=3), experiment_id=0)["model_config"]
    t_in, _ = O.get_padding(cfg, 300)
    eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
    eng.launch_descriptions(2)
    ups = [d for k, d in eng.step_launches if k == "upsample"]
    assert len(ups) == 3 and all(d["dvar"] >= 0 and d["mid_mode"] != 1 for d in ups)      # learned: dvar, never MID_CLAMP


def _tensor_view(eng, name, batch, training=True):
    import ctypes
    off, rows, ch = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int32()
    wun.check(wun.lib.wun_debug_tensor(eng._h, name.encode(), int(batch), 1 if training else 0, ctypes.byref(off), ctypes.byref(rows),
                                       ctypes.byref(ch)))
    return off.value, rows.value, ch.value


FWD_CASES = [
    ("m4_like", ["baseline_stereo"], dict(num_layers=4), 2, 500),
    ("m1_like_same_padding", ["baseline"], dict(num_layers=4), 2, 512),
    ("m5_like_learned", ["full"], dict(num_layers=3, num_initial_filters=16), 2, 400),
    ("m6_like_multi_instrument", ["full_multi_instrument"], dict(num_layers=3), 2, 300),
    ("same_learned_stereo", ["baseline_diff"], dict(num_layers=3, upsampling="learned", mono_downmix=False), 2, 256),
]


@pytest.mark.parametrize("pairs", [0, 1], ids=["two_class", "pair_merged"])
@pytest.mark.parametrize("name,named,ov,batch,nf", FWD_CASES, ids=[c[0] for c in FWD_CASES])
def test_exported_forward_launches_reproduce_the_oracle(name, named, ov, batch, nf, pairs, monkeypatch):
    """The planner's forward pass - live rows only, decimation / skip crop / upsampling folded into plane views, pair-merged
    classes - executed by the numpy interpreter on the host must reproduce every activation the engine keeps (dec_i, odd_i, z,
    up_i at their live rows, tests/helpers.py) of the oracle's get_output (UnetAudioSeparator.py:97-125) in float64."""
    import torch
    from helpers import live_rows
    for k, v in (("WUN_FIRST_LAYER", "0"), ("WUN_FOLD", "0"), ("WUN_PAIR_FWD", str(pairs)), ("WUN_PAIR_MIN_CTAS", "1")):
        monkeypatch.setenv(k, v)
    cfg = Config.build_config(named, ov, experiment_id=0)["model_config"]
    t_in, t_out = O.get_padding(cfg, nf)
    params = O.init_params(cfg, seed=3)
    rng = np.random.default_rng(4)
    for k in params:
        if k.endswith("/bias") or "interp" in k:
            params[k] = rng.uniform(-0.5, 0.5, size=params[k].shape).astype(np.float32)
    mix, _ = O.synthetic_batch(cfg, batch, t_in, t_out, seed=9)
    eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
    fwd = [d for d in eng.launch_descriptions(batch) if d["launch"]["pass"] == 0]
    L = cfg["num_layers"]
    assert [d["launch"]["layer"] for d in fwd] == list(range(2 * L + 1))           # incl. the first layer (generic path)
    if pairs:
        assert any(d["launch"]["pairC"] for d in fwd)
    par = np.zeros(eng.param_numel + 64)
    for pname, shape, off, numel in eng.param_table:
        par[off:off + numel] = np.asarray(params[pname], np.float64).reshape(-1)
    margin = 1 << 14
    n_ws = eng.workspace_bytes(batch, True) // 4
    ws_full = np.zeros(n_ws + 2 * margin)
    mem = {"ws": ws_full[margin:], "par": par, "mix": np.concatenate([mix.astype(np.float64).reshape(-1), np.zeros(64)])}
    if cfg["upsampling"] == "learned":                                           # sigmoid(interp_<level>) - launch_sigmoid in the engine
        for i in range(L):
            off, rows, ch = _tensor_view(eng, "wsig%d" % i, batch)
            var = np.asarray(params["separator/interp_%d" % i], np.float64).reshape(-1)
            mem["ws"][off:off + var.size] = 1.0 / (1.0 + np.exp(-var))
    for d in fwd:
        run_launch(mem, d)
    _, inter = O.forward(cfg, O._as_torch(params, torch.float64, False), torch.as_tensor(mix).to(torch.float64), False,
                         return_intermediates=True)
    keys = ["down%d" % i for i in range(L)] + ["bottleneck"] + ["up%d" % i for i in range(L)]
    checked = 0
    for idx, views in live_rows(cfg, t_in).items():
        want_full = inter[keys[idx]].numpy()
        for tname, rows in views:
            off, trows, ch = _tensor_view(eng, tname, batch)
            assert trows == len(rows) and ch == want_full.shape[2], (tname, trows, len(rows))
            got = mem["ws"][off:off + batch * trows * ch].reshape(batch, trows, ch)
            np.testing.assert_allclose(got, want_full[:, rows, :], rtol=1e-9, atol=1e-11, err_msg=tname)
            checked += 1
    assert checked == 2 * L + 1 + L



def _upsample_bwd(mem, eng, batch, up_i, L_layers, dg_launches, fwd_launch):
    """upsample_bwd_kernel (kernels_simt.cu) on the host: gradient w.r.t. the PRE-activation of the tensor that up block `up_i`
    upsamples, from the gradients w.r.t. its copied rows (g_ue) and interpolated rows (g_mid)."""
    views = []                                            # (base, bstride, rows) of g_ue and g_mid, from the dgrad launch that wrote them
    d = dg_launches[-1]                                   # second launch of the layer: the upsampled pair
    if d["launch"]["pairC"]:
        q = d["cls"][0]
        views = [(q["base"], q["bstride"], q["hi0"]), (q["base2"], q["bstride2"], q["hi1"])]
    else:
        views = [(q["base"], q["bstride"], q["m_hi"]) for q in d["cls"]]
    mid = [P for P in fwd_launch["planes"] if P["kind"] == 1][0]
    C = mid["C"]
    (ue_base, ue_bs, N), (gm_base, gm_bs, nmid) = views
    _, ue = decode(ue_base)
    _, gm = decode(gm_base)
    src = "z" if up_i == 0 else "up%d" % (up_i - 1)
    xoff, xrows, xc = _tensor_view(eng, src, batch)
    goff, _, _ = _tensor_view(eng, "g_" + src, batch)
    assert xrows == N and xc == C and ue_bs == N * C and gm_bs == nmid * C
    ws = mem["ws"]
    w = np.full(C, 0.5)
    if mid["blend"] >= 0:
        _, boff = decode(mid["blend"])
        w = ws[boff:boff + C].copy()
    for b in range(batch):
        x = ws[xoff + b * N * C: xoff + (b + 1) * N * C].reshape(N, C)
        due = ws[ue + b * N * C: ue + (b + 1) * N * C].reshape(N, C)
        dmid = ws[gm + b * nmid * C: gm + (b + 1) * nmid * C].reshape(nmid, C)
        dm = np.zeros((N, C)); dm[:nmid] = dmid
        dmp = np.zeros((N, C)); dmp[1:min(N, nmid + 1)] = dmid[:min(N, nmid + 1) - 1]
        g = due + w * dm + (1.0 - w) * dmp
        if mid["mid_mode"] == 1:                          # MID_CLAMP: the last row's "next" row is itself
            g[N - 1] += (1.0 - w) * dm[N - 1]
        ws[goff + b * N * C: goff + (b + 1) * N * C] = (g * np.where(x > 0.0, 1.0, 0.2)).reshape(-1)


def _host_backward(named, ov, batch, nf, pairs, monkeypatch):
    """Forward launches, then the dgrad chain seeded with the oracle's gradient at the last up block, all on the host.
    Returns (cfg, eng, mem, dpre, param_grads, keys, t_in): dpre / param_grads are torch autograd through the oracle in float64."""
    import torch
    for k, v in (("WUN_FIRST_LAYER", "0"), ("WUN_FOLD", "0"), ("WUN_PAIR_FWD", str(pairs)), ("WUN_PAIR_DGRAD", str(pairs)),
                 ("WUN_PAIR_MIN_CTAS", "1")):
        monkeypatch.setenv(k, v)
    cfg = Config.build_config(named, ov, experiment_id=0)["model_config"]
    t_in, t_out = O.get_padding(cfg, nf)
    params = O.init_params(cfg, seed=3)
    rng = np.random.default_rng(4)
    for k in params:
        if k.endswith("/bias") or "interp" in k:
            params[k] = rng.uniform(-0.5, 0.5, size=params[k].shape).astype(np.float32)
    mix, targets = O.synthetic_batch(cfg, batch, t_in, t_out, seed=9)
    eng = wun.Engine(wun.config_from_model_config(cfg), input_frames=t_in)
    desc = eng.launch_descriptions(batch)
    fwd = [d for d in desc if d["launch"]["pass"] == 0]
    dg = [d for d in desc if d["launch"]["pass"] == 1]
    L = cfg["num_layers"]
    if pairs:
        assert any(d["launch"]["pairC"] for d in dg)
    par = np.zeros(eng.param_numel + 64)
    for pname, shape, off, numel in eng.param_table:
        par[off:off + numel] = np.asarray(params[pname], np.float64).reshape(-1)
    margin = 1 << 14
    ws_full = np.zeros(eng.workspace_bytes(batch, True) // 4 + 2 * margin)
    mem = {"ws": ws_full[margin:], "par": par, "mix": np.concatenate([mix.astype(np.float64).reshape(-1), np.zeros(64)])}
    if cfg["upsampling"] == "learned":
        for i in range(L):
            off, rows, ch = _tensor_view(eng, "wsig%d" % i, batch)
            var = np.asarray(params["separator/interp_%d" % i], np.float64).reshape(-1)
            mem["ws"][off:off + var.size] = 1.0 / (1.0 + np.exp(-var))
    for d in fwd:
        run_launch(mem, d)
    # oracle: dL/d(pre-activation) of every layer output = autograd gradient w.r.t. the activation x LeakyReLU slope
    tp = O._as_torch(params, torch.float64, True)
    outs, inter = O.forward(cfg, tp, torch.as_tensor(mix).to(torch.float64), True, return_intermediates=True)
    loss = O.mse_loss(cfg, outs, {k: torch.as_tensor(v).to(torch.float64) for k, v in targets.items()})
    keys = ["down%d" % i for i in range(L)] + ["bottleneck"] + ["up%d" % i for i in range(L)]
    pnames = sorted(tp)
    grads = torch.autograd.grad(loss, [inter[k] for k in keys] + [tp[k] for k in pnames], allow_unused=True)
    dpre = {k: g.detach().numpy() * np.where(inter[k].detach().numpy() > 0.0, 1.0, 0.2) for k, g in zip(keys, grads)}      # (float64 0.2)
    param_grads = {k: (None if g is None else g.detach().numpy()) for k, g in zip(pnames, grads[len(keys):])}
    # seed: the gradient at the features (what output_dgrad / the fused epilogue writes)
    goff, grows, gch = _tensor_view(eng, "g_up%d" % (L - 1), batch)
    mem["ws"][goff:goff + batch * grows * gch] = dpre["up%d" % (L - 1)].reshape(-1)
    # the chain, in the engine's order: up blocks from the last to the first (each followed by the upsampling backward), bottleneck, down blocks
    by_layer = {}
    for d in dg:
        by_layer.setdefault(d["launch"]["layer"], []).append(d)
    for i in range(L - 1, -1, -1):
        launches = by_layer[L + 1 + i]
        for d in launches:
            run_launch(mem, d)
        _upsample_bwd(mem, eng, batch, i, L, launches, fwd[L + 1 + i])
    for layer in range(L, 0, -1):
        for d in by_layer[layer]:
            run_launch(mem, d)
    return cfg, eng, mem, dpre, param_grads, keys, t_in


@pytest.mark.parametrize("pairs", [0, 1], ids=["two_class", "pair_merged"])
@pytest.mark.parametrize("name,named,ov,batch,nf", FWD_CASES, ids=[c[0] for c in FWD_CASES])
def test_exported_dgrad_chain_reproduces_the_oracle(name, named, ov, batch, nf, pairs, monkeypatch):
    """The backward data path on the host: starting from the oracle's gradient at the last up block, the exported dgrad launches
    (roles swapped: class gradients are the planes; skip-window accumulate ranges; row ranges written first by the up block and
    then by the down block) plus the upsampling backward must reproduce dL/d(pre-activation) of EVERY saved activation at its live
    rows - torch autograd through the oracle's get_output, float64."""
    from helpers import live_rows
    cfg, eng, mem, dpre, _, keys, t_in = _host_backward(named, ov, batch, nf, pairs, monkeypatch)
    L = cfg["num_layers"]
    checked = 0
    for idx, views in live_rows(cfg, t_in).items():
        want_full = dpre[keys[idx]]
        for tname, rows in views:
            off, trows, ch = _tensor_view(eng, "g_" + tname, batch)
            got = mem["ws"][off:off + batch * trows * ch].reshape(batch, trows, ch)
            scale = max(1e-30, float(np.abs(want_full).max()))
            np.testing.assert_allclose(got / scale, want_full[:, rows, :] / scale, rtol=1e-8, atol=1e-10, err_msg="g_" + tname)
            checked += 1
    assert checked == 3 * L + 1


@pytest.mark.parametrize("name,named,ov,batch,nf", FWD_CASES, ids=[c[0] for c in FWD_CASES])
def test_exported_wgrad_groups_reproduce_the_oracle(name, named, ov, batch, nf, monkeypatch):
    """The weight-gradient groups the engine builds per layer ((class, plane) pairs with up to 8 taps each - what the split pass
    and the tensor-core wgrad kernel consume), executed on the host on the activations and pre-activation gradients the exported
    forward / dgrad launches produced, must give dL/dW of every convolution; the column sums of each class's gradient view give
    dL/db (fused into the split pass on the device).  Reference: torch autograd through the oracle (UnetAudioSeparator.py:97-125), float64."""
    cfg, eng, mem, _, param_grads, keys, t_in = _host_backward(named, ov, batch, nf, 1, monkeypatch)
    L = cfg["num_layers"]
    groups = eng.wgrad_groups
    assert sorted({G["wgrad"]["layer"] for G in groups}) == list(range(2 * L + 1))
    got = np.zeros(eng.param_numel + 64)
    seen = set()
    for G in groups:
        g = G["wgrad"]
        assert 1 <= g["nterms"] == len(G["terms"]) <= 8 and g["batch"] == batch
        assert max(t["d"] for t in G["terms"]) - min(t["d"] for t in G["terms"]) <= 15      # one staged slab serves every tap of the group
        run_wgrad_group(mem, G, got)
        key = (g["layer"], G["dpre"]["base"], G["dpre"]["r_lo"], G["dpre"]["r_hi"])
        if key not in seen:                                                       # bias: once per class
            seen.add(key)
            rows = np.arange(g["m_lo"], g["m_hi"])
            for b in range(batch):
                got[g["db"]:g["db"] + g["N"]] += plane_rows(mem, G["dpre"], b, rows)[:, :g["N"]].sum(0)
    conv_offsets = {G["wgrad"]["dW"] for G in groups} | {G["wgrad"]["db"] for G in groups}
    checked = []
    for pname, shape, off, numel in eng.param_table:
        if off not in conv_offsets:
            continue                                  # interp_<i> and the 1x1 output layer have their own kernels (OutputLayer.py:5-23)
        want = np.asarray(param_grads[pname], np.float64).reshape(-1)
        scale = max(1e-30, float(np.abs(want).max()))
        np.testing.assert_allclose(got[off:off + numel] / scale, want / scale, rtol=1e-8, atol=1e-10, err_msg=pname)
        checked.append(pname)
    assert len(checked) == 2 * (2 * L + 1), checked
