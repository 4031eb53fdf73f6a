"""Per-tensor gradient error of the engine (tensor cores on / off) vs the fp64 and fp32 oracle on one M4 window."""
import os, sys, numpy as np, torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO); sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
import Config
from Models.UnetAudioSeparator import UnetAudioSeparator
from oracle import wave_unet_oracle as O

preset = sys.argv[1] if len(sys.argv) > 1 else "baseline_stereo"
L = int(sys.argv[2]) if len(sys.argv) > 2 else 12
cfg = Config.build_config([preset], dict(num_layers=L), experiment_id=0)["model_config"]
t_in, t_out = O.get_padding(cfg, cfg["num_frames"])
seed = int(sys.argv[3]) if len(sys.argv) > 3 else 1337
params = O.init_params(cfg, seed=seed)
rng = np.random.default_rng(seed + 1)
for k in params:
    if k.endswith("/bias"): params[k] = rng.uniform(-0.05, 0.05, size=params[k].shape).astype(np.float32)
mix, targets = O.synthetic_batch(cfg, 1, t_in, t_out, seed=seed + 2)
torch.set_num_threads(os.cpu_count())
l64, o64, g64 = O.forward_backward(cfg, params, mix, targets, dtype=torch.float64)
l32, o32, g32 = O.forward_backward(cfg, params, mix, targets, dtype=torch.float32)
res = {}
MODES = {"umma": ("1", "1"), "fwd_only": ("1", "0"), "dgrad_only": ("0", "1"), "simt": ("0", "0")}
for mode, (f, d) in MODES.items():
    os.environ["WUN_UMMA_FWD"] = f; os.environ["WUN_UMMA_DGRAD"] = d
    sep = UnetAudioSeparator(cfg); sep.load_variables(params, input_frames=t_in)
    tg = {k: torch.from_numpy(v).cuda() for k, v in targets.items()}
    loss = sep.loss_and_gradients(torch.from_numpy(mix).cuda(), tg)
    res[mode] = (float(loss.item()), {n: g.cpu().numpy().copy() for n, g in sep.gradients().items()})
rel = lambda a, b: float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-300))
print("loss fp64 %.9f fp32 %.9f " % (l64, l32) + " ".join("%s %.9f" % (m, res[m][0]) for m in MODES))
print("%-30s %9s " % ("tensor", "oracle32") + " ".join("%10s" % m for m in MODES) + "   |g|")
worst = {m: (0, "") for m in MODES}
for n in params:
    errs = {m: rel(res[m][1][n], g64[n]) for m in MODES}
    for m in MODES:
        if errs[m] > worst[m][0]: worst[m] = (errs[m], n)
    print("%-30s %9.2e " % (n[10:], rel(g32[n], g64[n])) + " ".join("%10.2e" % errs[m] for m in MODES) + "  %.2e" % np.linalg.norm(g64[n]))
print("WORST", worst)

# ---- LeakyReLU mask flips: where does the engine's saved activation differ in SIGN from the fp64 oracle? ----
with torch.no_grad():
    pt = O._as_torch(params, torch.float64, False)
    _, inter = O.forward(cfg, pt, torch.from_numpy(mix).double(), True, return_intermediates=True)
os.environ["WUN_UMMA_FWD"] = "1"; os.environ["WUN_UMMA_DGRAD"] = "1"
sep = UnetAudioSeparator(cfg); sep.load_variables(params, input_frames=t_in)
sep.loss_and_gradients(torch.from_numpy(mix).cuda(), {k: torch.from_numpy(v).cuda() for k, v in targets.items()})
torch.cuda.synchronize()
eng = sep.engine(input_frames=t_in)
for i in range(L):
    ref = inter["down%d" % i].numpy()[:, ::2]
    got = eng.debug_tensor("dec%d" % i, 1, True).cpu().numpy()
    flips = (got > 0) != (ref > 0)
    mags = np.abs(ref[flips])
    print("dec%-2d elements %8d  sign flips %4d  max|ref| at flips %.2e  rel err of layer %.2e" %
          (i, ref.size, flips.sum(), mags.max() if mags.size else 0.0, rel(got, ref)))
