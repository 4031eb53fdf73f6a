"""GPU timing of one training step of the spectrogram U-Net baselines U7 (preset unet_spectrogram, L2 loss on audio) and
U7a (unet_spectrogram_l1, L1 loss on magnitudes) on 98 560-sample windows, random parameters and batches:
   - the step (UnetSpectrogramSeparator.loss_and_gradients + adam_step: STFT, both U-Nets forward and backward, loss,
     Adam) at batch 4 and 8: CUDA events over --iters steps after a warm-up, and the convolutions' rate from the closed
     form (wun_spec_train_flops: forward + input-gradient + weight-gradient FLOPs; 67 TFLOP/s is NVIDIA's data-sheet FP32
     rate of the H100 SXM at up to 700 W, so the share is of that figure, not of this card's clock);
   - with --profile, instead: per-kernel times of --iters U7 steps at batch 4 from torch.profiler (a separate run, since
     tracing slows the host), summed per kernel name.
Prints JSON with the card name, power limit and SM clock.
   python tools/spectrogram_train_table.py [--iters 20] [--profile] [--out FILE]"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import torch  # noqa: E402
import Config  # noqa: E402
from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator  # noqa: E402
from conv_table import card  # noqa: E402
from oracle import spectrogram_oracle as S  # noqa: E402

DATASHEET_FP32_TFLOPS = 67.0
LR = 1e-4


def setup(preset, batch):
    cfg = Config.build_config([preset], experiment_id=0)["model_config"]
    sep = UnetSpectrogramSeparator(cfg)
    T = cfg["num_frames"]
    sep.load_variables(S.random_params(cfg["num_layers"], cfg["num_initial_filters"], seed=1),
                       device=torch.device("cuda"), num_frames=T)
    g = torch.Generator().manual_seed(batch)
    targets = ((torch.rand((2, batch, T, 1), generator=g) - 0.5) * 0.5).cuda()
    mix = targets.sum(0).contiguous()
    return sep, mix, targets


def step(sep, mix, targets):
    sep.loss_and_gradients(mix, targets)
    sep.adam_step(LR)


def time_step(preset, batch, iters):
    sep, mix, targets = setup(preset, batch)
    for _ in range(3):
        step(sep, mix, targets)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        step(sep, mix, targets)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    flops = sep.engine(num_frames=mix.shape[1]).train_flops(batch)
    return {"preset": preset, "batch": batch, "step_ms": round(ms, 3), "conv_gflop": round(flops / 1e9, 3),
            "conv_tflops": round(flops / ms / 1e9, 3),
            "share_of_datasheet_fp32": round(flops / ms / 1e9 / DATASHEET_FP32_TFLOPS, 4)}


def profile(iters):
    from torch.profiler import ProfilerActivity, profile as tprofile
    sep, mix, targets = setup("unet_spectrogram", 4)
    for _ in range(3):
        step(sep, mix, targets)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            step(sep, mix, targets)
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            rows[e.key] = {"ms_per_step": round(e.device_time_total / 1e3 / iters, 4), "calls_per_step": e.count / iters}
    total = sum(r["ms_per_step"] for r in rows.values())
    return {"preset": "unet_spectrogram", "batch": 4, "kernel_ms_per_step": round(total, 3),
            "kernels": dict(sorted(rows.items(), key=lambda kv: -kv[1]["ms_per_step"]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spectrogram_train_table.py: no CUDA device")
    torch.cuda.set_device(0)
    if args.profile:
        res = {"profile": profile(args.iters)}
    else:
        res = {"steps": [time_step(p, b, args.iters) for p in ("unet_spectrogram", "unet_spectrogram_l1") for b in (4, 8)]}
    res["card"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
