"""GPU timing of the spectrogram U-Net baseline U7 (preset unet_spectrogram, random parameters, inference only).
   - the forward (wun.SpecEngine.forward, audio output) at batch 4 on 98 560-sample windows: CUDA events over --iters
     calls after a warm-up, against the FP32 bound from the shapes (2 FLOP per convolution MAC; 67 TFLOP/s is NVIDIA's
     data-sheet FP32 rate of the H100 SXM at up to 700 W, so the share is of that figure, not of this card's clock);
   - Evaluate.predict on 3 minutes of 44.1 kHz stereo: resampling to 8192 Hz and back included, host array in, host
     arrays out, host clock around work that ends in a device synchronise;
   - one Test.test pass (U7 MSE and U7a L1) over synthetic tracks staged into HBM at 8192 Hz (staging not timed).
Prints JSON with the card name, power limit and SM clock.
   python tools/spectrogram_table.py [--iters 20] [--out FILE]"""
import argparse
import json
import os
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
sys.path.insert(0, os.path.join(REPO, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import Config  # noqa: E402
import Datasets  # noqa: E402
import Evaluate  # noqa: E402
import Test  # noqa: E402
from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator  # noqa: E402
from conv_table import card  # noqa: E402
from dataset_fixtures import write_musdb  # noqa: E402
from oracle import spectrogram_oracle as S  # noqa: E402

DATASHEET_FP32_TFLOPS = 67.0
BATCH = 4


def model(preset):
    cfg = Config.build_config([preset], experiment_id=0)["model_config"]
    sep = UnetSpectrogramSeparator(cfg)
    sep.load_variables(S.random_params(cfg["num_layers"], cfg["num_initial_filters"], seed=1),
                       device=torch.device("cuda"), num_frames=cfg["num_frames"])
    return cfg, sep


def time_forward(cfg, sep, iters):
    eng = sep.engine(num_frames=cfg["num_frames"])
    g = torch.Generator().manual_seed(0)
    mix = (torch.rand((BATCH, eng.T_in, 1), generator=g) - 0.5).cuda()
    out = eng.forward(sep.params, mix, False)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        eng.forward(sep.params, mix, False, out=out)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    flops = eng.forward_flops(BATCH)
    return {"batch": BATCH, "window": int(eng.T_in), "launches": int(eng.launches(False)), "forward_ms": round(ms, 4),
            "gflop": round(flops / 1e9, 3), "achieved_tflops": round(flops / ms / 1e9, 3),
            "share_of_datasheet_fp32": round(flops / ms / 1e9 / DATASHEET_FP32_TFLOPS, 4)}


def time_predict(cfg, sep):
    rng = np.random.default_rng(7)
    audio = rng.uniform(-0.5, 0.5, size=(180 * 44100, 2)).astype(np.float32)
    Evaluate.predict(cfg, sep, audio[:44100 * 5], 44100)               # warm-up: workspaces, filter tables
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    Evaluate.predict(cfg, sep, audio, 44100)
    torch.cuda.synchronize()
    return {"seconds_of_audio": 180, "rate": 44100, "channels": 2, "predict_s": round(time.perf_counter() - t0, 4)}


def time_test(tmp):
    rows = {}
    tracks = {"t%d" % i: (8192, 8192 * 30 + 100 * i, 2, "float32") for i in range(4)}
    train = {"a": (8192, 8192 * 20, 1, "float32"), "b": (8192, 8192 * 20, 1, "float32")}
    musdb = write_musdb(os.path.join(tmp, "musdb"), train=train, test=tracks)
    for preset in ("unet_spectrogram", "unet_spectrogram_l1"):
        cfg, sep = model(preset)
        T = cfg["num_frames"]
        ds = Datasets.load_musdb(cfg, T, T, musdb, None, valid_tracks=1)
        Test.test(cfg, "test", "0", None, dataset=ds, separator=sep)          # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loss = Test.test(cfg, "test", "0", None, dataset=ds, separator=sep)
        torch.cuda.synchronize()
        p = ds.partitions["test"]
        n = len(Datasets.snippet_positions(p.offsets, p.lengths, T, T, cfg["batch_size"]))
        rows[preset] = {"snippets": n, "batch": cfg["batch_size"], "test_s": round(time.perf_counter() - t0, 4),
                        "loss": loss}
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spectrogram_table.py: no CUDA device")
    torch.cuda.set_device(0)
    cfg, sep = model("unet_spectrogram")
    res = {"forward": time_forward(cfg, sep, args.iters), "predict": time_predict(cfg, sep)}
    with tempfile.TemporaryDirectory() as tmp:
        res["test"] = time_test(tmp)
    res["card"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
