"""GPU timing of kaiser_best resampling (wun.resample) and of the reference's predict() built on it (Evaluate.predict).
   - wun.resample on 3 minutes of 44.1 kHz stereo to 22.05 kHz, and that result back to 44.1 kHz: CUDA events, after a
     warm-up, with the FP64 operations each call needs (from the exact tap counts of the resampy loop) and their rate.
   - M4 baseline_stereo (random parameters): Evaluate.predict_track on the 3-minute track at 22.05 kHz against
     Evaluate.predict on the same track at 44.1 kHz (resampling in and out included); host clock around work that ends in
     a device synchronise, host array in, host arrays out.
Prints JSON with the card name, power limit and SM clock.
   python tools/resample_table.py [--reps 5] [--out FILE]"""
import argparse
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import wun  # noqa: E402
from conv_table import card  # noqa: E402
from oracle import resample_oracle as R  # noqa: E402

SECONDS, RATE, SR = 180, 44100, 22050
DATASHEET_FP64_TFLOPS = 34.0          # H100 SXM, non-tensor FP64, a DFMA counted as 2 operations


def taps(n_in, sr_in, sr_out):
    """Filter taps resampy's loop applies over all output frames (left + right wing of every frame)."""
    ratio = float(sr_out) / sr_in
    n_valid = int(n_in * ratio)
    scale, p = min(1.0, ratio), wun.KAISER_BEST_PRECISION
    step, nwin = int(scale * p), wun.KAISER_BEST_ZEROS * p + 1
    tr = R.time_register(n_valid, ratio)
    n = tr.astype(np.int64)
    frac = scale * (tr - n)
    total = 0
    for f, limit in ((frac, n + 1), (scale - frac, n_in - n - 1)):
        off = (f * p).astype(np.int64)
        total += int(np.maximum(np.minimum(limit, (nwin - off) // step), 0).sum())
    return total


def time_resample(x, sr_in, sr_out, reps):
    wun.resample(x, sr_in, sr_out)                                   # warm-up: module load, filter tables, allocator
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        y = wun.resample(x, sr_in, sr_out)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    n_taps = taps(x.shape[0], sr_in, sr_out)
    ops = n_taps * (2 + 2 * x.shape[1])                              # weight: mul + add; per channel: mul + add
    best = min(times)
    return y, {"sr_in": sr_in, "sr_out": sr_out, "frames_in": int(x.shape[0]), "frames_out": int(y.shape[0]),
               "channels": int(x.shape[1]), "call_ms": [round(t, 4) for t in times], "taps_per_frame": n_taps / y.shape[0],
               "fp64_gop": round(ops / 1e9, 3), "fp64_tops_per_s": round(ops / (best * 1e-3) / 1e12, 2),
               "share_of_datasheet_fp64": round(ops / (best * 1e-3) / 1e12 / DATASHEET_FP64_TFLOPS, 3)}


def time_host(fn, reps):
    fn()
    best = None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resample_table.py: no CUDA device")
    import Config
    import Evaluate
    from Models.UnetAudioSeparator import UnetAudioSeparator
    rng = np.random.default_rng(1337)
    audio = (rng.uniform(-1.0, 1.0, size=(SECONDS * RATE, 2)) * 0.5).astype(np.float32)
    x = torch.from_numpy(audio).cuda()
    down, row_down = time_resample(x, RATE, SR, args.reps)
    _, row_up = time_resample(down, SR, RATE, args.reps)
    mix22 = down.cpu().numpy()

    mc = Config.build_config(["baseline_stereo"], experiment_id=0)["model_config"]
    sep = UnetAudioSeparator(mc)
    in_shape, _ = sep.get_padding(np.array([1, mc["num_frames"], 0]))
    sep._ensure_params(sep.engine(input_frames=int(in_shape[1])), torch.device("cuda"), create=True)
    t_track = time_host(lambda: Evaluate.predict_track(mc, sep, mix22), args.reps)
    t_pred = time_host(lambda: Evaluate.predict(mc, sep, audio, RATE), args.reps)
    res = {"workload": "wun.resample and Evaluate.predict, 3 min of 44.1 kHz stereo (kaiser_best)", "card": card(),
           "datasheet_fp64_tflops": DATASHEET_FP64_TFLOPS,
           "resample": [row_down, row_up],
           "predict_m4_baseline_stereo": {"predict_track_22050_s": round(t_track, 4), "predict_44100_s": round(t_pred, 4),
                                          "resampling_overhead_s": round(t_pred - t_track, 4)}}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
