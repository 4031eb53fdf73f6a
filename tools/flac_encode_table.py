"""FLAC encode cost on the GPU (DESIGN.md §4.11): for 3 minutes of 44.1 kHz stereo (oracle/flac_oracle.py's test signal) at
16 and 24 bits, the device time of each encoder kernel (torch.profiler, in a run of its own), the host MD5 and assembly,
wun.write_flac end to end and the compression ratio; then Predict.main end to end with output_format=flac against the float
WAV output.  Prints the card and its power limit with the numbers.

    python tools/flac_encode_table.py [--repeats 5]
"""
import argparse
import glob
import os
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "wave-u-net_b200")]

import numpy as np  # noqa: E402
import scipy.io.wavfile  # noqa: E402
import torch  # noqa: E402

import wun  # noqa: E402
from oracle import flac_oracle as F  # noqa: E402
from wun import flac as W  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def kernel_ms(xd, bps, repeats):
    """Mean device ms per encode of each encoder kernel and of the output memset over `repeats` encodes (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    wun.write_flac(xd, 44100, bps)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(repeats):
            wun.write_flac(xd, 44100, bps)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "flac_" in ev.key or ev.key.startswith("Memset"):
            name = ev.key.split("flac_")[1].split("_kernel")[0] if "flac_" in ev.key else "memset"
            total = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            out[name] = out.get(name, 0.0) + total / 1e3 / repeats
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    print("card: %s" % card())
    for bps in (16, 24):
        x = F.signal(bps, 180 * 44100, 2, bps).astype(np.int32)
        xd = torch.from_numpy(x).cuda()
        ks = kernel_ms(xd, bps, a.repeats)
        ends, md5s, asm = [], [], []
        for _ in range(a.repeats + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            data = wun.write_flac(xd, 44100, bps)
            ends.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            W.md5_of(xd, bps)
            md5s.append((time.perf_counter() - t0) * 1e3)
            start = W.parse_stream(data).frames_start
            area = data[start:]
            off = np.linspace(0, len(area), (len(x) + 4095) // 4096 + 1).astype(np.int64)   # as many frames, even sizes
            t0 = time.perf_counter()
            W.assemble(area, off, 4096, 44100, 2, bps, len(x), bytes(16))
            asm.append((time.perf_counter() - t0) * 1e3)
        med = lambda v: float(np.median(v[1:]))  # noqa: E731
        print("%d-bit: %s (device ms per encode) | md5 %.1f ms, assembly %.2f ms (host) | write_flac %.1f ms | "
              "%.2f MB, ratio %.3f of the %d-bit PCM" % (bps, ", ".join("%s %.3f" % kv for kv in sorted(ks.items())),
                                                          med(md5s), med(asm), med(ends), len(data) / 1e6,
                                                          len(data) / (x.size * bps / 8), bps))
    # Predict.main end to end: the flagship preset (random weights) on a 3-minute 16-bit WAV, estimates as float WAV and FLAC
    import Config
    import Predict
    import Training
    from Models.UnetAudioSeparator import UnetAudioSeparator
    from oracle import wave_unet_oracle as O
    cfg = Config.build_config(["full_44KHz"], experiment_id=0)
    mc = cfg["model_config"]
    x = F.signal(16, 180 * 44100, 2, 16)
    with tempfile.TemporaryDirectory() as tmp:
        sep = UnetAudioSeparator(mc)
        t_in, _ = O.get_padding(mc, mc["num_frames"])
        sep.load_variables(O.init_params(mc, seed=1), input_frames=t_in)
        model = Training.save_checkpoint(os.path.join(tmp, "model.npz"), sep)
        scipy.io.wavfile.write(os.path.join(tmp, "song.wav"), 44100, x.astype(np.int16))
        runs = [("wav", None), ("flac", 16), ("flac", 24)]
        times = {r: [] for r in runs}
        for _ in range(3):
            for fmt, depth in runs:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                Predict.main(cfg, model, os.path.join(tmp, "song.wav"), output_path=os.path.join(tmp, "out_%s%s" % (fmt, depth)),
                             output_format=fmt, bit_depth=depth)
                torch.cuda.synchronize()
                times[(fmt, depth)].append(time.perf_counter() - t0)
        sizes = {r: sum(os.path.getsize(p) for p in glob.glob(os.path.join(tmp, "out_%s%s_*" % r)))
                 for r in runs}
        for r in runs:
            print("Predict.main full_44KHz, 3 min stereo, %s%s: %.2f s (median of 2 after a warm-up), estimates %.1f MB"
                  % (r[0], "" if r[1] is None else " %d-bit" % r[1], float(np.median(times[r][1:])), sizes[r] / 1e6))


if __name__ == "__main__":
    main()
