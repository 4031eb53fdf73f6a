"""FLAC decode cost on the GPU (DESIGN.md §4.10): for 3 minutes of 44.1 kHz stereo written by oracle/flac_oracle.py
(LPC order 12, mid/side, 4096-sample blocks) at 16 and 24 bits, the device time of the frame search and of the decode
(CUDA events), the host time of metadata parsing + chaining and of the MD5, and wun.read_flac end to end; then Predict.main
end to end on the same track as FLAC and as 16-bit WAV.  Prints the card and its power limit with the numbers.

    python tools/flac_table.py [--repeats 5]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "wave-u-net_b200")]

import ctypes  # noqa: E402

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


def device_passes(data, repeats):
    """(find ms, decode ms, host parse + chain ms, md5 ms) medians, with the kernels timed by CUDA events."""
    info = W.parse_stream(data)
    area = data[info.frames_start:]
    buf = torch.frombuffer(bytearray(area), dtype=torch.uint8).cuda()
    si = (info.bps, info.channels, info.rate, info.max_block)
    cap = len(area) // 256 + 1024
    rec = torch.empty((cap, ctypes.sizeof(wun.WunFlacFrame)), dtype=torch.uint8, device="cuda")
    count = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    rows = {k: [] for k in ("find", "decode", "parse", "md5")}
    for _ in range(repeats + 1):
        t0 = time.perf_counter()
        info = W.parse_stream(data)
        t_parse = time.perf_counter() - t0
        wun.check(wun.lib.wun_flac_find_frames(buf.data_ptr(), len(area), *si, rec.data_ptr(), cap, count.data_ptr(), stream))
        found = int(count.item())
        dtype = np.dtype([(n, np.int64 if t is ctypes.c_int64 else np.int32) for n, t in wun.WunFlacFrame._fields_])
        t0 = time.perf_counter()
        frames = rec[:found].cpu().numpy().view(dtype).reshape(-1)
        offsets, firsts, n = W.chain_frames(frames, len(area), info)
        t_parse += time.perf_counter() - t0
        out = torch.empty((n, info.channels), dtype=torch.int32, device="cuda")
        status = torch.zeros(len(offsets), dtype=torch.int32, device="cuda")
        od, fd = torch.from_numpy(offsets).cuda(), torch.from_numpy(firsts).cuda()
        e[1].record()
        wun.check(wun.lib.wun_flac_decode_frames(buf.data_ptr(), len(area), *si, od.data_ptr(), fd.data_ptr(), len(offsets),
                                                 out.data_ptr(), n, status.data_ptr(), stream))
        e[2].record()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        assert W.md5_of(out, info.bps) == info.md5
        t_md5 = time.perf_counter() - t0
        rows["decode"].append(e[1].elapsed_time(e[2]))
        rows["parse"].append(t_parse * 1e3)
        rows["md5"].append(t_md5 * 1e3)
    # the find pass alone, timed without the host work between the events
    for _ in range(repeats + 1):
        e[0].record()
        wun.check(wun.lib.wun_flac_find_frames(buf.data_ptr(), len(area), *si, rec.data_ptr(), cap, count.data_ptr(), stream))
        e[1].record()
        torch.cuda.synchronize()
        rows["find"].append(e[0].elapsed_time(e[1]))
    return {k: float(np.median(v[1:])) for k, v in rows.items()}, len(offsets)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    print("card: %s" % card())
    tracks = {}
    for bps in (16, 24):
        x = F.signal(bps, 180 * 44100, 2, bps)
        t0 = time.perf_counter()
        data = F.write(x, 44100, bps, block_size=4096, predictor=("lpc", 12, 14), channel_mode="mid_side", seed=bps)
        t_write = time.perf_counter() - t0
        tracks[bps] = (x, data)
        ms, nframes = device_passes(data, a.repeats)
        ends = []
        for _ in range(a.repeats + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            wun.read_flac(data)
            torch.cuda.synchronize()
            ends.append((time.perf_counter() - t0) * 1e3)
        print("%d-bit: %.1f MB, %d frames (writer %.1f s) | find %.3f ms, decode %.3f ms (device) | parse+chain %.2f ms, "
              "md5 %.2f ms (host) | read_flac %.1f ms" % (bps, len(data) / 1e6, nframes, t_write, ms["find"], ms["decode"],
                                                          ms["parse"], ms["md5"], float(np.median(ends[1:]))))
    # Predict.main end to end on the 16-bit track, from FLAC and from WAV (the flagship preset's model, random weights)
    import Config
    import Predict
    from Models.UnetAudioSeparator import UnetAudioSeparator
    from oracle import wave_unet_oracle as O
    import Training
    cfg = Config.build_config(["full_44KHz"], experiment_id=0)
    mc = cfg["model_config"]
    x, data = tracks[16]
    with tempfile.TemporaryDirectory() as tmp:
        sep = UnetAudioSeparator(mc)
        t_in, _ = O.get_padding(mc, mc["num_frames"])
        sep.load_variables(O.init_params(mc, seed=1), input_frames=t_in)
        model = Training.save_checkpoint(os.path.join(tmp, "model.npz"), sep)
        scipy.io.wavfile.write(os.path.join(tmp, "song.wav"), 44100, x.astype(np.int16))
        with open(os.path.join(tmp, "song.flac"), "wb") as f:
            f.write(data)
        times = {"wav": [], "flac": []}
        for _ in range(3):
            for fmt in ("wav", "flac"):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                Predict.main(cfg, model, os.path.join(tmp, "song." + fmt), output_path=os.path.join(tmp, "out_" + fmt))
                torch.cuda.synchronize()
                times[fmt].append(time.perf_counter() - t0)
        print("Predict.main full_44KHz, 3 min stereo: from WAV %.2f s, from FLAC %.2f s (median of 2 after a warm-up)"
              % tuple(float(np.median(times[f][1:])) for f in ("wav", "flac")))


if __name__ == "__main__":
    main()
