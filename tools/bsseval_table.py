"""Per-stage timing of BSS Eval v4 on the GPU (wun.bss_eval) for a 3-minute, 44.1 kHz stereo input (the predict_3min_44k
length): the vocals/accompaniment scenario (2 sources) and 4 sources.  The whole call is timed with CUDA events; the
stages come from one profiled call (torch.profiler, kernels grouped by name).  Prints JSON with the card name, power limit
and SM clock, each stage's fp64 FLOPs from shapes, and the float64 oracle's CPU time on the same input.
   python tools/bsseval_table.py [--reps 3] [--no-oracle] [--out FILE]"""
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
from oracle import bsseval_oracle as B  # noqa: E402

N, RATE, L = 7938000, 44100, 512
STAGES = (("correlations", ("bss_xcorr", "bss_lag_reduce")), ("assembly", ("bss_assemble",)),
          ("solve", ("bss_ldl",)), ("framewise", ("bss_frame",)))


def stage_flops(nsrc, nchan, n, win, hop):
    """Algorithmic fp64 FLOPs (2 per multiply-add) of each stage."""
    nref, nwin, W = nsrc * nchan, (n - win) // hop + 1, win + L - 1
    g = (nref * L + nref * (nref - 1) // 2 * (2 * L - 1)) * n          # distinct lags of the reference pairs
    d = nref * nref * L * n
    big, small = nref * L, nchan * L
    solve = big ** 3 / 3 + nsrc * small ** 3 / 3 + 2 * big ** 2 * nref + 2 * small ** 2 * nchan * nsrc
    frames = nwin * nsrc * nchan * (nref + nchan) * L * W
    return {"correlations": 2.0 * (g + d), "assembly": 0.0, "solve": 2.0 * solve, "framewise": 2.0 * frames}


def inputs(nsrc, seed=0):
    rng = np.random.default_rng(seed)
    ref = rng.standard_normal((nsrc, N, 2)).astype(np.float32)
    est = (ref + 0.3 * np.roll(ref, 1, axis=0) + 0.1 * rng.standard_normal(ref.shape)).astype(np.float32)
    return ref, est


def measure(nsrc, reps, oracle):
    ref, est = inputs(nsrc)
    r, e = torch.from_numpy(ref).cuda(), torch.from_numpy(est).cuda()
    wun.bss_eval(r, e, RATE, RATE)                                   # warm-up: module load, allocator
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        wun.bss_eval(r, e, RATE, RATE)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        wun.bss_eval(r, e, RATE, RATE)
        torch.cuda.synchronize()
    ms = {s: 0.0 for s, _ in STAGES}
    for ev in prof.events():
        for s, prefixes in STAGES:
            if ev.device_type == torch.autograd.DeviceType.CUDA and any(p in ev.name for p in prefixes):
                ms[s] += ev.device_time / 1e3
    fl = stage_flops(nsrc, 2, N, RATE, RATE)
    row = {"nsrc": nsrc, "nchan": 2, "nsampl": N, "nwin": (N - RATE) // RATE + 1, "call_ms": times,
           "stages": {s: {"ms": round(ms[s], 3), "gflop": round(fl[s] / 1e9, 1),
                          "tflops": round(fl[s] / (ms[s] * 1e-3) / 1e12, 2) if ms[s] > 0 and fl[s] > 0 else None}
                      for s, _ in STAGES},
           "stages_sum_ms": round(sum(ms.values()), 3), "total_gflop": round(sum(fl.values()) / 1e9, 1)}
    if oracle:
        t0 = time.perf_counter()
        B.bss_eval(ref, est, RATE, RATE)
        row["oracle_cpu_s"] = round(time.perf_counter() - t0, 1)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bsseval_table.py: no CUDA device")
    rows = [measure(nsrc, args.reps, not args.no_oracle) for nsrc in (2, 4)]
    res = {"workload": "wun.bss_eval, 3 min 44.1 kHz stereo, win = hop = 1 s", "card": card(),
           "cpu_threads": os.cpu_count(), "rows": rows}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
