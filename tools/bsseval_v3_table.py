"""Timing of BSS Eval v3 on the GPU (wun.bss_eval(..., mode="v3"): the filters solved for every one-second frame) for a
3-minute, 44.1 kHz stereo input with 2 and 4 sources, on the inputs tools/bsseval_table.py uses.  The whole call is timed
with CUDA events after a warm-up; the stages come from a separate profiled call (torch.profiler, kernels grouped by name).
Prints JSON with the card name, power limit and SM clock, each stage's algorithmic fp64 FLOPs, the factorization's achieved
FP64 rate, and the float64 oracle's CPU time on a sample of frames, extrapolated to the track.
   python tools/bsseval_v3_table.py [--reps 3] [--oracle-frames 3] [--out FILE]"""
import argparse
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import torch  # noqa: E402
import wun  # noqa: E402
from bsseval_table import L, N, RATE, inputs  # noqa: E402
from conv_table import card  # noqa: E402
from oracle import bsseval_v3_oracle as V3  # noqa: E402

STAGES = (("correlations", ("bss_xcorr", "bss_lag_reduce")), ("assembly", ("bss_assemble",)),
          ("factorization", ("bss_ldl_diag", "bss_ldl_panel", "bss_ldl_update")), ("solves", ("bss_ldl_solve",)),
          ("framewise", ("bss_frame",)))


def stage_flops(nsrc, nchan, n, win, hop):
    """Algorithmic fp64 FLOPs (2 per multiply-add) of each stage over every frame (none is silent in these inputs)."""
    nref, nwin, W = nsrc * nchan, (n - win) // hop + 1, win + L - 1
    g = (nref * L + nref * (nref - 1) // 2 * (2 * L - 1)) * win       # distinct lags of the reference pairs, per frame
    d = nref * nref * L * win
    big, small = nref * L, nchan * L
    return {"correlations": 2.0 * nwin * (g + d), "assembly": 0.0,
            "factorization": 2.0 * nwin * (big ** 3 / 6 + nsrc * small ** 3 / 6),
            "solves": 2.0 * nwin * (2 * big ** 2 * nref + 2 * small ** 2 * nchan * nsrc),
            "framewise": 2.0 * nwin * nsrc * nchan * (nref + nchan) * L * W}


def measure(nsrc, reps, oracle_frames):
    ref, est = inputs(nsrc)
    r, e = torch.from_numpy(ref).cuda(), torch.from_numpy(est).cuda()
    wun.bss_eval(r, e, RATE, RATE, mode="v3")                        # warm-up: module load, allocator
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        wun.bss_eval(r, e, RATE, RATE, mode="v3")
        b.record()
        torch.cuda.synchronize()
        times.append(round(a.elapsed_time(b), 2))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        wun.bss_eval(r, e, RATE, RATE, mode="v3")
        torch.cuda.synchronize()
    ms = {s: 0.0 for s, _ in STAGES}
    for ev in prof.events():
        for s, prefixes in STAGES:
            if ev.device_type == torch.autograd.DeviceType.CUDA and any(p in ev.name for p in prefixes):
                ms[s] += ev.device_time / 1e3
    fl = stage_flops(nsrc, 2, N, RATE, RATE)
    nwin = (N - RATE) // RATE + 1
    row = {"nsrc": nsrc, "nchan": 2, "nsampl": N, "nwin": nwin, "call_ms": times,
           "stages": {s: {"ms": round(ms[s], 3), "gflop": round(fl[s] / 1e9, 1),
                          "tflops": round(fl[s] / (ms[s] * 1e-3) / 1e12, 2) if ms[s] > 0 and fl[s] > 0 else None}
                      for s, _ in STAGES},
           "stages_sum_ms": round(sum(ms.values()), 3), "total_gflop": round(sum(fl.values()) / 1e9, 1)}
    if oracle_frames:
        step = nwin // oracle_frames
        t0 = time.perf_counter()
        for t in range(0, step * oracle_frames, step):
            V3.bss_eval_v3(*V3.frame_slices(ref, est, t, RATE, RATE), RATE, RATE)
        per = (time.perf_counter() - t0) / oracle_frames
        row["oracle_cpu"] = {"frames_run": oracle_frames, "s_per_frame": round(per, 2),
                             "track_s_extrapolated": round(per * nwin, 1)}
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-frames", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bsseval_v3_table.py: no CUDA device")
    rows = [measure(nsrc, args.reps, args.oracle_frames) for nsrc in (2, 4)]
    res = {"workload": "wun.bss_eval(mode='v3'), 3 min 44.1 kHz stereo, win = hop = 1 s",
           "workspace_cap_bytes": wun.BSS_V3_WORKSPACE_BYTES, "card": card(), "cpu_threads": os.cpu_count(), "rows": rows}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
