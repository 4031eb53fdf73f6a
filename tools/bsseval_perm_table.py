"""Timing of museval's bss_eval switches on the GPU (wun.bss_eval(..., permutation=, sources_version=), wun_bss_eval_ex)
for a 3-minute, 44.1 kHz stereo input with 2 and 4 sources, on the inputs tools/bsseval_table.py uses: filters over the
whole track (v4) and per one-second frame (v3), each without and with the permutation search (images version; the sources
version differs in one energy per pair).  The whole call is timed with CUDA events after a warm-up; the stages come from a
separate profiled call (torch.profiler, kernels grouped by name).  Prints JSON with the card name, power limit and SM clock.
   python tools/bsseval_perm_table.py [--reps 3] [--out FILE]"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import torch  # noqa: E402
import wun  # noqa: E402
from bsseval_table import N, RATE, inputs  # noqa: E402
from conv_table import card  # noqa: E402

STAGES = (("correlations", ("bss_xcorr", "bss_lag_reduce")), ("assembly", ("bss_assemble",)),
          ("factorization", ("bss_ldl_diag", "bss_ldl_panel", "bss_ldl_update")), ("solves", ("bss_ldl_solve",)),
          ("framewise", ("bss_frame_energy",)), ("metrics", ("bss_frame_metrics", "bss_frame_silent", "bss_frame_list")),
          ("selection", ("bss_perm_select",)))


def measure(r, e, mode, permutation, reps):
    call = lambda: wun.bss_eval(r, e, RATE, RATE, mode=mode, permutation=permutation)   # noqa: E731
    call()                                                            # warm-up: module load, allocator
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        torch.cuda.synchronize()
        times.append(round(a.elapsed_time(b), 2))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    ms = {s: 0.0 for s, _ in STAGES}
    for ev in prof.events():
        for s, prefixes in STAGES:
            if ev.device_type == torch.autograd.DeviceType.CUDA and any(p in ev.name for p in prefixes):
                ms[s] += ev.device_time / 1e3
    return {"mode": mode, "permutation": permutation, "call_ms": times, "stages_ms": {s: round(v, 3) for s, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bsseval_perm_table.py: no CUDA device")
    rows = []
    for nsrc in (2, 4):
        ref, est = inputs(nsrc)
        r, e = torch.from_numpy(ref).cuda(), torch.from_numpy(est).cuda()
        for mode in ("v4", "v3"):
            for permutation in (False, True):
                rows.append(dict(nsrc=nsrc, **measure(r, e, mode, permutation, args.reps)))
    res = {"workload": "wun.bss_eval(permutation=False/True), 3 min 44.1 kHz stereo (%d samples), win = hop = 1 s" % N,
           "workspace_cap_bytes": wun.BSS_V3_WORKSPACE_BYTES, "card": card(), "rows": rows}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
