"""Where the weight-gradient family's time goes: every conv layer's wgrad pass of the M4 (batch 16) training step run alone
(Engine.run_layer_pass, on the tensors one training step left in the workspace) under torch.profiler with CUDA activities, and
its kernel time split per layer into the split pass (split_views_kernel), the tensor-core wgrad (wgrad_umma_bulk_kernel) and the
fixed-order reduction (wgrad_reduce_kernel); the first layer's CUDA-core kernels are listed as "other".  Kernel times are summed
device durations from the trace, divided by the repetitions; the card, power limit and SM clock are read in the same run.
   python tools/wgrad_profile.py [--iters N] [--out FILE]          (prints the JSON; --out also writes it to FILE)"""
import argparse
import json
import os
import sys
from collections import defaultdict

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import torch  # noqa: E402
import bench  # noqa: E402
from conv_table import card  # noqa: E402

PARTS = (("split", "split_views_kernel"), ("wgrad", "wgrad_umma_bulk_kernel"), ("reduce", "wgrad_reduce_kernel"))


def part_of(kernel_name):
    for part, key in PARTS:
        if key in kernel_name:
            return part
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10, help="repetitions of each layer's wgrad pass inside the trace")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wgrad_profile.py: no CUDA device")
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    run = bench.TrainingRun(bench.PRESET, bench.BATCH_PER_GPU, bench.BATCH_PER_GPU, 0, 1, dev, None)
    L = run.cfg["num_layers"]
    names = ["down%d" % i for i in range(L)] + ["bottleneck"] + ["up%d" % i for i in range(L)]
    scratch = torch.zeros_like(run.sep.grads)
    with torch.cuda.stream(run.stream):
        run.step()
        for layer in range(2 * L + 1):                       # warm-up: every launch shape once
            run.eng.run_layer_pass(layer, 2, 1, run.sep.params, run.mix_d, scratch)
        run.stream.synchronize()
        rows = []
        for layer in range(2 * L + 1):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.iters):
                    run.eng.run_layer_pass(layer, 2, 1, run.sep.params, run.mix_d, scratch)
                run.stream.synchronize()
            us = defaultdict(float)
            for ev in prof.events():
                if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time_total > 0:
                    us[part_of(ev.name)] += ev.device_time_total / args.iters
            row = {"layer": names[layer], **{p: round(us.get(p, 0.0), 2) for p, _ in PARTS}, "other": round(us.get("other", 0.0), 2)}
            row["total"] = round(sum(us.values()), 2)
            rows.append(row)
    fam = {k: round(sum(r[k] for r in rows), 1) for k in ("split", "wgrad", "reduce", "other", "total")}
    res = {"workload": "M4 %s, batch %d: each layer's wgrad pass alone, kernel time per pass (us)" % (bench.PRESET, bench.BATCH_PER_GPU),
           "lib": os.environ.get("WUN_LIB") or "in-tree libwun.so", "card": card(), "family_us": fam, "rows": rows}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
