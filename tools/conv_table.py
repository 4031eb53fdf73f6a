"""Per-launch timing table of the M4 (batch 16) training step: every conv layer x pass (fwd, dgrad, wgrad) timed alone with
CUDA events (bench.layer_table), with GFLOP and TFLOP/s, the family sums, and the card, power limit and SM clock it ran on.
   python tools/conv_table.py [--out FILE]          (prints the JSON; --out also writes it to FILE)"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
import torch  # noqa: E402
import bench  # noqa: E402


def card():
    """Name, power limit and SM clocks of GPU 0, read now (nvidia-smi)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=True).stdout.strip().split(",")
    name, pl, sm, smax = (x.strip() for x in out)
    return {"name": name, "power_limit_w": float(pl), "sm_mhz_after": float(sm), "sm_max_mhz": float(smax)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=6, help="launches per (layer, pass) timing")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv_table.py: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    run = bench.TrainingRun(bench.PRESET, bench.BATCH_PER_GPU, bench.BATCH_PER_GPU, 0, 1, dev, None)
    with torch.cuda.stream(run.stream):
        run.step()
        run.stream.synchronize()
    rows, fam = bench.layer_table(run, iters=args.iters)
    res = {"workload": "M4 %s, batch %d, one training step, then every layer x pass alone" % (bench.PRESET, bench.BATCH_PER_GPU),
           "kernel_source_hash": bench.kernel_source_hash(), "lib": os.environ.get("WUN_LIB") or "in-tree libwun.so",
           "card": card(), "families": fam, "rows": rows}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
