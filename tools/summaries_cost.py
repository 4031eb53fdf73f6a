"""GPU cost of the sep_loss summaries: Training.train epochs of --steps steps of baseline_stereo at batch 16 (the device-side
synthetic feeder), with summaries off and on, alternated --rounds times in one process so that both settings see the same
machine state.  Each epoch is timed with the host clock around train() (which ends with a checkpoint save and, with
summaries, the epoch's one device wait and the events file); the step time is that over --steps.  Prints JSON with every
epoch's time, the per-setting median and spread, and the card name, power limit and SM clock.
   python tools/summaries_cost.py [--steps 200] [--rounds 4] [--out FILE]"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import torch  # noqa: E402
import Config  # noqa: E402
import Training  # noqa: E402
from conv_table import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("summaries_cost.py: no CUDA device")
    torch.cuda.set_device(0)
    with tempfile.TemporaryDirectory() as tmp:
        cfg = Config.build_config(["baseline_stereo"], dict(batch_size=16, epoch_it=args.steps,
                                                            model_base_dir=os.path.join(tmp, "ck"),
                                                            log_dir=os.path.join(tmp, "logs")),
                                  experiment_id=1)["model_config"]
        _, sep = Training.train(dict(cfg, epoch_it=5), 1, log_every=0)         # warm-up: engine, feeder, workspace
        ms = {False: [], True: []}
        for r in range(args.rounds):
            for summaries in ((False, True) if r % 2 == 0 else (True, False)):
                torch.cuda.synchronize()
                t = time.perf_counter()
                _, sep = Training.train(dict(cfg), 1, sep=sep, log_every=0, summaries=summaries)
                torch.cuda.synchronize()
                ms[summaries].append((time.perf_counter() - t) * 1e3 / args.steps)
    res = {"preset": "baseline_stereo", "batch": 16, "steps_per_epoch": args.steps, "rounds": args.rounds}
    for summaries, name in ((False, "off"), (True, "on")):
        v = ms[summaries]
        res[name] = {"step_ms": [round(x, 4) for x in v], "median_step_ms": round(statistics.median(v), 4),
                     "spread_ms": round(max(v) - min(v), 4)}
    res["median_difference_ms"] = round(res["on"]["median_step_ms"] - res["off"]["median_step_ms"], 4)
    res["card"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
