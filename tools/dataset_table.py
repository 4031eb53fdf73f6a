"""GPU timing of dataset staging (Datasets.stage_partition) and of one validation pass (Test.test).
   - Writes a synthetic MUSDB18-WAV-layout partition (--tracks tracks of --seconds at 44.1 kHz stereo, 16-bit PCM, five
     stems each) under a temporary directory, which is removed at the end.
   - Stages it for M4 baseline_stereo (22.05 kHz, stereo): host seconds for WAV reading, upload, and resampling + copy into
     the pool (device phases synchronised), summed over the tracks.
   - Test.test over the staged partition at batch 16 (random parameters): host seconds of a whole pass (it ends in its one
     synchronisation), the first pass (graph capture included) and the best of --reps; snippets per second.
   - CUDA events over --reps launches of each part of one batch: wun_snippet_batch, wun_forward (test mode) and
     wun_eval_batch_loss.
Prints JSON with the card name, power limit and SM clock.
   python tools/dataset_table.py [--tracks 10] [--seconds 180] [--reps 3] [--out FILE]"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import numpy as np  # noqa: E402
import scipy.io.wavfile  # noqa: E402
import torch  # noqa: E402
import wun  # noqa: E402
from conv_table import card  # noqa: E402

RATE, BATCH = 44100, 16


def write_partition(root, n_tracks, seconds):
    rng = np.random.default_rng(1337)
    for i in range(n_tracks):
        d = os.path.join(root, "train", "track_%02d" % i)
        os.makedirs(d)
        stems = {s: rng.integers(-8000, 8000, size=(seconds * RATE, 2), dtype=np.int16)
                 for s in ("bass", "drums", "other", "vocals")}
        stems["mixture"] = sum(v.astype(np.int32) for v in stems.values()).clip(-32768, 32767).astype(np.int16)
        for s, v in stems.items():
            scipy.io.wavfile.write(os.path.join(d, s + ".wav"), RATE, v)


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return [round(t, 4) for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=10)
    ap.add_argument("--seconds", type=int, default=180)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dataset_table.py: no CUDA device")
    import Config
    import Datasets
    import Test
    from Models.UnetAudioSeparator import UnetAudioSeparator
    mc = Config.build_config(["baseline_stereo"], dict(batch_size=BATCH), experiment_id=0)["model_config"]
    sep = UnetAudioSeparator(mc)
    in_shape, out_shape = sep.get_padding(np.array([BATCH, mc["num_frames"], 0]))
    t_in, t_out = int(in_shape[1]), int(out_shape[1])
    eng = sep.engine(input_frames=t_in)
    sep._ensure_params(eng, torch.device("cuda"), create=True)
    root = tempfile.mkdtemp(prefix="wun_dataset_table_")
    try:
        t0 = time.perf_counter()
        write_partition(root, args.tracks, args.seconds)
        t_write = time.perf_counter() - t0
        tracks = Datasets.musdb_tracks(root, "train")
        timings = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        part = Datasets.stage_partition(tracks, mc, t_in, t_out, timings=timings)
        t_stage = time.perf_counter() - t0
    finally:
        shutil.rmtree(root, ignore_errors=True)
    ds = Datasets.Dataset({"valid": part}, mc, t_in, t_out)
    n_snip = int(ds.positions("valid", BATCH).numel())
    passes = []
    for _ in range(1 + args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loss = Test.test(mc, "valid", "0", None, dataset=ds, separator=sep)
        passes.append(time.perf_counter() - t0)
    best = min(passes[1:])

    K, C = len(mc["source_names"]), 2
    pos = ds.positions("valid", BATCH)
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    mix = torch.empty((BATCH, t_in, C), device="cuda")
    tg = torch.empty((K, BATCH, t_out, C), device="cuda")
    out = torch.empty_like(tg)
    state = torch.zeros(2, dtype=torch.float64, device="cuda")
    slots = torch.empty(K * wun.EVAL_LOSS_CTAS, dtype=torch.float64, device="cuda")
    kernels = {
        "snippet_batch_ms": event_ms(lambda: wun.snippet_batch(part.pool, pos, BATCH, counter, mix, tg), args.reps),
        "forward_ms": event_ms(lambda: eng.forward(sep.params, mix, False, out=out), args.reps),
        "eval_batch_loss_ms": event_ms(lambda: wun.eval_batch_loss(out, tg, state, slots), args.reps),
        "snippet_batch_bytes": (BATCH * t_in * C + K * BATCH * t_out * C) * 4 * 2,
        "eval_batch_loss_bytes": 2 * K * BATCH * t_out * C * 4,
    }
    res = {"workload": "Datasets.stage_partition + Test.test, %d tracks x %d s of 44.1 kHz stereo PCM16, M4 baseline_stereo "
                       "(22.05 kHz), batch %d" % (args.tracks, args.seconds, BATCH),
           "card": card(), "t_in": t_in, "t_out": t_out,
           "write_fixture_s": round(t_write, 2),
           "staging_s": {"total": round(t_stage, 3), **{k: round(v, 3) for k, v in sorted(timings.items())}},
           "pool_bytes": int(part.pool.numel() * 4),
           "test_pass": {"snippets": n_snip, "batches": n_snip // BATCH, "first_s": round(passes[0], 4),
                         "best_s": round(best, 4), "all_s": [round(p, 4) for p in passes],
                         "snippets_per_s": round(n_snip / best, 1), "ms_per_batch": round(best / (n_snip // BATCH) * 1e3, 4),
                         "loss": loss},
           "per_batch_kernels": kernels}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
