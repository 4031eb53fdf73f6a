"""One data-parallel training step of the spectrogram U-Net under NCCL against the one-rank step at the same global batch, for
a box with several GPUs:

    torchrun --nproc-per-node N tools/spectrogram_dp_check.py [--preset unet_spectrogram_l1] [--batch 8] [--layers 6]

Every rank runs its shard with sync_batch_norm (wun.parallel.BatchStatsGather, all_gather_into_tensor on the engine's
stream), all-reduces the gradients, and compares with the whole batch run alone on its own GPU: the loss, the moving
statistics and the largest gradient difference relative to each tensor's largest value.  Rank 0 prints one JSON line.
"""
import argparse
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "wave-u-net_b200"))


def main():
    import torch
    import torch.distributed as dist

    import Config
    from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator
    from oracle import spectrogram_oracle as S
    from wun import parallel

    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="unet_spectrogram")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--layers", type=int, default=6)
    ap.add_argument("--filters", type=int, default=16)
    ap.add_argument("--frames", type=int, default=768 * 127 + 1024)
    args = ap.parse_args()

    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl")
    dev = torch.device("cuda", local_rank)
    cfg = Config.build_config([args.preset], dict(num_layers=args.layers, num_initial_filters=args.filters,
                                                  num_frames=args.frames), experiment_id=0)["model_config"]
    B, T = args.batch, args.frames
    params = S.random_params(args.layers, args.filters, seed=3)
    rng = np.random.default_rng(4)
    src = [rng.uniform(-0.25, 0.25, (B, T, 1)).astype(np.float32) for _ in range(2)]
    mix = torch.from_numpy(src[0] + src[1]).to(dev)
    tg = torch.from_numpy(np.stack(src)).to(dev)

    def separator():
        sep = UnetSpectrogramSeparator(cfg)
        sep.load_variables(params, device=dev, num_frames=T)
        return sep

    whole = separator()
    whole.loss_and_gradients(mix, tg)
    shard = parallel.BatchStatsGather(B)
    lo, n = shard.sample_offset, shard.local_batch
    dp = separator()
    dp.loss_and_gradients(mix[lo:lo + n].contiguous(), tg[:, lo:lo + n].contiguous(),
                          grad_scale=parallel.grad_scale_for(n, B), sync_batch_norm=shard)
    parallel.allreduce_gradients(dp.grads)
    loss = parallel.batch_loss_history(dp._loss.clone(), n, B)
    torch.cuda.synchronize()
    eng = dp.engine(num_frames=T)
    worst_grad, worst_moving = 0.0, 0.0
    for name, _, o, c in eng.param_table:
        a, b = dp.params[o:o + c].double(), whole.params[o:o + c].double()
        if name.endswith(("/moving_mean", "/moving_variance")):
            worst_moving = max(worst_moving, float(((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()))
        else:
            g, h = dp.grads[o:o + c].double(), whole.grads[o:o + c].double()
            worst_grad = max(worst_grad, float(((g - h).abs().max() / h.abs().max().clamp_min(1e-30)).item()))
    out = {"world": shard.world, "batch": B, "preset": args.preset, "loss_dp": float(loss[0].item()),
           "loss_one_rank": float(whole._loss[0].item()), "worst_moving_rel": worst_moving, "worst_grad_rel": worst_grad,
           "gpu": torch.cuda.get_device_name(dev)}
    worst = torch.tensor([worst_grad, worst_moving], dtype=torch.float64, device=dev)
    dist.all_reduce(worst, op=dist.ReduceOp.MAX)
    out["worst_grad_rel"], out["worst_moving_rel"] = [float(v) for v in worst.tolist()]
    if shard.rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
