"""Data parallelism for the Wave-U-Net engine: one process per GPU, torch.distributed for the plumbing.

The reference is single-device (SURVEY 2.2).  Training minibatches are independent through the whole network
(no batch-norm), so a step shards the batch over the ranks, every rank runs forward/backward on its shard with
the gradient pre-scaled by 1/world (the loss is a mean over the batch, /root/reference/Training.py:62), and ONE
all-reduce (sum) of the flat fp32 gradient buffer makes every replica apply the same Adam update.  Inference
windows (/root/reference/Evaluate.py:125-139) are independent: contiguous ranges per rank, no collective.

The spectrogram U-Net (U7 / U7a) has batch norm: its data-parallel step (sync_batch_norm) gathers every layer's
per-channel sums from all ranks through BatchStatsGather, so that each rank normalises with the whole batch's statistics.

Everything here works on CPU tensors with the gloo backend too (tests/test_parallel_cpu.py).
"""
import torch


def world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_range(n_items, rank, world_size):
    """Contiguous [lo, hi) of `n_items` for `rank`; sizes differ by at most one (first ranks get the extra)."""
    base, extra = divmod(int(n_items), int(world_size))
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(tensor, rank, world_size, dim=0):
    lo, hi = shard_range(tensor.shape[dim], rank, world_size)
    return tensor.narrow(dim, lo, hi - lo)


def grad_scale_for(local_batch, global_batch):
    """Factor each rank applies to its local mean-loss gradient so that the SUM over ranks is the gradient of the
    global mean loss (ranks may hold different numbers of examples)."""
    return float(local_batch) / float(global_batch)


def batch_loss_history(history, local_batch, global_batch, group=None):
    """Per-step mean losses of this rank's shard -> those of the whole batch, on every rank (in place): each rank weights
    its history by B_r / B and ONE all-reduce (sum) adds the ranks' histories - one collective per epoch, none per step."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        history.mul_(grad_scale_for(local_batch, global_batch))
        dist.all_reduce(history, op=dist.ReduceOp.SUM, group=group)
    return history


def allreduce_gradients(flat_grads, group=None):
    """The single collective of a training step: in-place sum of the flat gradient buffer over all ranks."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(flat_grads, op=dist.ReduceOp.SUM, group=group)
    return flat_grads


def bucket_offsets(param_table, n_buckets=4):
    """First flat offsets of `n_buckets` gradient buckets in PRODUCTION order (descending, last = 0) for
    Engine.set_grad_buckets.  Backward produces gradients from the end of the flat buffer (output convs, up blocks) to its
    start (first down block), layer by layer; buckets are cut at layer boundaries (a layer = consecutive table entries
    up to and including a '/bias'), with about the same number of layers each."""
    starts, cur = [], None
    for name, _, off, _ in param_table:
        if cur is None:
            cur = off
        if name.endswith("/bias"):
            starts.append(cur)
            cur = None
    if cur is not None:
        starts.append(cur)
    starts = sorted(set(starts), reverse=True)            # production order: highest offsets first
    n = max(1, min(int(n_buckets), len(starts)))
    per = len(starts) / float(n)
    firsts = []
    for k in range(1, n + 1):
        idx = min(len(starts) - 1, int(round(k * per)) - 1)
        o = 0 if k == n else starts[idx]
        if not firsts or o < firsts[-1]:
            firsts.append(o)
    if firsts[-1] != 0:
        firsts.append(0)
    return firsts


class BucketedAllReduce(object):
    """The step's single collective, overlapped with backward: the flat gradient buffer is all-reduced (sum) in buckets on
    a communication stream, each bucket as soon as the engine reports its gradients final (Engine.set_grad_buckets /
    stream_wait_grad_bucket), while the remaining backward kernels keep running on the compute stream.

        ar = BucketedAllReduce(engine, sep.grads)
        sep.loss_and_gradients(mix, targets, grad_scale=1/world)     # enqueue forward + backward
        ar.run()                                                     # enqueue the bucket all-reduces + the join
        sep.adam_step(lr)

    Plain stream / event ordering only, so the whole step (NCCL included) can be captured in one CUDA graph."""

    def __init__(self, engine, flat_grads, n_buckets=4, group=None):
        self.engine, self.grads, self.group = engine, flat_grads, group
        firsts = bucket_offsets(engine.param_table, n_buckets)
        engine.set_grad_buckets(firsts)
        his = [engine.param_numel] + firsts[:-1]
        self.views = [flat_grads[lo:hi] for lo, hi in zip(firsts, his)]
        self.comm = torch.cuda.Stream(device=flat_grads.device)
        self.done = torch.cuda.Event()

    def run(self):
        import torch.distributed as dist
        dev = self.grads.device
        cur = torch.cuda.current_stream(dev)
        for k, view in enumerate(self.views):
            self.engine.stream_wait_grad_bucket(k, self.comm)
            with torch.cuda.stream(self.comm):
                dist.all_reduce(view, op=dist.ReduceOp.SUM, group=self.group)
        self.done.record(self.comm)
        cur.wait_event(self.done)


class BatchStatsGather(object):
    """The shard of this rank in a data-parallel step of the spectrogram U-Net (wun.SpecEngine.forward_backward's `shard`):
    examples [sample_offset, sample_offset + local_batch) of `global_batch` (shard_range), and the all-gather of the
    batch-norm sums.  Under NCCL the gather is enqueued on the engine's stream, so a step stays capturable in a CUDA graph;
    under another backend (gloo) it waits for the stream and goes through host memory."""

    def __init__(self, global_batch, group=None):
        import torch.distributed as dist
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.global_batch = int(global_batch)
        lo, hi = shard_range(self.global_batch, self.rank, self.world)
        self.sample_offset, self.local_batch = lo, hi - lo
        self.nccl = dist.get_backend(group) == "nccl"

    def gather(self, local, gathered, stream):
        """Every rank's float64 CUDA tensor `local` [count] into `gathered` [world * count], rank r's at r * count."""
        import torch
        import torch.distributed as dist
        with torch.cuda.stream(stream):
            if self.nccl:
                dist.all_gather_into_tensor(gathered, local, group=self.group)
                return
            stream.synchronize()
            parts = [torch.empty(local.numel(), dtype=local.dtype) for _ in range(self.world)]
            dist.all_gather(parts, local.cpu(), group=self.group)
            gathered.copy_(torch.cat(parts))


def broadcast_parameters(flat_params, src=0, group=None):
    """Make every replica start from rank `src`'s variables (the DP invariant)."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.broadcast(flat_params, src=src, group=group)
    return flat_params


def max_over_ranks(value, device="cpu", group=None):
    """Timing reduction for benchmarks: the slowest rank defines the step time."""
    import torch.distributed as dist
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t.item())


def gather_window_predictions(local_preds, n_windows_total, group=None):
    """Inference: every rank predicted a contiguous range of windows [K, n_local, T_out, C]; returns the full
    [K, n_windows_total, T_out, C] on every rank (all_gather of padded shards)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local_preds
    ws, rank = dist.get_world_size(group), dist.get_rank(group)
    K, _, T, C = local_preds.shape
    max_local = (n_windows_total + ws - 1) // ws
    pad = torch.zeros((K, max_local, T, C), dtype=local_preds.dtype, device=local_preds.device)
    pad[:, :local_preds.shape[1]] = local_preds
    parts = [torch.empty_like(pad) for _ in range(ws)]
    dist.all_gather(parts, pad, group=group)
    out = []
    for r in range(ws):
        lo, hi = shard_range(n_windows_total, r, ws)
        out.append(parts[r][:, :hi - lo])
    return torch.cat(out, dim=1)
