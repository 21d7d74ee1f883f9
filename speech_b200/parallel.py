"""Data-parallel gradient synchronisation: one process per GPU, minibatch sharded B/N per rank,
the gradients summed over ranks once per step over NCCL (NVLink / NVSwitch).

The reference has no multi-GPU path at all (train.py:92, SURVEY.md §2.4); this adds exactly the
collective the north star names.  Gradients are SUMMED (not averaged): the reference's loss is a
sum over the minibatch (ctc_model.py:38-39), so the sum over ranks of per-shard gradients equals
the single-GPU gradient of the global batch.

All parameter gradients are views into one flat fp32 buffer (339.5 MB at the north-star config),
so `zero_grad(set_to_none=False)` is one memset and the all-reduce runs over contiguous slices of
it: one per GRU layer, started from inside the backward pass (BucketReducer), plus the rest.
"""
import torch


class BucketReducer:
    """Overlapped gradient all-reduce over one flat buffer (SURVEY.md §8e: "bucketed, issued from
    the GRU-backward wgrad epilogues so it overlaps").

    `ready(lo, hi)` is called while the backward pass is still running, as soon as every gradient
    inside flat[lo:hi] is final (speech_b200.ops calls it after each GRU layer's weight-gradient
    GEMMs have been enqueued).  The slice is all-reduced asynchronously: the process group's own
    stream waits for the work enqueued so far and then runs concurrently with the remaining layers
    (the persistent recurrence kernels leave 20 SMs free, which is where the NCCL channels run).
    `finish()` waits for those, then reduces whatever was not announced (conv, output layer, and
    everything when no hook fired) with one call per gap."""

    def __init__(self, flat, world_size, group=None):
        self.flat = flat
        self.world = world_size
        self.group = group
        self.pending = []     # (lo, hi, work)

    def ready(self, lo, hi):
        if self.world <= 1 or hi <= lo:
            return
        import torch.distributed as dist
        work = dist.all_reduce(self.flat[lo:hi], op=dist.ReduceOp.SUM, group=self.group,
                               async_op=True)
        self.pending.append((lo, hi, work))

    def finish(self):
        if self.world <= 1:
            return
        import torch.distributed as dist
        done = sorted((lo, hi) for lo, hi, _ in self.pending)
        pos, gaps = 0, []
        for lo, hi in done:
            if lo < pos:
                raise RuntimeError("overlapping gradient buckets [%d,%d) announced twice" % (lo, hi))
            if lo > pos:
                gaps.append((pos, lo))
            pos = hi
        if pos < self.flat.numel():
            gaps.append((pos, self.flat.numel()))
        works = [w for _, _, w in self.pending]
        for lo, hi in gaps:
            works.append(dist.all_reduce(self.flat[lo:hi], op=dist.ReduceOp.SUM, group=self.group,
                                         async_op=True))
        for w in works:
            w.wait()          # current stream waits; no host synchronisation on CUDA
        self.pending = []


class GradSync:
    def __init__(self, model, world_size, backend_group=None):
        self.world = world_size
        self.group = backend_group
        self.params = [p for p in model.parameters() if p.requires_grad]
        n = sum(p.numel() for p in self.params)
        dev = self.params[0].device
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        off = 0
        self.offsets = {}
        for p in self.params:
            p.grad = self.flat[off:off + p.numel()].view_as(p)
            self.offsets[id(p)] = (off, off + p.numel())
            off += p.numel()
        self.reducer = BucketReducer(self.flat, world_size, backend_group)

    def ready(self, params):
        """announce that the gradients of `params` (consecutive in parameter order) are final."""
        spans = [self.offsets[id(p)] for p in params]
        self.reducer.ready(min(s[0] for s in spans), max(s[1] for s in spans))

    def all_reduce(self):
        self.reducer.finish()

    def shard(self, items, rank):
        """contiguous B/N shard of a per-utterance list for `rank`."""
        if len(items) % self.world != 0:
            raise ValueError("minibatch of %d utterances is not divisible by world size %d"
                             % (len(items), self.world))
        per = len(items) // self.world
        return items[rank * per:(rank + 1) * per]
