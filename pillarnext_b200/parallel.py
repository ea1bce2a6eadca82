"""Data-parallel plumbing for the frame-sharded path (SURVEY.md section 8e): one process per GPU, frames sharded by
the sampler, gradients averaged over the ranks (reference: torch DDP with 25 MB buckets overlapped with the backward,
tools/train.py:53-62).  BatchNorm statistics are local unless modules.enable_sync_batchnorm() is used.

BucketedGradAllReduce is this package's version of the DDP reducer for this model: the parameters are grouped into a few
buckets in backward order (head, neck, backbone + reader); a bucket is reduced as soon as the last of its gradients has
been accumulated -- one fused `cat` into a flat fp32 buffer, one NCCL all-reduce (NVLink/NVSwitch) and one fused copy
back, all on a side stream -- while the backward of the earlier layers is still running on the main stream.  Per step
that is ~3 x (1 cat + 1 all-reduce + 1 foreach copy) instead of one copy kernel per parameter."""
import torch
import torch.distributed as dist


def shard_frames(n_frames, rank, world):
    """DistributedSampler-style assignment (det3d/datasets/loader/build_loader.py:11-12): frame i -> rank i % world."""
    return list(range(rank, n_frames, world))


def _active():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


class FlatGradAllReduce:
    """Averages the gradients of `params` over the default process group with a single collective on a flat
    buffer (10.4 M fp32 = 41.5 MB for PillarNeXt-B) after the backward.  Works with NCCL (GPU) and gloo (CPU tests)."""

    def __init__(self, params):
        self.params = [p for p in params if p.requires_grad]

    def __call__(self):
        if not _active():
            return
        for p in self.params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        grads = [p.grad for p in self.params]
        flat = torch.cat([g.reshape(-1) for g in grads])                   # one fused kernel
        dist.all_reduce(flat)
        flat.div_(dist.get_world_size())
        torch._foreach_copy_(grads, [c.view_as(g) for c, g in zip(flat.split([g.numel() for g in grads]), grads)])


def default_buckets(model):
    """Buckets in backward order for SingleStageDetector: head | neck | backbone + reader."""
    groups = []
    for names in (("head",), ("neck",), ("backbone", "reader")):
        ps = [p for n in names if getattr(model, n, None) is not None for p in getattr(model, n).parameters() if p.requires_grad]
        if ps:
            groups.append(ps)
    seen = {id(p) for g in groups for p in g}
    rest = [p for p in model.parameters() if p.requires_grad and id(p) not in seen]
    if rest:
        groups.append(rest)
    return groups


class BucketedGradAllReduce:
    """Overlapped gradient averaging.  Usage:
        reducer = BucketedGradAllReduce(default_buckets(model))
        loss.backward(); reducer.finish(); optimizer.step()
    Every parameter of a bucket has a post-accumulate-grad hook; when the last one has fired the bucket is packed and
    all-reduced on `self.stream` (after an event recorded on the backward's stream).  finish() makes the current stream
    wait for the reductions and scatters the averaged values back into the .grad tensors."""

    def __init__(self, buckets):
        self.buckets = [[p for p in b if p.requires_grad] for b in buckets]
        self.buckets = [b for b in self.buckets if b]
        self.active = _active()
        self.stream = None
        self._pending, self._flat, self._work = [], [], []
        self._hooks = []
        if not self.active:
            return
        dev = self.buckets[0][0].device
        self.stream = torch.cuda.Stream(device=dev) if dev.type == "cuda" else None
        self._reset()
        for k, b in enumerate(self.buckets):
            for p in b:
                self._hooks.append(p.register_post_accumulate_grad_hook(lambda _p, k=k: self._ready(k)))

    def _reset(self):
        self._pending = [len(b) for b in self.buckets]
        self._flat = [None] * len(self.buckets)
        self._work = [None] * len(self.buckets)

    def _launch(self, k):
        grads = [p.grad if p.grad is not None else torch.zeros_like(p) for p in self.buckets[k]]
        if self.stream is not None:
            ev = torch.cuda.Event()
            ev.record()                                       # the gradients of this bucket are complete on the main stream
            with torch.cuda.stream(self.stream):
                self.stream.wait_event(ev)
                flat = torch.cat([g.reshape(-1) for g in grads])
                self._work[k] = dist.all_reduce(flat, async_op=True)
            for g in grads:
                g.record_stream(self.stream)
        else:
            flat = torch.cat([g.reshape(-1) for g in grads])
            self._work[k] = dist.all_reduce(flat, async_op=True)
        self._flat[k] = (flat, grads)

    def _ready(self, k):
        self._pending[k] -= 1
        if self._pending[k] == 0:
            self._launch(k)

    def finish(self):
        if not self.active:
            return
        world = dist.get_world_size()
        for k in range(len(self.buckets)):
            if self._flat[k] is None:                         # parameters that received no gradient this step
                self._launch(k)
            self._work[k].wait()                              # the current stream waits for the collective
            flat, grads = self._flat[k]
            if self.stream is not None:
                flat.record_stream(torch.cuda.current_stream())
            flat.div_(world)
            for p, g in zip(self.buckets[k], grads):
                if p.grad is None:
                    p.grad = g
            torch._foreach_copy_(grads, [c.view_as(g) for c, g in zip(flat.split([g.numel() for g in grads]), grads)])
        self._reset()

    def remove(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []
