"""Data-parallel wrapper replacing torch DDP for models executed by the H100 runtime
(reference: tools/utils.py:175-202 build_training_mode wraps the model in
nn.parallel.DistributedDataParallel; tools/scripts.py:168-181 uses ``model.no_sync()``).

One process per GPU.  Parameter gradients are produced by the runtime directly into flat fp32
buckets (reverse registration order, like DDP's reducer); as soon as every gradient of a bucket
has been written, the bucket is all-reduced (average) over NCCL on a side stream so that the
collective overlaps the remaining backward kernels.  The parameters whose gradients are produced
LAST (the first layers of the network) get a small bucket of their own (``tail_cap_mb``), so the
only all-reduce that cannot hide under backward compute is a short one.  There is no per-forward
buffer broadcast and no barrier; replicas start identical because rank 0's parameters and buffers
are broadcast once at construction, and every rank verifies at construction that all ranks built
the same bucket layout.  Parameters that receive no gradient in a step are reduced as zeros (fixed
bucket layout, SURVEY.md 8e).

A model whose parameters are written by several runtimes (distillation with a trainable teacher) returns the list of
their sinks from ``grad_sink()``; every runtime of the list must run its backward in every step, and the step's
gradients are complete, and the incomplete buckets reduced, once all of them have ended.
"""
import contextlib
import hashlib

import torch
import torch.distributed as dist
import torch.nn as nn


class _Bucket:
    def __init__(self, flat, params):
        self.flat = flat
        self.params = params      # [(param, view)]
        self.ready = set()
        self.work = None


class B200DataParallel(nn.Module):

    def __init__(self, module, process_group=None, bucket_cap_mb=25, tail_cap_mb=1, broadcast_from_rank0=True):
        super().__init__()
        self.module = module
        self.process_group = process_group
        self.world_size = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.require_sync = True
        params = [p for p in module.parameters() if p.requires_grad]
        assert params, 'no trainable parameters'
        self.device = params[0].device
        if broadcast_from_rank0 and self.world_size > 1:
            for t in list(module.parameters()) + list(module.buffers()):
                dist.broadcast(t.data, src=dist.get_global_rank(process_group, 0) if process_group else 0,
                               group=process_group)
        sinks = module.grad_sink()
        sinks = list(sinks) if isinstance(sinks, (list, tuple)) else [sinks]
        cap = max(1, int(bucket_cap_mb * 1024 * 1024) // 4)
        tail_cap = int(tail_cap_mb * 1024 * 1024) // 4
        # tail bucket: the leading parameters (registration order) whose gradients backward produces last
        n_tail, tail_n = 0, 0
        while tail_cap > 0 and n_tail < len(params) - 1 and tail_n + params[n_tail].numel() <= tail_cap:
            tail_n += params[n_tail].numel()
            n_tail += 1
        self.buckets, self.bucket_of = [], {}
        cur, cur_n = [], 0
        for p in reversed(params[n_tail:]):
            if cur and cur_n + p.numel() > cap:
                self._make_bucket(cur, sinks)
                cur, cur_n = [], 0
            cur.append(p)
            cur_n += p.numel()
        if cur:
            self._make_bucket(cur, sinks)
        if n_tail:
            self._make_bucket(list(reversed(params[:n_tail])), sinks)
        self._verify_layout_across_ranks()
        self._sinks, self._ended = sinks, set()
        for sink in sinks:
            sink.on_ready = self._param_ready
            sink.on_backward_end = lambda s=sink: self._sink_ended(s)
        self.comm_stream = torch.cuda.Stream(device=self.device) if self.device.type == 'cuda' else None

    def _make_bucket(self, params, sinks):
        total = sum((p.numel() + 63) // 64 * 64 for p in params)  # 256 B aligned views
        flat = torch.zeros(total, device=self.device, dtype=torch.float32)
        off, pv = 0, []
        for p in params:
            v = flat[off:off + p.numel()].view_as(p)
            for sink in sinks:      # a runtime only asks its sink for the views of its own parameters
                sink.views[id(p)] = v
            pv.append((p, v))
            off += (p.numel() + 63) // 64 * 64
        b = _Bucket(flat, pv)
        for p in params:
            self.bucket_of[id(p)] = b
        self.buckets.append(b)

    def layout_signature(self):
        """Digest of the bucket layout (bucket sizes and the shape of every view, in order)."""
        h = hashlib.sha256()
        for b in self.buckets:
            h.update(f'B{b.flat.numel()}:'.encode())
            for p, _ in b.params:
                h.update((','.join(map(str, p.shape)) + ';').encode())
        return int.from_bytes(h.digest()[:7], 'little')

    def _verify_layout_across_ranks(self):
        """A rank with a different model (or different requires_grad flags) would all-reduce buffers of
        another size or meaning: fail at construction instead of hanging or corrupting gradients."""
        if self.world_size <= 1:
            return
        sig = torch.tensor([self.layout_signature()], dtype=torch.int64, device=self.device)
        sigs = [torch.empty_like(sig) for _ in range(self.world_size)]
        dist.all_gather(sigs, sig, group=self.process_group)
        if any(int(s) != int(sig) for s in sigs):
            raise RuntimeError('B200DataParallel: ranks built different gradient-bucket layouts '
                               f'({[int(s) for s in sigs]}); the wrapped models differ across ranks')

    # ---- hooks fired by the runtime during backward
    def _param_ready(self, p):
        b = self.bucket_of.get(id(p))
        if b is None:
            return
        b.ready.add(id(p))
        if self.require_sync and self.world_size > 1 and len(b.ready) == len(b.params) and b.work is None:
            self._launch(b)

    def _launch(self, b):
        if self.comm_stream is not None:
            self.comm_stream.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self.comm_stream):
                b.work = dist.all_reduce(b.flat, op=dist.ReduceOp.AVG, group=self.process_group, async_op=True)
        else:  # gloo (CPU tests): no AVG
            b.work = dist.all_reduce(b.flat, op=dist.ReduceOp.SUM, group=self.process_group, async_op=True)

    def _sink_ended(self, sink):
        """The backward pass of one runtime is enqueued; the step's gradients are complete when every sink has ended."""
        self._ended.add(id(sink))
        if len(self._ended) == len(self._sinks):
            self._finish()

    def _finish(self):
        self._ended.clear()
        if self.require_sync and self.world_size > 1:
            for b in self.buckets:
                if b.work is None:
                    # Parameters that have no gradient at all take part as zeros.  A view that already
                    # holds a gradient accumulated under no_sync() (p.grad is the view) is kept even
                    # when this backward pass did not touch it.
                    for p, v in b.params:
                        if id(p) not in b.ready and p.grad is None:
                            v.zero_()
                            p.grad = v
                    self._launch(b)
            for b in self.buckets:
                b.work.wait()
                if self.comm_stream is None:
                    b.flat.div_(self.world_size)
                b.work = None
            if self.comm_stream is not None:
                torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
        for b in self.buckets:
            b.ready.clear()

    def reduce_now(self):
        """All-reduce (average) the current contents of every bucket, e.g. after backward passes run
        under no_sync().  Parameters without a gradient take part as zeros."""
        old, self.require_sync = self.require_sync, True
        try:
            for b in self.buckets:
                b.ready.update(id(p) for p, _ in b.params if p.grad is not None)
            self._finish()
        finally:
            self.require_sync = old

    @contextlib.contextmanager
    def no_sync(self):
        """Gradient accumulation: skip the all-reduce for backward passes run inside."""
        old, self.require_sync = self.require_sync, False
        try:
            yield
        finally:
            self.require_sync = old

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)


def overlap_self_check(ddp, step_fn):
    """Bit-exactness check of the overlapped bucket all-reduce (used by tests/ddp_check.py and, once per
    run, by bench.py at N > 1).  ``step_fn()`` must run one forward + backward of the SAME batch.

    Pass A: backward under no_sync(), then reduce_now() (no overlap: every gradient is complete before
    any collective starts).  Pass B: the production path (buckets all-reduced from the backward hooks
    while later kernels still run).  The kernels are deterministic and NCCL reduces equal-sized buffers
    in a fixed order, so the two passes must agree BIT FOR BIT; a race between the comm stream and the
    backward kernels would break that.  Returns the number of differing elements (0 = ok)."""
    params = [p for p in ddp.module.parameters() if p.requires_grad]
    for p in params:
        p.grad = None
    with ddp.no_sync():
        step_fn()
    ddp.reduce_now()
    a = [b.flat.clone() for b in ddp.buckets]
    for p in params:
        p.grad = None
    step_fn()
    torch.cuda.synchronize(ddp.device) if ddp.device.type == 'cuda' else None
    diff = sum(int((x != b.flat).sum()) for x, b in zip(a, ddp.buckets))
    for p in params:
        p.grad = None
    return diff
