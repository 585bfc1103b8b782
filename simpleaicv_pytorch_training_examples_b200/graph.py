"""One CUDA graph per training step.

A step of the H100 runtime is several hundred small-to-medium kernel launches issued from Python through the C ABI
(ResNet-50: ~600, ViT-B: ~450).  When the host has to wait for every step's loss (tools/scripts.py reads it each
iteration, like the reference does), the launch work of step i+1 cannot be hidden behind step i and the GPU idles
for several milliseconds per step.  ``GraphedTrainStep`` captures forward + criterion + backward + optimizer step
once (torch.cuda.graph: the kernels, their tensor maps and all buffers of the step live in a private memory pool, so
addresses are stable) and replays it with ONE launch per step.

Constraints (checked / documented): fixed batch shape; the optimizer's hyper-parameters are baked at capture time
unless they are device tensors (use a tensor ``lr`` for per-iteration schedules; AdamW needs ``capturable=True``).
Under data parallelism the model may be the ``B200DataParallel`` wrapper: its bucket all-reduces (NCCL, issued on the
side stream from the backward's gradient-ready callbacks with event fork / join against the compute stream) are captured
into the same graph (measured at N = 2: 28.7 -> 27.4 ms per ResNet-50 step, end to end 34.6 -> 27.9 ms).  Dropout is
graph-safe: the runtimes draw one random word per forward on the device (captured: a new word every replay) and the
dropout / attention kernels add their per-site constants to it (saicv_dropout's seed_base), so the masks change from
step to step although the launch arguments are constants of the graph.
"""
import torch


class GraphedTrainStep:

    def __init__(self, model, criterion, optimizer, example_x, example_y, warmup=3):
        assert example_x.is_cuda, 'capture needs device-resident example inputs'
        self.model, self.criterion, self.optimizer = model, criterion, optimizer
        self.static_x = torch.empty_like(example_x)
        self.static_y = torch.empty_like(example_y)
        self.static_x.copy_(example_x)
        self.static_y.copy_(example_y)
        side = torch.cuda.Stream(example_x.device)
        side.wait_stream(torch.cuda.current_stream(example_x.device))
        with torch.cuda.stream(side):      # warm-up on a side stream (allocator / lazy-init work must not be captured)
            for _ in range(warmup):
                self._step_body()
        torch.cuda.current_stream(example_x.device).wait_stream(side)
        torch.cuda.synchronize(example_x.device)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.static_loss = self._step_body()

    def _step_body(self):
        loss = self.criterion(self.model(self.static_x), self.static_y)
        loss.backward()
        self.optimizer.step()
        self.optimizer.zero_grad()
        return loss.detach()

    def _replay(self):
        # fused optimizers (optim.py) read their hyper-parameters from a pinned table through a copy node of the graph:
        # per-iteration learning rates are a host write before the launch
        sync = getattr(self.optimizer, 'sync_hyper', None)
        if sync is not None:
            sync()
        self.graph.replay()
        if sync is not None:
            self.optimizer.after_replay()

    def replay(self):
        """Replays the step on the batch already in the static buffers; returns the loss tensor."""
        self._replay()
        return self.static_loss

    def __call__(self, x, y):
        """Runs one training step on (x, y) (device tensors of the captured shape); returns the loss tensor
        (valid until the next call)."""
        self.static_x.copy_(x, non_blocking=True)
        self.static_y.copy_(y, non_blocking=True)
        self._replay()
        return self.static_loss


class GraphedSplitStep:
    """Two CUDA graphs around an eager criterion, for steps whose loss needs the host (DETR's Hungarian matcher,
    detection/losses.py): graph A = model forward, then the criterion runs eagerly on the (detached) outputs and autograd
    gives their gradients, graph B = the runtime's backward + optimizer step + zero_grad, replayed with those gradients in
    static buffers.  Both graphs share one memory pool, so the activations A leaves on the runtime's tape are exactly what
    B reads.  ``model_fn(*inputs)`` returns a tensor or a list / tuple of tensors; ``criterion(outputs, targets)`` a scalar
    or a dict of loss terms (summed)."""

    def __init__(self, model_fn, criterion, optimizer, example_inputs, example_targets, warmup=3):
        dev = example_inputs[0].device
        self.model_fn, self.criterion, self.optimizer = model_fn, criterion, optimizer
        self.static_in = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):      # warm-up on a side stream (allocator / lazy-init work must not be captured)
            for _ in range(warmup):
                outs = self._as_list(model_fn(*self.static_in))
                self._loss(outs, example_targets).backward()
                optimizer.step()
                optimizer.zero_grad()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph_fwd = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph_fwd):
            self.outs = self._as_list(model_fn(*self.static_in))
        self.static_grads = [torch.zeros_like(o) for o in self.outs]
        self.graph_bwd = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph_bwd, pool=self.graph_fwd.pool()):
            torch.autograd.backward(self.outs, self.static_grads)
            optimizer.step()
            optimizer.zero_grad()

    @staticmethod
    def _as_list(o):
        return [o] if torch.is_tensor(o) else list(o)

    def _loss(self, outs, targets):
        value = self.criterion(outs if len(outs) > 1 else outs[0], targets)
        return sum(value.values()) if isinstance(value, dict) else value

    def __call__(self, inputs, targets):
        """One training step; returns the (eager) loss tensor."""
        for s, t in zip(self.static_in, inputs):
            s.copy_(t, non_blocking=True)
        self.graph_fwd.replay()
        leaves = [o.detach().requires_grad_(True) for o in self.outs]
        loss = self._loss(leaves, targets)
        grads = torch.autograd.grad(loss, leaves, allow_unused=True)
        for s, g in zip(self.static_grads, grads):
            if g is None:
                s.zero_()
            else:
                s.copy_(g)
        sync = getattr(self.optimizer, 'sync_hyper', None)
        if sync is not None:
            sync()
        self.graph_bwd.replay()
        if sync is not None:
            self.optimizer.after_replay()
        return loss.detach()
