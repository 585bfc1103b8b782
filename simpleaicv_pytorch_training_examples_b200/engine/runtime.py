"""The one boundary between torch and a model runtime.

A runtime (``ResNetRT``, ``ViTRT``, ``DetrRT``, ...) runs a whole model forward and backward on the kernels of
libsaicv_b200.so; its nn.Module shell (``RuntimeModule``) hands it the batch through ``run``, and the loss tail stays in
torch.  ``run`` couples the two through one autograd node, and every runtime keeps this contract:

  * ``rt.forward(*inputs, training, keep_tape)`` returns ``(*outputs, tape)``; the tape, which holds what the backward
    needs, is None unless keep_tape.
  * ``rt.backward(*grads, tape)`` receives one gradient per differentiable output, each contiguous.  An output that
    took no part in the loss gets zeros of its shape (autograd materializes them for a Function).
  * The last ``rt.non_differentiable_outputs`` outputs (MAE's mask) are marked non-differentiable and get no gradient.
  * Parameter gradients never travel through autograd: the runtime writes them through its ``GradSink``, and the node
    fires ``sink.on_backward_end()`` once ``rt.backward`` has enqueued the whole backward pass.
"""
import contextlib

import torch
import torch.nn as nn

from . import syncbn


class GradSink:
    """Where parameter gradients go: ``param.grad`` by default, or bucket views supplied by the
    data-parallel wrapper (distributed.py) so that the all-reduce runs on flat buffers."""

    def __init__(self):
        self.views = {}       # id(param) -> fp32 tensor view with the parameter's shape
        self.on_ready = None  # callback(param) fired as soon as a gradient is complete
        self.on_backward_end = None  # callback() fired when the whole backward pass is enqueued

    def _buffer(self, param):
        """The buffer the gradient of `param` is written into; it holds param.grad when there is one."""
        buf = self.views.get(id(param))
        if buf is None:
            buf = self.views[id(param)] = torch.empty_like(param, dtype=torch.float32)
        if param.grad is not None and param.grad.data_ptr() != buf.data_ptr():
            buf.copy_(param.grad)
        return buf

    @contextlib.contextmanager
    def grad(self, *params):
        """``with sink.grad(*params) as (accumulate, *buffers):`` the body writes the gradient of each parameter into its
        buffer (parameter shape, fp32), adding to what the buffer holds when `accumulate`: a gradient is already there.
        The parameters share one flag because one kernel writes them, so they must agree on it.  On normal exit each buffer
        becomes its parameter's .grad and on_ready fires, in argument order; if the body raises, neither happens."""
        accumulate = params[0].grad is not None
        if any((p.grad is not None) != accumulate for p in params):
            raise RuntimeError('parameters whose gradients one kernel writes must all have a gradient or all have none; '
                               f'.grad is set on {[tuple(p.shape) for p in params if p.grad is not None]} only')
        bufs = [self._buffer(p) for p in params]
        yield (accumulate, *bufs)
        for p, buf in zip(params, bufs):
            p.grad = buf
            if self.on_ready is not None:
                self.on_ready(p)

    def add(self, param, g):
        """Writes `g`, a gradient computed in the parameter's shape: copied into the buffer, or added to the gradient
        already there."""
        with self.grad(param) as (accumulate, buf):
            if accumulate:
                buf.add_(g)
            else:
                buf.copy_(g)


class Runtime:
    """What every runtime owns: its GradSink and the units holding the bf16 weight-operand copies.  ``operands()``
    lists those copies for the fused optimizer in ``units`` order; ``prep()`` refreshes them before a forward."""

    non_differentiable_outputs = 0
    bn_group = None   # process group of synchronized BatchNorm (engine/syncbn.py), None: per-rank statistics

    def __init__(self, units):
        self.sink = GradSink()
        self._units = units

    def operands(self):
        return [u.op for u in self._units]

    def prep(self):
        for u in self._units:
            u.prep()


class _RuntimeFunction(torch.autograd.Function):
    """Torch differentiates the outputs; this node receives their gradients and runs the whole backward pass on the
    runtime's kernels.  No parameter is an input; the zero-dim ``anchor`` requires grad so that the outputs do.  The tape
    belongs to THIS forward (it lives on ctx), so several forwards of one module may be in flight before their
    backwards run."""

    @staticmethod
    def forward(ctx, anchor, rt, *inputs):
        ctx.rt, ctx.n_inputs = rt, len(inputs)
        with syncbn.exchanging(rt.bn_group):
            *outs, ctx.tape = rt.forward(*inputs, True, True)
        if rt.non_differentiable_outputs:
            ctx.mark_non_differentiable(*outs[-rt.non_differentiable_outputs:])
        return outs[0] if len(outs) == 1 else tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        tape, ctx.tape = ctx.tape, None
        assert tape is not None, 'the graph of this forward pass was already differentiated'
        rt = ctx.rt
        grads = grads[:len(grads) - rt.non_differentiable_outputs]
        with syncbn.exchanging(rt.bn_group):   # checkpointed stages re-run their forward (and its exchanges) in here
            rt.backward(*(g.contiguous() for g in grads), tape)
        if rt.sink.on_backward_end is not None:
            rt.sink.on_backward_end()
        return (None, None) + (None,) * ctx.n_inputs


def run(rt, training, *inputs):
    """Runs the runtime `rt` on `inputs`: its output, or the tuple of its outputs.  Builds a graph only in training
    with grad enabled; otherwise the forward keeps no tape."""
    if training and torch.is_grad_enabled():
        anchor = torch.zeros((), device=inputs[0].device, requires_grad=True)
        return _RuntimeFunction.apply(anchor, rt, *inputs)
    with torch.no_grad(), syncbn.exchanging(rt.bn_group):
        *outs, _ = rt.forward(*inputs, training, False)
    return outs[0] if len(outs) == 1 else tuple(outs)


class RuntimeModule(nn.Module):
    """Base of the nn.Module shells: parameter containers whose ``forward`` hands the batch to the runtime that the
    subclass's ``_build_runtime()`` makes."""

    def _runtime(self):
        rt = self.__dict__.get('_rt')
        if rt is None:
            rt = self.__dict__['_rt'] = self._build_runtime()  # not a submodule / not in state_dict
            rt.bn_group = self.__dict__.get('_bn_group')
        return rt

    def set_bn_group(self, group):
        """Synchronized BatchNorm (nn.SyncBatchNorm's semantics): in training, every BatchNorm of the model computes its
        statistics and gradient sums over all ranks of `group`, a process group dedicated to these exchanges (see
        engine/syncbn.py); None restores per-rank statistics.  Like the runtime, the group lives outside state_dict."""
        self.__dict__['_bn_group'] = group
        rt = self.__dict__.get('_rt')
        if rt is not None:
            rt.bn_group = group

    def grad_sink(self):
        """Where the runtime deposits parameter gradients (used by distributed.B200DataParallel)."""
        return self._runtime().sink

    def _run(self, *inputs):
        if not inputs[0].is_cuda:
            raise RuntimeError('this model runs on H100 kernels only; move the batch to the GPU (no CPU fallback exists)')
        return run(self._runtime(), self.training, *inputs)
