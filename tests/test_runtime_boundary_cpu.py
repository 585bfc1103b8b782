"""The autograd boundary of engine/runtime.py, driven on the CPU by a stand-in runtime made of plain torch ops that
keeps the runtime contract: forward(*inputs, training, keep_tape) -> (*outputs, tape), backward(*grads, tape); and the
GradSink that every runtime writes its parameter gradients through."""
import pytest
import torch

from simpleaicv_pytorch_training_examples_b200.engine.runtime import GradSink, Runtime, run


class _FakeRT(Runtime):
    """y = x * w and s = rowsum(x * w); with mask=True also a trailing non-differentiable (x > 0)."""

    def __init__(self, mask=False):
        super().__init__([])
        self.non_differentiable_outputs = int(mask)
        self.events = []

    def forward(self, x, w, training, keep_tape):
        self.events.append(('forward', training, keep_tape, torch.is_grad_enabled()))
        y = x * w
        outs = (y, y.sum(1)) + (((x > 0).float(),) if self.non_differentiable_outputs else ())
        return (*outs, {'x': x} if keep_tape else None)

    def backward(self, dy, ds, tape):
        self.events.append(('backward', tape['x'], dy, ds))


def _backwards(rt):
    return [e for e in rt.events if e[0] == 'backward']


def test_forwards_in_flight_each_backward_gets_its_own_tape():
    rt = _FakeRT()
    x1, x2, w = torch.randn(3, 4), torch.randn(3, 4), torch.tensor(2.)
    y1, _ = run(rt, True, x1, w)
    y2, _ = run(rt, True, x2, w)
    assert rt.events == [('forward', True, True, False)] * 2
    y2.sum().backward()
    y1.sum().backward()
    (_, t2, _, _), (_, t1, _, _) = _backwards(rt)
    assert t2 is x2 and t1 is x1


def test_second_backward_of_one_graph_raises():
    rt = _FakeRT()
    y, _ = run(rt, True, torch.randn(3, 4), torch.tensor(2.))
    loss = y.sum()
    loss.backward(retain_graph=True)
    with pytest.raises(AssertionError, match='the graph of this forward pass was already differentiated'):
        loss.backward()
    assert len(_backwards(rt)) == 1


def test_unused_output_gets_zeros_and_gradients_arrive_contiguous():
    rt = _FakeRT()
    y, s = run(rt, True, torch.randn(3, 4), torch.tensor(2.))
    (y.t() * torch.arange(12.).view(4, 3)).sum().backward()      # the gradient of y arrives transposed, s is unused
    [(_, _, dy, ds)] = _backwards(rt)
    assert dy.is_contiguous() and torch.equal(dy, torch.arange(12.).view(4, 3).t())
    assert ds.shape == s.shape and ds.is_contiguous() and not ds.any()


def test_non_differentiable_output_gets_no_gradient_slot():
    rt = _FakeRT(mask=True)
    y, s, m = run(rt, True, torch.randn(3, 4), torch.tensor(2.))
    assert y.requires_grad and s.requires_grad and not m.requires_grad
    (y.sum() + s.sum()).backward()       # _FakeRT.backward takes exactly the two differentiable gradients
    [(_, _, dy, ds)] = _backwards(rt)
    assert torch.equal(dy, torch.ones(3, 4)) and torch.equal(ds, torch.ones(3))


def test_on_backward_end_fires_once_after_the_runtime_backward():
    rt = _FakeRT()
    rt.sink.on_backward_end = lambda: rt.events.append(('end',))
    y, s = run(rt, True, torch.randn(3, 4), torch.tensor(2.))
    (y.sum() + s.sum()).backward()
    assert [e[0] for e in rt.events] == ['forward', 'backward', 'end']


@pytest.mark.parametrize('training,grad', [(False, True), (True, False), (False, False)])
def test_eval_and_no_grad_keep_no_tape_and_build_no_graph(training, grad):
    rt = _FakeRT(mask=True)
    with torch.set_grad_enabled(grad):
        outs = run(rt, training, torch.randn(3, 4), torch.tensor(2.))
    assert rt.events == [('forward', training, False, False)]
    assert len(outs) == 3 and all(o.grad_fn is None and not o.requires_grad for o in outs)


def _recording_sink():
    sink, ready = GradSink(), []
    sink.on_ready = ready.append
    return sink, ready


def test_grad_becomes_the_sink_buffer_and_each_parameter_is_reported_once_in_order():
    sink, ready = _recording_sink()
    w, b = torch.nn.Parameter(torch.ones(3, 2)), torch.nn.Parameter(torch.ones(3))
    with sink.grad(w, b) as (acc, wbuf, bbuf):
        assert not acc and wbuf.shape == w.shape and bbuf.shape == b.shape and wbuf.dtype == torch.float32
        assert w.grad is None and not ready        # nothing is published before the body has written the gradients
        wbuf.fill_(2.)
        bbuf.fill_(3.)
    assert w.grad is wbuf and b.grad is bbuf
    assert w.grad is sink.views[id(w)] and b.grad is sink.views[id(b)]
    assert [id(p) for p in ready] == [id(w), id(b)]


def test_accumulates_onto_an_existing_grad_held_in_another_tensor():
    sink, ready = _recording_sink()
    w = torch.nn.Parameter(torch.zeros(4))
    prev = torch.arange(4.)
    w.grad = prev
    with sink.grad(w) as (acc, buf):
        assert acc and buf is not prev and torch.equal(buf, prev)
        buf.add_(1.)
    assert w.grad is buf and torch.equal(w.grad, torch.arange(4.) + 1) and torch.equal(prev, torch.arange(4.))
    with sink.grad(w) as (acc, buf2):               # .grad is now the buffer itself: accumulate in place
        assert acc and buf2 is buf
        buf2.add_(1.)
    assert torch.equal(w.grad, torch.arange(4.) + 2) and len(ready) == 2


def test_a_raising_body_publishes_nothing():
    sink, ready = _recording_sink()
    w, b = torch.nn.Parameter(torch.ones(2)), torch.nn.Parameter(torch.ones(2))
    with pytest.raises(ValueError, match='kernel failed'):
        with sink.grad(w, b) as (_, wbuf, bbuf):
            wbuf.zero_()
            raise ValueError('kernel failed')
    assert w.grad is None and b.grad is None and not ready


@pytest.mark.parametrize('with_grad', ['first', 'second'])
def test_parameters_written_by_one_kernel_must_agree_on_accumulate(with_grad):
    sink, ready = _recording_sink()
    w, b = torch.nn.Parameter(torch.ones(2)), torch.nn.Parameter(torch.ones(2))
    has, other = (w, b) if with_grad == 'first' else (b, w)
    has.grad = torch.full((2,), 5.)
    with pytest.raises(RuntimeError, match='all have a gradient or all have none'):
        with sink.grad(w, b):
            pass
    assert other.grad is None and torch.equal(has.grad, torch.full((2,), 5.)) and not ready


def test_add_copies_the_first_gradient_and_adds_the_next():
    sink, ready = _recording_sink()
    w = torch.nn.Parameter(torch.ones(3))
    g = torch.tensor([-0., 1., 2.])
    sink.add(w, g)
    assert w.grad is sink.views[id(w)] and w.grad is not g
    assert torch.equal(w.grad, g) and torch.signbit(w.grad[0])     # a copy: -0.0 stays -0.0
    sink.add(w, g)
    assert torch.equal(w.grad, 2 * g) and [id(p) for p in ready] == [id(w)] * 2
